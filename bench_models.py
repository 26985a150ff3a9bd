"""Model-level harness for BASELINE.json configs 4 and 5 (`python bench.py --workload cfg4|cfg5`).

The generators are the REFERENCE'S OWN `PoseGenerator` / `FaceGenerator` (model/networks/generator.py:13-30,
388-426), byte-identical, from the git-ignored snapshot `baseline/_ref/` (baseline/snapshot.py) -- stock torch.nn
code that is out of scope to rewrite (SURVEY.md section 2 row 6) and serves as the harness around the warping ops.
Constructor arguments are the task models' (pose_model.py:62-64, face_model.py:78-80); weights are random
(orthogonal init, base_network.py:29-55), inputs synthetic.

Arms (what sits under `ExtractorAttn`, base_function.py:790-818):
  fused    this package's ExtractorAttn: conv logits + ONE fused local-attention kernel (the product path)
  literal  the reference's ExtractorAttn class, unchanged, on this package's unfused BlockExtractor / LocalAttnReshape
  refcuda  the reference's ExtractorAttn class on the reference's own CUDA kernels recompiled for sm_90a
           (oracle/_ref/libgfla_ref_cuda.so) -- the "patched reference ops" baseline of SURVEY.md section 8(d)

cfg4  PoseGenerator forward + backward under DistributedDataParallel (NCCL gradient all-reduce -- the only collective
      anywhere near this path), 256x256 (256x176 does not fit the reference's FlowNet, SURVEY.md section 7), batch 8 / GPU; img/s
cfg5  FaceGenerator inference (recurrent over 6 frames), 8 sequences / GPU; frames/s
"""
from __future__ import annotations

import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))

POSE_KW = dict(image_nc=3, structure_nc=18, ngf=64, img_f=512, layers=3, num_blocks=2, use_spect=False,
               attn_layer=[2, 3], norm="instance", activation="LeakyReLU", extractor_kz={"2": 5, "3": 3})
FACE_KW = dict(POSE_KW, structure_nc=16)


def reference_root():
    from baseline import snapshot
    if os.path.isdir("/root/reference/model/networks"):
        snapshot.snapshot()
    return snapshot.root()


def _purge():
    for name in [m for m in sys.modules if m == "model" or m.startswith("model.")]:
        del sys.modules[name]


def load_generators(arm: str):
    """-> (PoseGenerator, FaceGenerator) classes of the reference, wired to the chosen arm."""
    import types
    import torch
    import gfla_b200
    root = reference_root()
    if root is None:
        raise FileNotFoundError("baseline/_ref snapshot missing: run __graft_entry__.build() where /root/reference exists")
    _purge()
    gfla_b200.compat.install(reference_root=root, fuse_extractor_attn=(arm == "fused"))
    if arm == "refcuda":
        import oracle.ref_cuda as rc

        class BlockExtractor(torch.nn.Module):          # block_extractor.py:45-54 on the reference kernels
            def __init__(self, kernel_size=3):
                super().__init__()
                self.kernel_size = kernel_size

            def forward(self, source, flow_field):
                return rc.ExtractFn.apply(source.contiguous(), flow_field.contiguous(), self.kernel_size)

        class LocalAttnReshape(torch.nn.Module):        # local_attn_reshape.py:40-46
            def forward(self, inputs, kernel_size=3):
                return rc.ReshapeFn.apply(inputs.contiguous(), kernel_size)

        be = types.ModuleType("model.networks.block_extractor.block_extractor")
        be.BlockExtractor = BlockExtractor
        lr = types.ModuleType("model.networks.local_attn_reshape.local_attn_reshape")
        lr.LocalAttnReshape = LocalAttnReshape
        sys.modules[be.__name__], sys.modules[lr.__name__] = be, lr
    import importlib
    gen = importlib.import_module("model.networks.generator")
    return gen.PoseGenerator, gen.FaceGenerator


def _events(torch, n):
    return [torch.cuda.Event(enable_timing=True) for _ in range(n)]


def run(args):
    import torch
    import torch.distributed as dist
    from gfla_b200 import _lib
    from gfla_b200.sharding import reduce_max_time

    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    _lib.check(_lib.lib().gfla_device_check(), "device check")
    steps, warmup = max(1, args.steps), max(3, args.warmup)
    cfg4 = args.workload == "cfg4"
    dtype = torch.bfloat16 if args.model_dtype == "bf16" else torch.float32
    cl = args.model_dtype == "bf16"        # bf16 runs channels_last (the tile kernels' layout); fp32 keeps the reference's NCHW
    per_gpu = 8
    torch.manual_seed(1234 + rank)

    def barrier():
        if world > 1:
            dist.barrier(device_ids=[local_rank])
        torch.cuda.synchronize(dev)

    def make(arm):
        Pose, Face = load_generators(arm)
        torch.manual_seed(7)                               # identical weights on every rank and in every arm
        net = (Pose(**POSE_KW) if cfg4 else Face(**FACE_KW))
        net.init_weights("orthogonal")
        net = net.to(dev, dtype)
        if cl:
            net = net.to(memory_format=torch.channels_last)
        return net

    def inputs():
        g = torch.Generator(device="cpu").manual_seed(99 + rank)
        fmt = torch.channels_last if cl else torch.contiguous_format
        mk = lambda *s: torch.randn(*s, generator=g).to(dev, dtype)
        if cfg4:
            return [mk(per_gpu, 3, 256, 256).contiguous(memory_format=fmt), mk(per_gpu, 18, 256, 256).contiguous(memory_format=fmt),
                    mk(per_gpu, 18, 256, 256).contiguous(memory_format=fmt)]
        return [mk(per_gpu, 6, 16, 256, 256), mk(per_gpu, 3, 256, 256).contiguous(memory_format=fmt),
                mk(per_gpu, 16, 256, 256).contiguous(memory_format=fmt), None, None]

    results, launches, allreduce = {}, {}, None
    arms = [a for a in args.arms.split(",") if a]
    for arm in arms:
        try:
            net = make(arm)
        except Exception as exc:   # e.g. refcuda library not built on this box
            results[arm] = {"unavailable": repr(exc)[:200]}
            continue
        x = inputs()
        if cfg4:
            model = torch.nn.parallel.DistributedDataParallel(net, device_ids=[local_rank]) if world > 1 else net
            target = torch.randn(per_gpu, 3, 256, 256, device=dev, dtype=dtype)

            def step():
                model.zero_grad(set_to_none=True)
                img, flows, masks = model(*x)
                loss = (img - target).abs().mean() + sum(f.float().pow(2).mean() for f in flows) * 1e-3
                loss.backward()                              # DDP: bucketed NCCL all-reduce of net_G's gradients
                return loss.detach()
        else:
            net.eval()

            def step():
                with torch.no_grad():
                    imgs, _, _, _ = net(*x)
                return imgs[-1].float().mean()

        try:
            for _ in range(warmup):
                step()
            err = None
        except Exception as exc:       # e.g. the reference's kernels have no bf16 (AT_DISPATCH_FLOATING_TYPES: float, double)
            err = repr(exc)[:200]
        flag = torch.tensor([1.0 if err else 0.0], device=dev)
        if world > 1:
            dist.all_reduce(flag)
        if flag.item() > 0:
            results[arm] = {"unavailable": err or "failed on another rank"}
            del net, x
            torch.cuda.empty_cache()
            continue
        barrier()
        n0 = _lib.lib().gfla_debug_launch_count()
        ev = _events(torch, 2)
        ev[0].record()
        for _ in range(steps):
            loss = step()
        ev[1].record()
        barrier()
        ms = reduce_max_time(ev[0].elapsed_time(ev[1]), dev) / steps
        units = per_gpu * world * (1 if cfg4 else 6)
        results[arm] = {"value": units / (ms * 1e-3), "ms_per_step": ms, "loss": float(loss)}
        launches[arm] = int(_lib.lib().gfla_debug_launch_count() - n0)
        # share of the step spent in the warping ops and in NCCL, from one profiled step (CUPTI, in-process)
        if arm == arms[0]:
            try:
                from torch.profiler import profile, ProfilerActivity
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    step()
                    torch.cuda.synchronize(dev)
                tot = nccl = ours = 0.0
                for e in prof.key_averages():
                    t = float(getattr(e, "device_time_total", 0.0) or getattr(e, "cuda_time_total", 0.0))
                    tot += t
                    if "nccl" in e.key.lower():
                        nccl += t
                    if "gfla::" in e.key or "k_local_attn" in e.key or "k_block_extract" in e.key or "k_attn_reshape" in e.key:
                        ours += t
                results[arm]["kernel_time_share"] = {"warp_ops": ours / tot if tot else None, "nccl_allreduce": nccl / tot if tot else None,
                                                     "device_kernel_ms": tot / 1e3}
                if cfg4 and world > 1:
                    nbytes = sum(p.numel() * p.element_size() for p in net.parameters())
                    allreduce = {"bytes_per_step": nbytes, "nccl_kernel_ms": nccl / 1e3, "share_of_kernel_time": nccl / tot if tot else None}
            except Exception as exc:
                results[arm]["kernel_time_share"] = {"error": repr(exc)[:120]}
        del net, x
        torch.cuda.empty_cache()

    if rank == 0:
        main_arm = arms[0]
        r = results.get(main_arm, {})
        line = {"metric": "PoseGenerator fwd+bwd img/s (DDP)" if cfg4 else "FaceGenerator inference frames/s",
                "value": r.get("value"), "unit": "img/s" if cfg4 else "frames/s", "n_gpus": world, "steps": steps, "warmup": warmup,
                "ms_per_step": r.get("ms_per_step"), "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
                "dtype": args.model_dtype, "data": "synthetic",
                "config": {"workload": f"{args.workload}: reference {'PoseGenerator' if cfg4 else 'FaceGenerator'} (random orthogonal init), "
                                       f"{per_gpu} {'images' if cfg4 else 'sequences x 6 frames'} per GPU, 256x256, attn_layer=2,3 kernel=5,3, "
                                       f"{'forward+backward, DDP' if cfg4 else 'inference'}", "arm": main_arm,
                           "layout": "channels_last" if cl else "contiguous NCHW", "per_gpu_batch": per_gpu},
                "arms": results, "gpu_launches": launches.get(main_arm), "gpu_launches_by_arm": launches, "allreduce": allreduce}
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()
    return 0
