"""Per-op timings at BASELINE.json's configurations (CUDA events, warm-up 3, mean of N) -> JSON lines.
Secondary to bench.py (which carries the headline contract)."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from gfla_b200 import functional as F_
PEAK = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists("MEASURED_PEAKS.json") else 3350.0   # H100 SXM data sheet
dev = "cuda:0"

def timed(fn, n=5, w=3):
    for _ in range(w): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n

def emit(name, ms, px, alg_bytes, **kw):
    print(json.dumps({"op": name, "ms": round(ms, 4), "Mpixels_per_s": round(px / ms / 1e3, 1),
                      "algorithmic_GB": round(alg_bytes / 1e9, 3), "GBps": round(alg_bytes / ms / 1e6, 1),
                      "frac_of_measured_hbm_peak": round(alg_bytes / ms / 1e6 / PEAK, 4), **kw}), flush=True)

def smooth(B, H, W):
    c = (torch.rand(B, 2, H // 16, W // 16, device=dev) * 16 - 8)
    return torch.nn.functional.interpolate(c, size=(H, W), mode="bilinear", align_corners=True).contiguous()

which = sys.argv[1:] or ["cfg3", "cfg2_unfused", "cfg2_fp32", "module"]
torch.manual_seed(0)
if "cfg3" in which:   # resample2d fwd+bwd, B=32 C=128 512x512 fp32 (BASELINE.json configs[2]); ks=2 sigma=5 and ks=4 sigma=2
    B, C, H, W = 32, 128, 512, 512
    x = torch.randn(B, C, H, W, device=dev)
    g = torch.randn(B, C, H, W, device=dev)
    # "blocky" = nearest-neighbour x16 up-sampling of a coarse flow + sub-pixel jitter, the shape PerceptualCorrectness feeds
    # (external_function.py:243: F.interpolate(flow, [h, w]), default mode 'nearest'): constant integer tap shift per block
    coarse = (torch.rand(B, 2, H // 16, W // 16, device=dev) * 16 - 8).floor() + 0.25
    blocky = (torch.nn.functional.interpolate(coarse, size=(H, W), mode="nearest") + 0.5 * torch.rand(B, 2, H, W, device=dev)).contiguous()
    for ks, sigma in ((2, 5.0), (4, 2.0)):
        px = B * H * W
        for fname, fl in (("smooth", smooth(B, H, W)), ("blocky", blocky)):
            in2 = torch.cat([fl, torch.full((B, 1, H, W), sigma, device=dev)], 1).contiguous()
            f = timed(lambda: F_.resample2d_fwd(x, in2, ks, 1))
            b = timed(lambda: F_.resample2d_bwd(x, in2, g, ks, 1), n=3, w=1)
            emit(f"resample2d_fwd ks={ks} {fname} flow", f, px, px * (2 * C * 4 + 12), config="cfg3 B=32 C=128 512x512 fp32")
            emit(f"resample2d_bwd ks={ks} {fname} flow", b, px, px * (3 * C * 4 + 24), config="cfg3")
            emit(f"resample2d_fwd+bwd ks={ks} {fname} flow", f + b, px, px * (5 * C * 4 + 36), config="cfg3")
if "cfg2_unfused" in which:   # the unfused ops at cfg2-like size (B=2: the [B,C,kH,kW] block tensor is 25x the input)
    B, C, H, W, k = 2, 256, 256, 256, 5
    s = torch.randn(B, C, H, W, device=dev).bfloat16(); fl = smooth(B, H, W)
    px = B * H * W
    t = timed(lambda: F_.block_extract_fwd(s, fl, k))
    emit("block_extract_fwd bf16 k=5", t, px, px * (C * 2 + C * 2 * k * k + 8), config="B=2 C=256 256x256")
    a = torch.randn(B, k * k, H, W, device=dev).bfloat16()
    t = timed(lambda: F_.attn_reshape_fwd(a, k))
    emit("attn_reshape_fwd bf16 k=5", t, px, px * (2 * k * k * 2), config="B=2 256x256")
if "cfg2_fp32" in which:   # fused op in fp32 (CUDA-core gather kernels), B=4
    B, C, H, W, k = 4, 256, 256, 256, 5
    s = torch.randn(B, C, H, W, device=dev); fl = smooth(B, H, W); l = torch.randn(B, k * k, H, W, device=dev); g = torch.randn(B, C, H, W, device=dev)
    px = B * H * W
    t = timed(lambda: F_.local_attn_fwd(s, fl, l, k))
    emit("local_attn_fwd fp32 (gather kernel)", t, px, px * (2 * C * 4 + 8 + k * k * 4), config="B=4 C=256 256x256 k=5")
    t = timed(lambda: F_.local_attn_bwd(s, fl, l, g, k), n=2, w=1)
    emit("local_attn_bwd fp32 (gather kernel, scalar atomics)", t, px, px * (3 * C * 4 + 16 + 2 * k * k * 4), config="B=4 C=256 256x256 k=5")

if "patch_conv" in which:   # ExtractorAttn's source-half conv: materialised (BlockExtractor + cuDNN) vs patch_conv, bf16 channels-last
    import subprocess
    import gfla_b200
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    card = q.stdout.strip() or torch.cuda.get_device_name(0)
    torch.backends.cudnn.allow_tf32 = False
    for (B, C, HW, k) in ((8, 256, 32, 3), (8, 128, 64, 5), (2, 256, 256, 5)):
        cl = torch.channels_last
        src = torch.randn(B, C, HW, HW, device=dev).bfloat16().contiguous(memory_format=cl).requires_grad_()
        flow = smooth(B, HW, HW).requires_grad_()
        w = (torch.randn(128, C, k, k, device=dev) / (C * k * k) ** 0.5).bfloat16().requires_grad_()
        g = torch.randn(B, 128, HW, HW, device=dev).bfloat16().contiguous(memory_format=cl)
        ex = gfla_b200.BlockExtractor(k)
        arms = {"materialised": lambda: torch.nn.functional.conv2d(ex(src, flow), w, None, stride=k),
                "patch_conv": lambda: gfla_b200.patch_conv(src, flow, w, k)}
        with torch.no_grad():
            outs = {a: fn() for a, fn in arms.items()}
        diff = (outs["patch_conv"].float() - outs["materialised"].float()).abs().max().item()
        del outs
        res = {a: {"fwd": [], "fwd_bwd": []} for a in arms}
        for rep in range(5):                      # alternate the arms so that clocks and heat affect both alike
            for a, fn in arms.items():
                with torch.no_grad():
                    res[a]["fwd"].append(timed(fn, n=5, w=2))
                res[a]["fwd_bwd"].append(timed(lambda: fn().backward(g), n=3, w=1))
        gflop = 2 * B * HW * HW * 128 * C * k * k / 1e9
        for a, fn in arms.items():
            src.grad = flow.grad = w.grad = None
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            fn().backward(g)
            torch.cuda.synchronize()
            peak = torch.cuda.max_memory_allocated() - base
            f, fb = sorted(res[a]["fwd"])[2], sorted(res[a]["fwd_bwd"])[2]
            print(json.dumps({"op": f"patch conv, {a}", "config": f"B={B} C={C} {HW}x{HW} k={k} N=128 bf16 channels_last",
                              "fwd_ms": round(f, 4), "fwd_bwd_ms": round(fb, 4),
                              "fwd_TFLOPs": round(gflop / f, 2), "fwd_bwd_TFLOPs": round(3 * gflop / fb, 2),
                              "frac_of_989_TFLOPs_fwd_bwd": round(3 * gflop / fb / 989.0, 4),
                              "peak_MB_above_inputs_fwd_bwd": round(peak / 2 ** 20, 1),
                              "max_abs_diff_vs_materialised": diff, "card_and_power_limit": card,
                              "timing": "CUDA events, median of 5 alternating rounds"}), flush=True)
        del src, flow, w, g
        torch.cuda.empty_cache()

if "det" in which:   # torch.use_deterministic_algorithms(True) against the default mode, alternated in one process
    import statistics
    import subprocess
    from torch.profiler import ProfilerActivity, profile
    from gfla_b200.extractor_attn import PatchConvFunction
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    card = q.stdout.strip() or torch.cuda.get_device_name(0)
    cl = torch.channels_last
    B, C, HW, k = 16, 256, 256, 5          # cfg2
    src = torch.randn(B, C, HW, HW, device=dev).bfloat16().contiguous(memory_format=cl)
    flow = smooth(B, HW, HW)
    logits = torch.randn(B, k * k, HW, HW, device=dev).bfloat16()
    gout = torch.randn(B, C, HW, HW, device=dev).bfloat16().contiguous(memory_format=cl)

    def step():
        F_.local_attn_fwd(src, flow, logits, k)
        F_.local_attn_bwd(src, flow, logits, gout, k)

    def bwd():
        F_.local_attn_bwd(src, flow, logits, gout, k)

    def in_mode(det, fn):
        torch.use_deterministic_algorithms(det)
        try:
            return fn()
        finally:
            torch.use_deterministic_algorithms(False)

    res = {False: {"step": [], "bwd": []}, True: {"step": [], "bwd": []}}
    for _ in range(5):
        for det in (False, True):
            res[det]["step"].append(in_mode(det, lambda: timed(step, n=5, w=2)))
            res[det]["bwd"].append(in_mode(det, lambda: timed(bwd, n=5, w=2)))
    peak = {}
    for det in (False, True):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        in_mode(det, step)
        torch.cuda.synchronize()
        peak[det] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)

    def breakdown(det):
        in_mode(det, bwd)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            in_mode(det, bwd)
            torch.cuda.synchronize()
        parts = {"pre-pass (k_fx_amax, k_fx_exponents)": 0.0, "memset": 0.0, "backward kernel": 0.0, "k_fold_border": 0.0,
                 "narrowing (k_fx_narrow)": 0.0, "other": 0.0}
        for e in prof.key_averages():
            us = getattr(e, "device_time_total", 0.0) or getattr(e, "cuda_time_total", 0.0)
            n = e.key
            key = ("pre-pass (k_fx_amax, k_fx_exponents)" if ("k_fx_amax" in n or "k_fx_exponents" in n) else
                   "memset" if "emset" in n else "backward kernel" if "k_local_attn_bwd" in n else
                   "k_fold_border" if "k_fold_border" in n else "narrowing (k_fx_narrow)" if "k_fx_narrow" in n else "other")
            parts[key] += us / 1e3
        return {a: round(b, 4) for a, b in parts.items()}

    med = lambda v: round(statistics.median(v), 4)
    print(json.dumps({"op": "local attention fwd+bwd, default vs deterministic mode",
                      "config": f"cfg2: B={B} C={C} {HW}x{HW} k={k} bf16 channels_last, smooth flow",
                      "step_ms": {"default": med(res[False]["step"]), "deterministic": med(res[True]["step"])},
                      "bwd_ms": {"default": med(res[False]["bwd"]), "deterministic": med(res[True]["bwd"])},
                      "step_ms_all": {"default": [round(v, 4) for v in res[False]["step"]],
                                      "deterministic": [round(v, 4) for v in res[True]["step"]]},
                      "bwd_breakdown_ms": {"default": breakdown(False), "deterministic": breakdown(True)},
                      "peak_MB_above_inputs_step": {"default": peak[False], "deterministic": peak[True]},
                      "card_and_power_limit": card,
                      "timing": "CUDA events, median of 5 alternating rounds of 5 calls; breakdown from one profiled call"}),
          flush=True)
    del src, flow, logits, gout
    torch.cuda.empty_cache()
    for (Bp, Cp, HWp, kp) in ((8, 256, 32, 3), (8, 128, 64, 5), (2, 256, 256, 5)):
        s_ = torch.randn(Bp, Cp, HWp, HWp, device=dev).bfloat16().contiguous(memory_format=cl).requires_grad_()
        f_ = (torch.rand(Bp, 2, HWp, HWp, device=dev) * 8 - 4).requires_grad_()
        w_ = (torch.randn(128, Cp, kp, kp, device=dev) / (Cp * kp * kp) ** 0.5).bfloat16().requires_grad_()
        g_ = torch.randn(Bp, 128, HWp, HWp, device=dev).bfloat16().contiguous(memory_format=cl)
        fb = lambda: PatchConvFunction.apply(s_, f_, w_, kp).backward(g_)
        pr = {False: [], True: []}
        for _ in range(5):
            for det in (False, True):
                pr[det].append(in_mode(det, lambda: timed(fb, n=3, w=1)))
        print(json.dumps({"op": "patch conv fwd+bwd, default vs deterministic mode",
                          "config": f"B={Bp} C={Cp} {HWp}x{HWp} k={kp} N=128 bf16 channels_last",
                          "fwd_bwd_ms": {"default": med(pr[False]), "deterministic": med(pr[True])},
                          "card_and_power_limit": card, "timing": "CUDA events, median of 5 alternating rounds"}), flush=True)
        del s_, f_, w_, g_
        torch.cuda.empty_cache()

if "module" in which:   # ExtractorAttn at the shapes the pose generator uses (SURVEY.md section 3): fused module vs the literal op chain
    import gfla_b200
    for (C, HW, k) in ((256, 32, 3), (128, 64, 5)):
        B = 8
        cl = torch.channels_last
        m = gfla_b200.ExtractorAttn(C, k, softmax=True).to(dev).bfloat16().to(memory_format=cl)
        src = torch.randn(B, C, HW, HW, device=dev).bfloat16().contiguous(memory_format=cl).requires_grad_()
        tgt = torch.randn(B, C, HW, HW, device=dev).bfloat16().contiguous(memory_format=cl).requires_grad_()
        flow = (torch.rand(B, 2, HW, HW, device=dev) * 8 - 4).requires_grad_()
        ex, rs = gfla_b200.BlockExtractor(k), gfla_b200.LocalAttnReshape()

        def ours(train):
            out = m(src, tgt, flow)
            if train: out.float().sum().backward()

        def literal(train):   # base_function.py:804-810 verbatim, on our unfused kernels
            bs = ex(src, flow); bt = ex(tgt, torch.zeros_like(flow))
            attn = m.fully_connect_layer(torch.cat((bt, bs), 1))
            out = torch.nn.functional.avg_pool2d(rs(attn, k) * bs, k, k)
            if train: out.float().sum().backward()

        px = B * HW * HW
        for name, fn in (("ExtractorAttn (fused tail, this library)", ours), ("literal reference op chain on our unfused kernels", literal)):
            with torch.no_grad():
                f = timed(lambda: fn(False))
            fb = timed(lambda: fn(True), n=3, w=2)
            print(json.dumps({"op": name, "config": f"B={B} C={C} {HW}x{HW} k={k} bf16 channels_last", "fwd_ms": round(f, 4),
                              "fwd_bwd_ms": round(fb, 4), "Mpixels_per_s_fwd_bwd": round(px / fb / 1e3, 2)}), flush=True)

if "resample16" in which:   # resample2d and the fused resample2d -> cosine on bf16 feature maps: three arms alternated in one process
    # (a) bf16 on the 16-bit kernels; (b) fp32 data on the fp32 kernels; (c) bf16 -> .float() -> fp32 kernels -> .to(bf16)
    import statistics
    import subprocess
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    card = q.stdout.strip() or torch.cuda.get_device_name(0)
    bf = torch.bfloat16

    def arms3(name, px, fns, alg, cfg, rounds=5, **kw):
        """fns: {arm: fn}; alg: {arm: algorithmic bytes}; median of `rounds` alternated rounds per arm"""
        t = {a: [] for a in fns}
        for _ in range(rounds):
            for a, fn in fns.items():
                t[a].append(timed(fn, n=3, w=1))
        for a in fns:
            emit(f"{name} ({a})", statistics.median(t[a]), px, alg[a], config=cfg, card=card, rounds=rounds, **kw)
        return {a: statistics.median(v) for a, v in t.items()}

    B, C, H, W = 32, 128, 512, 512           # cfg3
    px = B * H * W
    x32 = torch.randn(B, C, H, W, device=dev)
    g32 = torch.randn(B, C, H, W, device=dev)
    x16, g16 = x32.to(bf), g32.to(bf)
    coarse = (torch.rand(B, 2, H // 16, W // 16, device=dev) * 16 - 8).floor() + 0.25
    blocky = (torch.nn.functional.interpolate(coarse, size=(H, W), mode="nearest") + 0.5 * torch.rand(B, 2, H, W, device=dev)).contiguous()
    # the fp32 grad_in1 buffer of arm (a): zero fill (4 B), 4 B instead of 2 B per element, narrowing (read 4 B, write 2 B)
    extra = px * C * 12
    for ks, sigma in ((2, 5.0), (4, 2.0)):
        for fname, fl in (("smooth", smooth(B, H, W)), ("blocky", blocky)):
            in2 = torch.cat([fl, torch.full((B, 1, H, W), sigma, device=dev)], 1).contiguous()
            fwd = {"a bf16": lambda: F_.resample2d_fwd(x16, in2, ks, 1),
                   "b fp32": lambda: F_.resample2d_fwd(x32, in2, ks, 1),
                   "c bf16 via fp32": lambda: F_.resample2d_fwd(x16.float(), in2, ks, 1).to(bf)}
            arms3(f"resample2d_fwd ks={ks} {fname} flow", px, fwd,
                  {"a bf16": px * (2 * C * 2 + 12), "b fp32": px * (2 * C * 4 + 12), "c bf16 via fp32": px * (2 * C * 2 + 12)},
                  "cfg3 B=32 C=128 512x512")

            def bwd_c():
                g1, g2 = F_.resample2d_bwd(x16.float(), in2, g16.float(), ks, 1)
                return g1.to(bf), g2
            bwd = {"a bf16": lambda: F_.resample2d_bwd(x16, in2, g16, ks, 1),
                   "b fp32": lambda: F_.resample2d_bwd(x32, in2, g32, ks, 1),
                   "c bf16 via fp32": bwd_c}
            arms3(f"resample2d_bwd ks={ks} {fname} flow", px, bwd,
                  {"a bf16": px * (3 * C * 2 + 24), "b fp32": px * (3 * C * 4 + 24), "c bf16 via fp32": px * (3 * C * 2 + 24)},
                  "cfg3", extra_impl_GB_arm_a=round(extra / 1e9, 3))
            torch.cuda.empty_cache()
    del x32, g32, x16, g16, blocky, coarse
    torch.cuda.empty_cache()

    for lname, (B, C, H, W) in (("relu3_1", (16, 256, 64, 64)), ("relu2_1", (16, 128, 128, 128))):   # bench.py's f4 shapes
        px = B * H * W
        s32, t32 = torch.randn(B, C, H, W, device=dev), torch.randn(B, C, H, W, device=dev)
        s16, t16 = s32.to(bf), t32.to(bf)
        in2 = torch.cat([smooth(B, H, W), torch.full((B, 1, H, W), 2.0, device=dev)], 1).contiguous()
        gc32 = torch.randn(B, H, W, device=dev)
        gc16 = gc32.to(bf)
        st16 = F_.resample2d_cosine_fwd(s16, in2, t16, 4, 1)[1]
        st32 = F_.resample2d_cosine_fwd(s32, in2, t32, 4, 1)[1]

        def step_a():
            c, st = F_.resample2d_cosine_fwd(s16, in2, t16, 4, 1)
            F_.resample2d_cosine_bwd(s16, in2, t16, st, gc16, 4, 1)

        def step_b():
            c, st = F_.resample2d_cosine_fwd(s32, in2, t32, 4, 1)
            F_.resample2d_cosine_bwd(s32, in2, t32, st, gc32, 4, 1)

        def step_c():
            a, t = s16.float(), t16.float()
            c, st = F_.resample2d_cosine_fwd(a, in2, t, 4, 1)
            c.to(bf)
            F_.resample2d_cosine_bwd(a, in2, t, st, gc16.float(), 4, 1)

        # forward: source, target, flow, cos, stats; flow-only backward: source, target, stats, grad_cos, flow, grad_flow
        alg = {"a bf16": px * (4 * C + 2 + 12 + 12) + px * (4 * C + 12 + 2 + 12 + 12),
               "b fp32": px * (8 * C + 4 + 12 + 12) + px * (8 * C + 12 + 4 + 12 + 12),
               "c bf16 via fp32": px * (4 * C + 2 + 12 + 12) + px * (4 * C + 12 + 2 + 12 + 12)}
        arms3(f"resample2d_cosine fwd+flow bwd {lname}", px, {"a bf16": step_a, "b fp32": step_b, "c bf16 via fp32": step_c}, alg,
              f"f4 {lname} B={B} C={C} {H}x{W} ks=4 sigma=2")
        del s32, t32, s16, t16
        torch.cuda.empty_cache()

    # peak memory of one PerceptualCorrectness forward + backward (random-weight VGG19, frozen) in bf16 and in fp32
    import torchvision
    import gfla_b200
    torch.manual_seed(0)
    feats = torchvision.models.vgg19(weights=None).features[:21].to(dev).eval()
    for p in feats.parameters():
        p.requires_grad_(False)
    cuts = {"relu1_1": 1, "relu2_1": 6, "relu3_1": 11, "relu4_1": 20}

    class VGG(torch.nn.Module):
        def __init__(self, f):
            super().__init__()
            self.f = f

        def forward(self, x):
            out, h = {}, x
            for i, layer in enumerate(self.f):
                h = layer(h)
                out.update({n: h for n, c in cuts.items() if c == i})
            return out
    for dt in (bf, torch.float32):
        vgg = VGG(feats.to(dt))
        imgs = [torch.rand(16, 3, 256, 256, device=dev).to(dt) for _ in range(2)]
        flows = [(torch.rand(16, 2, h, h, device=dev) * 4 - 2).to(dt).requires_grad_() for h in (64, 128)]
        loss_fn = gfla_b200.PerceptualCorrectness(vgg=vgg)
        loss_fn(imgs[0], imgs[1], flows, [2, 1]).backward()          # warm-up
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        loss_fn(imgs[0], imgs[1], flows, [2, 1]).backward()
        torch.cuda.synchronize()
        print(json.dumps({"op": "PerceptualCorrectness fwd+bwd peak memory", "dtype": str(dt), "card": card,
                          "config": "VGG19 features to relu4_1, 16x3x256x256 images, flows at relu3_1 and relu2_1",
                          "peak_extra_MB": round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)}), flush=True)
        del vgg, imgs, flows, loss_fn
        torch.cuda.empty_cache()

if "fp16" in which:   # fp16 local attention: (a) the fp16 tile kernels, (b) bf16 on the same kernels, (c) fp16 as it ran before
    # the fp16 tile instances (the gather forward, the backward on fp32 copies), alternated in one process; then one
    # PoseGenerator training step (fp32 weights, channels-last) under autocast fp16, autocast bf16 and in plain fp32
    import statistics
    import subprocess
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    card = q.stdout.strip() or torch.cuda.get_device_name(0)
    cl = torch.channels_last
    med = lambda v: round(statistics.median(v), 4)
    ARMS = {"a fp16 tile": (torch.float16, "auto"), "b bf16 tile": (torch.bfloat16, "auto"), "c fp16 gather / fp32 copies": (torch.float16, "gather")}
    for (B, C, HW, k, flows) in ((16, 256, 256, 5, ("smooth", "iid")), (8, 256, 32, 3, ("smooth",)), (8, 128, 64, 5, ("smooth",))):
        for fname in flows:
            flow = smooth(B, HW, HW) if fname == "smooth" else (torch.rand(B, 2, HW, HW, device=dev) * 8 - 4)
            base = [torch.randn(B, C, HW, HW, device=dev), torch.randn(B, k * k, HW, HW, device=dev), torch.randn(B, C, HW, HW, device=dev)]
            data = {}
            for arm, (dt, algo) in ARMS.items():
                s_, l_, g_ = base[0].to(dt).contiguous(memory_format=cl), base[1].to(dt), base[2].to(dt).contiguous(memory_format=cl)
                data[arm] = (s_, l_, g_, algo)
            del base
            res = {arm: {"fwd": [], "bwd": [], "step": []} for arm in ARMS}
            for _ in range(5):
                for arm, (s_, l_, g_, algo) in data.items():
                    n, w = (2, 1) if algo == "gather" and B * HW * HW > 2 ** 20 else (5, 2)
                    fwd = lambda: F_.local_attn_fwd(s_, flow, l_, k, algo=algo)
                    bwd = lambda: F_.local_attn_bwd(s_, flow, l_, g_, k, algo=algo)
                    res[arm]["fwd"].append(timed(fwd, n=n, w=w))
                    res[arm]["bwd"].append(timed(bwd, n=n, w=w))
                    res[arm]["step"].append(timed(lambda: (fwd(), bwd()), n=n, w=w))
            print(json.dumps({"op": "local attention fwd / bwd / step by dtype",
                              "config": f"B={B} C={C} {HW}x{HW} k={k} channels_last, {fname} flow (fp32)",
                              **{f"{part}_ms": {arm: med(res[arm][part]) for arm in ARMS} for part in ("fwd", "bwd", "step")},
                              "step_ms_all": {arm: [round(v, 4) for v in res[arm]["step"]] for arm in ARMS},
                              "card_and_power_limit": card,
                              "timing": "CUDA events, median of 5 alternating rounds (5 calls after 2 warm-up; 2 after 1 for arm c at cfg2)"}),
                  flush=True)
            del data, flow
            torch.cuda.empty_cache()
    import bench_models
    if bench_models.reference_root() is None:
        print(json.dumps({"op": "PoseGenerator step by precision", "skipped": "baseline/_ref snapshot of the reference generators missing"}))
    else:
        Pose, _ = bench_models.load_generators("fused")
        torch.manual_seed(11)
        net = Pose(**bench_models.POSE_KW)
        net.init_weights("orthogonal", gain=0.5)
        net = net.to(dev).to(memory_format=cl)
        gen = torch.Generator(device="cpu").manual_seed(3)
        x = [torch.randn(4, c, 256, 256, generator=gen).to(dev).contiguous(memory_format=cl) for c in (3, 18, 18)]
        tf32 = {"cudnn.allow_tf32": torch.backends.cudnn.allow_tf32, "cuda.matmul.allow_tf32": torch.backends.cuda.matmul.allow_tf32}

        def train_step(dt):
            net.zero_grad(set_to_none=True)
            with torch.autocast("cuda", dtype=dt or torch.float32, enabled=dt is not None):
                img, flows, _ = net(*x)
                loss = img.float().mean() + sum(f.float().pow(2).mean() for f in flows)
            loss.backward()
        parms = {"autocast fp16": torch.float16, "autocast bf16": torch.bfloat16, "fp32": None}
        pres = {a: [] for a in parms}
        for _ in range(5):
            for a, dt in parms.items():
                pres[a].append(timed(lambda: train_step(dt), n=3, w=1))
        print(json.dumps({"op": "PoseGenerator forward+backward by precision (fp32 weights, channels_last)",
                          "config": "B=4 256x256, POSE_KW of bench_models, fused ExtractorAttn",
                          "ms": {a: med(v) for a, v in pres.items()}, "ms_all": {a: [round(t, 2) for t in v] for a, v in pres.items()},
                          "tf32_state_of_the_fp32_arm": tf32, "card_and_power_limit": card,
                          "timing": "CUDA events, median of 5 alternating rounds of 3 steps after 1 warm-up"}), flush=True)
