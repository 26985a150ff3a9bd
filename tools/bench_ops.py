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
