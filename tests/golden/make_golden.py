#!/usr/bin/env python
"""Generate the golden vectors in tests/golden/*.npz.

Run in the BUILD container only (needs /root/reference to build oracle/_ref):

    python tests/golden/make_golden.py

Ground truth = the reference's own CUDA kernel bodies compiled for the host
(``oracle/_ref/libgfla_ref.so``, one thread, see oracle/Makefile) and, for the
``ExtractorAttn`` tail, those bodies composed with stock torch CPU ops exactly
as ``model/networks/base_function.py:804-810`` composes them (Softmax(dim=1),
broadcast multiply, ``avg_pool2d(k, k)``), differentiated by torch autograd
with the reference backward bodies plugged in as custom Functions -- the same
structure as ``block_extractor.py:5-42`` / ``local_attn_reshape.py:5-37``.

The reference ships no golden files; the only results its own tests pin are two
layout identities (``test_block_extractor.py:55``, ``test_local_attn_reshape.py:29-43``)
and two double-precision gradchecks (``test_block_extractor.py:74-78``,
``test_local_attn_reshape.py:66-70``).  Both identities are stored here as
cases; the gradcheck shapes are reproduced in tests/.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import oracle.oracle as orc  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def smooth_flow(rng, B, H, W, amp, cell=4):
    """bilinear up-sampling of coarse U(-amp, amp) noise (SURVEY.md 8d 'smooth')."""
    coarse = torch.from_numpy(rng.uniform(-amp, amp, (B, 2, max(H // cell, 2), max(W // cell, 2))))
    return torch.nn.functional.interpolate(coarse, size=(H, W), mode="bilinear", align_corners=True).numpy()


def main():
    orc.build(ref=True)
    R = orc.Ref(threads=1)
    rng = np.random.default_rng(20260923)

    # ------------------------------------------------------------------ block_extractor
    be = {}
    cases = [
        # name, dtype, B, C, Hs, Ws, Hf, Wf, k, flow kind
        ("cfg1", np.float32, 1, 8, 32, 32, 32, 32, 3, "iid8"),          # BASELINE.json configs[0]
        ("k4_border", np.float32, 2, 3, 9, 7, 9, 7, 4, "border"),       # even k: offsets -2..1; taps cross every border
        ("k5_smooth", np.float32, 2, 5, 16, 16, 16, 16, 5, "smooth"),
        ("src_gt_flow", np.float32, 1, 2, 12, 14, 10, 12, 3, "const"),  # external_function.py:61-66 usage
        ("zero_flow", np.float32, 2, 3, 8, 8, 8, 8, 3, "zero"),         # test_block_extractor.py:46-55
        ("gradcheck_shape", np.float64, 4, 6, 14, 10, 14, 10, 3, "rand1.8"),  # test_block_extractor.py:74-78
        ("k2", np.float64, 1, 2, 6, 5, 6, 5, 2, "iid8"),
    ]
    for name, dt, B, C, Hs, Ws, Hf, Wf, k, kind in cases:
        src = rng.standard_normal((B, C, Hs, Ws)).astype(dt)
        if kind == "iid8":
            flow = rng.uniform(-8, 8, (B, 2, Hf, Wf))
        elif kind == "border":
            flow = rng.uniform(-1.5 * Wf, 1.5 * Wf, (B, 2, Hf, Wf))
        elif kind == "smooth":
            flow = smooth_flow(rng, B, Hf, Wf, 6.0)
        elif kind == "const":
            flow = np.full((B, 2, Hf, Wf), float(k // 2))
        elif kind == "zero":
            flow = np.zeros((B, 2, Hf, Wf))
        elif kind == "rand1.8":
            flow = rng.uniform(0, 1, (B, 2, Hf, Wf)) * 1.8
        flow = np.ascontiguousarray(flow.astype(dt))
        out = R.block_extract_fwd(src, flow, k)
        gout = rng.standard_normal(out.shape).astype(dt)
        gs, gf = R.block_extract_bwd(src, flow, gout, k)
        for key, v in dict(source=src, flow=flow, out=out, grad_out=gout, grad_source=gs, grad_flow=gf,
                           k=np.int32(k)).items():
            be[f"{name}/{key}"] = v
    big = ("k5_smooth", "gradcheck_shape")          # each in a file of its own: every file stays under 1 MB
    np.savez_compressed(os.path.join(OUT, "block_extractor.npz"), **{n: v for n, v in be.items() if n.split("/")[0] not in big})
    for case in big:
        np.savez_compressed(os.path.join(OUT, f"block_extractor.{case}.npz"), **{n: v for n, v in be.items() if n.split("/")[0] == case})

    # ------------------------------------------------------------------ local_attn_reshape
    lr = {}
    x = np.arange(9, dtype=np.float32).reshape(1, 9, 1, 1).repeat(2, 0).repeat(10, 2).repeat(10, 3)
    x = np.ascontiguousarray(x)                       # test_local_attn_reshape.py:29-31
    lr["layout/in"], lr["layout/out"], lr["layout/k"] = x, R.attn_reshape_fwd(x, 3), np.int32(3)
    for name, dt, B, H, W, k in [("k3", np.float64, 4, 14, 10, 3), ("k5", np.float32, 2, 6, 7, 5), ("k4", np.float32, 1, 3, 5, 4)]:
        x = rng.standard_normal((B, k * k, H, W)).astype(dt)
        out = R.attn_reshape_fwd(x, k)
        g = rng.standard_normal(out.shape).astype(dt)
        lr[f"{name}/in"], lr[f"{name}/out"], lr[f"{name}/grad_out"] = x, out, g
        lr[f"{name}/grad_in"], lr[f"{name}/k"] = R.attn_reshape_bwd(x, g, k), np.int32(k)
    np.savez_compressed(os.path.join(OUT, "local_attn_reshape.npz"), **lr)

    # ------------------------------------------------------------------ resample2d
    rs = {}
    cases = [
        # name, dtype, B, C, Hi, Wi, H, W, ks, dil, sigma, flow amp
        ("ks2_default", np.float32, 2, 4, 12, 10, 12, 10, 2, 1, 5.0, 3.0),   # Resample2d() defaults, resample2d.py:43
        ("ks4_sigma2", np.float32, 2, 3, 10, 12, 10, 12, 4, 1, 2.0, 3.0),    # external_function.py:233
        ("ks4_border", np.float32, 1, 2, 8, 8, 8, 8, 4, 1, 2.0, 14.0),       # x+dx < 0: int() vs floor() quirk (:137-138)
        ("ks4_dil2", np.float64, 1, 2, 9, 9, 9, 9, 4, 2, 2.0, 3.0),
        ("in_ne_out", np.float32, 1, 3, 14, 9, 7, 11, 2, 1, 5.0, 3.0),
        ("sigma0", np.float32, 1, 2, 6, 6, 6, 6, 2, 1, 0.0, 2.0),            # SAFE_DIV EPS branch (:14-15)
    ]
    for name, dt, B, C, Hi, Wi, H, W, ks, dil, sigma, amp in cases:
        in1 = rng.standard_normal((B, C, Hi, Wi)).astype(dt)
        flow = rng.uniform(-amp, amp, (B, 2, H, W)).astype(dt)
        in2 = np.ascontiguousarray(np.concatenate([flow, np.full((B, 1, H, W), sigma, dt)], 1))  # resample2d.py:51-52
        out = R.resample2d_fwd(in1, in2, ks, dil)
        g = rng.standard_normal(out.shape).astype(dt)
        g1, g2 = R.resample2d_bwd(in1, in2, g, ks, dil)
        for key, v in dict(in1=in1, in2=in2, out=out, grad_out=g, grad_in1=g1, grad_in2=g2,
                           ks=np.int32(ks), dil=np.int32(dil)).items():
            rs[f"{name}/{key}"] = v
    np.savez_compressed(os.path.join(OUT, "resample2d.npz"), **rs)

    # ------------------------------------------------------------------ ExtractorAttn tail (fused op)
    from oracle.ref_pipeline import local_attn_fwd_bwd

    la = {}
    cases = [
        ("k3", np.float32, 2, 6, 10, 9, 3, "smooth"),
        ("k5", np.float32, 1, 8, 12, 12, 5, "iid8"),
        ("k5_border", np.float32, 1, 3, 7, 8, 5, "border"),
        ("k4_f64", np.float64, 1, 4, 6, 6, 4, "iid8"),
        ("k3_f64", np.float64, 2, 5, 9, 8, 3, "smooth"),
    ]
    for name, dt, B, C, H, W, k, kind in cases:
        src = rng.standard_normal((B, C, H, W)).astype(dt)
        if kind == "iid8":
            flow = rng.uniform(-8, 8, (B, 2, H, W))
        elif kind == "border":
            flow = rng.uniform(-1.5 * W, 1.5 * W, (B, 2, H, W))
        else:
            flow = smooth_flow(rng, B, H, W, 4.0)
        flow = np.ascontiguousarray(flow.astype(dt))
        logits = (2.0 * rng.standard_normal((B, k * k, H, W))).astype(dt)
        g = rng.standard_normal((B, C, H, W)).astype(dt)
        out, probs, gs, gf, gl = local_attn_fwd_bwd(R, src, flow, logits, g, k)   # base_function.py:804-810
        for key, v in dict(source=src, flow=flow, logits=logits, out=out, probs=probs, grad_out=g, grad_source=gs,
                           grad_flow=gf, grad_logits=gl, k=np.int32(k)).items():
            la[f"{name}/{key}"] = v
    np.savez_compressed(os.path.join(OUT, "local_attn.npz"), **la)

    for f in sorted(os.listdir(OUT)):
        if f.endswith(".npz"):
            print(f, os.path.getsize(os.path.join(OUT, f)), "bytes")


if __name__ == "__main__":
    main()
