"""CPU: the patch convolution (ExtractorAttn's source-half conv, gfla_b200.patch_conv) -- its C entry points reject bad
arguments before touching a device, its fp64 reference agrees with the composition it replaces, and the per-element
bounds the GPU tests apply (tests/test_gpu_patch_conv.py) accept a correctly rounding kernel and reject the faults a
wrong one would make.

    patch_conv(source, flow, weight, k) == conv2d(BlockExtractor(k)(source, flow), weight, None, stride=k)

The reference is ref64.block_extract (the block tensor and its backward, fp64 after fp32 tap selection) composed with
an fp64 convolution written as tensor contractions.
"""
import ctypes

import numpy as np
import pytest

import ref64
from test_ref64 import bf16, make_flow

N_OUT = 128          # output channels the kernels serve (hidden_nc of ExtractorAttn)


# ------------------------------------------------------------------------------------------------------- reference
def conv_blocks(blk, w, k):
    """stride-k conv of a block tensor [B,C,kH,kW] with w [N,C,k,k] -> [B,N,H,W] (fp64)"""
    B, C, KH, KW = blk.shape
    b6 = np.asarray(blk, np.float64).reshape(B, C, KH // k, k, KW // k, k)
    return np.einsum("bchiwj,ncij->bnhw", b6, np.asarray(w, np.float64), optimize=True)


def conv_blocks_t(g, w, k):
    """its transpose: grad_out [B,N,H,W] -> grad_block [B,C,kH,kW]"""
    B, _, H, W = g.shape
    gb = np.einsum("bnhw,ncij->bchiwj", np.asarray(g, np.float64), np.asarray(w, np.float64), optimize=True)
    return gb.reshape(B, w.shape[1], k * H, k * W)


def conv_blocks_wgrad(g, blk, k):
    """weight gradient: sum over pixels of grad_out x block -> [N,C,k,k]"""
    B, C, KH, KW = blk.shape
    b6 = np.asarray(blk, np.float64).reshape(B, C, KH // k, k, KW // k, k)
    return np.einsum("bnhw,bchiwj->ncij", np.asarray(g, np.float64), b6, optimize=True)


def patch_ref(src, flow, w, k, gout=None, block=None):
    """fp64 patch convolution.  block: the [B,C,kH,kW] tensor the forward and the weight gradient contract (default the
    fp64 block_extract; the GPU tests pass block_extract_fwd's bf16 output, which the kernels' gather reproduces bit for
    bit).  -> dict out, M = sum |W||A|; with gout also gs, gf, gw and the magnitudes Mgs, Mgf (block_extract's, taken
    with |G||W| as the block gradient: the error of each fp32 GA = G W^T element scales with that) and Mgw = sum |G||A|,
    plus n = the number of corner contributions each source position receives."""
    src = np.asarray(src, np.float64)
    w = np.asarray(w, np.float64)
    blk = ref64.block_extract(src, flow, k)["out"] if block is None else np.asarray(block, np.float64)
    r = {"out": conv_blocks(blk, w, k), "M": conv_blocks(np.abs(blk), np.abs(w), k)}
    if gout is None:
        return r
    g = np.asarray(gout, np.float64)
    val = ref64.block_extract(src, flow, k, conv_blocks_t(g, w, k))
    mag = ref64.block_extract(src, flow, k, conv_blocks_t(np.abs(g), np.abs(w), k))
    t = ref64.Taps(flow, k, src.shape[2], src.shape[3])
    n = np.stack([np.bincount(t.pos[b].ravel(), minlength=t.Hs * t.Ws) for b in range(t.B)]).reshape(t.B, 1, t.Hs, t.Ws)
    r.update(gs=val["gs"], gf=val["gf"], Mgs=mag["Mgs"], Mgf=mag["Mgf"], n=n,
             gw=conv_blocks_wgrad(g, blk, k), Mgw=conv_blocks_wgrad(np.abs(g), np.abs(blk), k))
    return r


# ---------------------------------------------------------------------------------------------------------- bounds
# Per-element bounds on |y - ref| of the patch-convolution kernels (csrc/patch_conv_tc.cu), in the style of ref64.
U, ETA = ref64.U_BF16, ref64.ETA_BF16


def bound_out(r, M, C, k, u=U, eta=ETA):
    """forward: A is exact (gather_row reproduces block_extract's bf16 store bit for bit) and so are its bf16 x bf16
    products in fp32; the MMAs sum C k^2 of them in fp32 (gamma(C k^2) M); one bf16 store (u |r + error|: the 1.01 pays
    for u of the error term)"""
    return u * np.abs(r) + 1.01 * ref64.gamma(C * k * k) * M + eta


def bound_gw(r, Mgw, P, u=U, eta=ETA, init=0.0):
    """weight gradient: P = B H W exact bf16 products per element summed in fp32 (MMA accumulators over each slice of
    pixel groups, then the slices' 16-byte fp32 reductions): gamma(P) of sum |G||A| and of the buffer's initial value;
    one bf16 rounding by gfla_convert (u |r|, absent when the fp32 buffer itself is checked: u = 0)"""
    return u * np.abs(r) + 1.01 * ref64.gamma(P + 1) * (Mgw + np.abs(init)) + eta


def bound_gs(r, Mgs, n, u=U, eta=ETA, init=0.0):
    """grad_source: GA = G W^T sums N = 128 bf16 products in fp32 (gamma(N) of |G||W|, which Mgs carries), one product
    with the corner weight (+1), n fp32 reductions into the buffer plus its initial value (gamma(n + 1)); one bf16
    rounding (u |r|)"""
    return u * np.abs(r) + 1.01 * (ref64.gamma(N_OUT + 1) + ref64.gamma(n + 1)) * (Mgs + np.abs(init)) + eta


def bound_gf(r, Mgf, C, k, init=0.0):
    """grad_flow: the GA error (gamma(N) of |G||W|, inside Mgf), the corner-difference terms of k_block_extract_bwd
    (block_extract.cu:92-93: four products and three sums per channel) and the fp32 sum over k^2 C of them in
    registers (gamma(k^2 C + N + 4) Mgf); the add of the buffer's initial value and the final add of the two half
    sums (FP32_SLACK)"""
    return ref64.gamma(k * k * C + N_OUT + 4) * Mgf + ref64.FP32_SLACK * (np.abs(r) + np.abs(init))


# ------------------------------------------------------------------------------------------------------------- ABI
@pytest.fixture(scope="module")
def so():
    import __graft_entry__ as ge
    ge.build_cuda()
    import gfla_b200
    return gfla_b200._lib.lib()


def test_patch_conv_argument_validation_needs_no_device(so):
    buf = (ctypes.c_float * 64)()
    p = ctypes.addressof(buf)
    q = p + (-p) % 16                     # a 16-byte-aligned pointer inside the buffer
    ok = (1, 64, 4, 4, 4, 4, 3, 128, 2, 0, 1)   # B C Hs Ws H W k N dtype=bf16 flow_dtype=f32 layout=NHWC

    def fwd(ptrs, args):
        return so.gfla_patch_conv_fwd(*ptrs, *args, None)

    def bwd(ptrs, args, accumulate=0):
        return so.gfla_patch_conv_bwd(*ptrs, *args[:-1], args[-1], accumulate, None)

    f4, b7 = [q] * 4, [q] * 7
    for i in range(4):
        assert fwd(f4[:i] + [None] + f4[i + 1:], ok) == -1
    for i in range(7):
        assert bwd(b7[:i] + [None] + b7[i + 1:], ok) == -1
    rep = lambda i, v: ok[:i] + (v,) + ok[i + 1:]
    for i in range(7):                     # a non-positive size
        assert fwd(f4, rep(i, 0)) == -2 and bwd(b7, rep(i, -1)) == -2
    for kk in (0, 10):
        assert fwd(f4, rep(6, kk)) == -2 and bwd(b7, rep(6, kk)) == -2
    assert fwd(f4, rep(7, 0)) == -2                       # N = 0
    assert fwd(f4, rep(10, 5)) == -2                      # unknown layout code
    for dt, fdt in ((0, 0), (3, 0), (1, 1), (2, 2), (7, 0)):   # not bf16 data with an fp32 flow
        args = ok[:8] + (dt, fdt, 1)
        assert fwd(f4, args) == -3 and bwd(b7, args) == -3
    assert fwd(f4, rep(1, 48)) == -5 and bwd(b7, rep(1, 96)) == -5      # C % 64
    assert fwd(f4, rep(7, 64)) == -5 and bwd(b7, rep(7, 256)) == -5    # N != 128
    assert fwd(f4, rep(10, 0)) == -5 and bwd(b7, rep(10, 0)) == -5     # NCHW
    for i in (0, 2, 3):                    # source, weight, out off 16 bytes
        assert fwd(f4[:i] + [q + 4] + f4[i + 1:], ok) == -4
    assert fwd([q, q + 2, q, q], ok) == -4                # fp32 flow off 4 bytes
    for i in (0, 2, 3, 4, 6):
        assert bwd(b7[:i] + [q + 8] + b7[i + 1:], ok) == -4
    assert bwd([q, q, q, q, q, q + 2, q], ok) == -4       # grad_flow


# ------------------------------------------------------------------------------------------------------- reference
def inputs(B, C, Hs, Ws, H, W, k, kind, seed):
    rng = np.random.default_rng(seed)
    s = bf16(rng.standard_normal((B, C, Hs, Ws)))
    f = make_flow(kind, rng, B, H, W, k)
    w = bf16(rng.standard_normal((N_OUT, C, k, k)) / np.sqrt(C * k * k))
    g = bf16(rng.standard_normal((B, N_OUT, H, W)))
    return s, f, w, g


def test_reference_matches_the_composition_on_the_oracle(oracle_lib):
    """value and all three gradients of the fp64 reference against the CPU oracle's block_extract (fp64) composed with
    torch's fp64 conv2d and its autograd.  The flow is a multiple of 1/64 so the oracle's fp64 tap arithmetic and the
    reference's fp32 one select the same taps with the same weights."""
    import torch
    for (B, C, Hs, Ws, H, W, k, kind) in ((1, 16, 13, 17, 11, 15, 3, "smooth"), (2, 8, 9, 12, 9, 12, 4, "border"),
                                          (1, 8, 12, 10, 7, 9, 5, "outside")):
        s, f, w, g = inputs(B, C, Hs, Ws, H, W, k, kind, seed=7 * k)
        f =(np.round(f.astype(np.float64) * 64) / 64).astype(np.float32)
        r = patch_ref(s, f, w, k, g)
        s64, f64 = s.astype(np.float64), f.astype(np.float64)
        blk = torch.from_numpy(oracle_lib.block_extract_fwd(s64, f64, k)).requires_grad_()
        wt = torch.from_numpy(w.astype(np.float64)).requires_grad_()
        out = torch.nn.functional.conv2d(blk, wt, None, stride=k)
        out.backward(torch.from_numpy(g.astype(np.float64)))
        ogs, ogf = oracle_lib.block_extract_bwd(s64, f64, blk.grad.numpy(), k)
        tol = lambda ref, mag: 1e-12 * (np.abs(ref) + mag) + 1e-300
        assert np.all(np.abs(out.detach().numpy() - r["out"]) <= tol(r["out"], r["M"]))
        assert np.all(np.abs(wt.grad.numpy() - r["gw"]) <= tol(r["gw"], r["Mgw"]))
        assert np.all(np.abs(ogs - r["gs"]) <= tol(r["gs"], r["Mgs"]))
        assert np.all(np.abs(ogf - r["gf"]) <= tol(r["gf"], r["Mgf"]))
        assert np.abs(r["gf"]).max() > 0 and np.abs(r["gs"]).max() > 0


# -------------------------------------------------------------------------------------------- bounds reject faults
SHAPE = (2, 128, 14, 21, 12, 20, 3)          # B C Hs Ws H W k: two 64-channel chunks, ragged 16x8 pixel groups


@pytest.fixture(scope="module")
def case():
    B, C, Hs, Ws, H, W, k = SHAPE
    s, f, w, g = inputs(B, C, Hs, Ws, H, W, k, "smooth", seed=3)
    blk = ref64.round_bf16(ref64.block_extract(s, f, k)["out"])         # what block_extract_fwd stores in bf16
    r = patch_ref(s, f, w, k, g, block=blk)
    return dict(s=s, f=f, w=w, g=g, blk=blk, r=r)


def emulated(c, w=None, blk=None, g=None):
    """a correctly rounding kernel: fp64 sums, each output rounded once (bf16 out / grad_source / grad_weight, fp32
    grad_flow)"""
    k = SHAPE[-1]
    w = c["w"] if w is None else w
    blk = c["blk"] if blk is None else blk
    g = c["g"] if g is None else g
    out = ref64.round_bf16(conv_blocks(blk, w, k))
    be = ref64.block_extract(c["s"], c["f"], k, conv_blocks_t(g, w, k))
    return dict(out=out, gs=ref64.round_bf16(be["gs"]), gf=be["gf"].astype(np.float32).astype(np.float64),
                gw=ref64.round_bf16(conv_blocks_wgrad(g, blk, k)))


def checks(c, y):
    """-> {output: (worst ratio, message)}"""
    B, C, Hs, Ws, H, W, k = SHAPE
    r = c["r"]
    return {"out": ref64.check("out", y["out"], r["out"], bound_out(r["out"], r["M"], C, k)),
            "gs": ref64.check("gs", y["gs"], r["gs"], bound_gs(r["gs"], r["Mgs"], r["n"])),
            "gf": ref64.check("gf", y["gf"], r["gf"], bound_gf(r["gf"], r["Mgf"], C, k)),
            "gw": ref64.check("gw", y["gw"], r["gw"], bound_gw(r["gw"], r["Mgw"], B * H * W))}


def test_bounds_accept_emulated_kernels(case):
    res = checks(case, emulated(case))
    for name, (worst, msg) in res.items():
        assert msg is None, msg
    for name in ("out", "gs", "gw"):       # the bf16 outputs: one rounding is a visible fraction of the bound
        assert res[name][0] > 0.1, (name, res[name][0])


class _SwappedCorners(ref64.Taps):
    """bilinear corner weights of the x axis swapped (wlo <-> whi)"""

    def build(self):
        lo, hi, fl, wlo, whi = self.tx
        self.tx = (lo, hi, fl, whi, wlo)
        super().build()
        self.tx = (lo, hi, fl, wlo, whi)


class _NoRBCorner(ref64.Taps):
    """the RB corner of every tap dropped"""

    def build(self):
        super().build()
        self.cw = self.cw.copy()
        self.cw[:, :, :, 3] = 0.0


def with_taps(monkeypatch, cls, fn):
    monkeypatch.setattr(ref64, "Taps", cls)
    try:
        return fn()
    finally:
        monkeypatch.undo()


def test_bounds_reject_faults(case, monkeypatch):
    c = case
    B, C, Hs, Ws, H, W, k = SHAPE
    assert np.abs(c["f"]).max() > 0.5
    faults = {}
    # forward: the weight's taps (i, j) transposed; a dropped 64-channel chunk; swapped bilinear corner weights
    assert np.abs(c["w"] - c["w"].transpose(0, 1, 3, 2)).max() > 0
    faults["taps transposed"] = ("out", emulated(c, w=c["w"].transpose(0, 1, 3, 2)))
    w_drop = c["w"].copy()
    w_drop[:, 64:128] = 0.0
    faults["chunk dropped"] = ("out", emulated(c, w=w_drop))
    blk_sw = with_taps(monkeypatch, _SwappedCorners, lambda: ref64.round_bf16(ref64.block_extract(c["s"], c["f"], k)["out"]))
    faults["corner weights swapped"] = ("out", emulated(c, blk=blk_sw))
    # backward: a dropped grad_source corner; grad_flow with its x / y planes exchanged; one pixel group missing from
    # the weight gradient's sum
    y = emulated(c)
    gb = conv_blocks_t(c["g"], c["w"], k)
    gs_no_rb = with_taps(monkeypatch, _NoRBCorner, lambda: ref64.block_extract(c["s"], c["f"], k, gb)["gs"])
    faults["grad_source corner dropped"] = ("gs", dict(y, gs=ref64.round_bf16(gs_no_rb)))
    faults["grad_flow axes flipped"] = ("gf", dict(y, gf=y["gf"][:, ::-1]))
    g_hole = c["g"].copy()
    g_hole[1, :, 8:16, 16:32] = 0.0        # image 1, pixel group row 1, column 1 (the ragged corner group)
    faults["weight-gradient group missing"] = ("gw", dict(y, gw=emulated(c, g=g_hole)["gw"]))
    for name, (out, yf) in faults.items():
        worst, msg = checks(c, yf)[out]
        assert msg is not None, f"{name}: fault not detected by the {out} bound (worst ratio {worst:.3g})"
