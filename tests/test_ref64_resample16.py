"""CPU checks of the 16-bit bound (ref64_resample16): the numpy emulations of the fp32 kernels (test_ref64_resample), run on
16-bit-valued inputs with an fp32 flow and rounded once to bf16 / fp16 where the 16-bit kernels store a 16-bit output,
stay within it; the 16-bit implementations the kernels deliberately avoid do not."""
import numpy as np
import pytest

import ref64
import ref64_resample as rr
from ref64_resample16 import check16, round16
from test_ref64_resample import EPS, FLOWS, cos_case, emu_cos, emu_fwd, emu_in1, emu_store, emu_weights, gather, std_case

f32, f64 = np.float32, np.float64
KINDS = ["bf16", "fp16"]


def case16(kind, flow, ks, dil, seed):
    """std_case with source and grad_out rounded to the 16-bit type; the flow stays fp32"""
    a, in2, g = std_case(flow, ks, dil, seed)
    return round16(a, kind), in2, round16(g, kind)


def emu_in2_16(t, src, g):
    """k_resample2d16_bwd_in2: emu_in2 of test_ref64_resample (the corner sums in fp32 over the widened values)"""
    taps = gather(t, src)
    B, C = g.shape[:2]
    g = g.reshape(B, C, -1)
    D = np.zeros((t.n, B, t.H * t.W), f32)
    for c in range(C):
        D = D + g[None, :, c] * taps[:, :, c]
    return emu_store(t, D)


def plain_checks(kind, a, in2, g, ks, dil, order, taps_from=None):
    """-> {output: (worst, message)} of the emulated 16-bit forward and backward.  taps_from: a different flow to take the
    taps from (a fault)"""
    r = rr.resample2d(a, in2, ks, dil, g)
    u, eta = rr.unit(f32)
    src2 = in2 if taps_from is None else taps_from
    t = rr.Resample2d(src2, ks, dil, *a.shape[2:])
    tt = rr.Resample2d(src2, ks, dil, *a.shape[2:], trunc=True)
    return {
        "fwd": check16("fwd16", round16(emu_fwd(t, a), kind), r["out"], rr.bound_fwd(r["out"], r["mags_out"], u, eta), kind),
        "gin1": check16("gin1_16", round16(emu_in1(tt, g, order), kind), r["gin1"],
                        rr.bound_in1(r["gin1"], r["mags_in1"], u, eta), kind),
        "gin2": ref64.check("gin2", emu_in2_16(t, a, g), r["gin2"], rr.bound_in2(r["gin2"], r["mags_in2"], u, eta)),
    }


@pytest.mark.parametrize("order", ["seq", "rev"])
@pytest.mark.parametrize("flow", FLOWS)
@pytest.mark.parametrize("kind", KINDS)
def test_fp32_emulation_rounded_once_within_bound(kind, flow, order):
    for ks, dil in [(4, 1), (3, 2), (6, 1)]:
        a, in2, g = case16(kind, flow, ks, dil, seed=3 * ks + dil)
        for name, (worst, msg) in plain_checks(kind, a, in2, g, ks, dil, order).items():
            assert msg is None, msg


def cos_checks16(kind, c, y, y_in1):
    u, eta = rr.unit(f32)
    cos, stats, gv, gt, g2 = y
    return {"cos": check16("cos16", round16(cos, kind), c["cos"], rr.bound_cos(c, u, eta), kind),
            "stats": ref64.check("stats", stats, c["stats"], rr.bound_stats(c, u, eta)),
            "gt": check16("gt16", round16(gt, kind), c["gt"], rr.bound_gt(c, u, eta), kind),
            "gin2": ref64.check("cos gin2", g2, c["gin2"], rr.bound_in2(c["gin2"], c["mags_in2"], u, eta)),
            "gin1": check16("cos gin1_16", round16(y_in1, kind), c["gin1"], rr.bound_in1(c["gin1"], c["mags_in1"], u, eta), kind)}


def cos16(kind, C=66):
    a, in2, t, gc, ks, dil = cos_case(C=C)
    a, t, gc = (round16(x, kind) for x in (a, t, gc))
    return a, in2, t, gc, ks, dil, rr.cosine(a, in2, t, ks, dil, EPS, gc)


@pytest.mark.parametrize("TS", [1, 4])
@pytest.mark.parametrize("C", [9, 67])
@pytest.mark.parametrize("kind", KINDS)
def test_fp32_cosine_emulation_rounded_once_within_bound(kind, C, TS):
    a, in2, t, gc, ks, dil, c = cos16(kind, C)
    assert (c["nv"] == 0).any() and (c["nt"] == 0).any()
    y = emu_cos(c["taps"], a, t, gc, TS)
    tt = rr.Resample2d(in2, ks, dil, *a.shape[2:], trunc=True)
    for name, (worst, msg) in cos_checks16(kind, c, y, emu_in1(tt, y[2], "seq")).items():   # grad_val stays fp32
        assert msg is None, msg


# --------------------------------------------------------------------------------------------------- injected faults
def scatter16(tt, g, kind):
    """grad_input1 summed in the 16-bit type: every partial added to the element and rounded (a 16-bit atomicAdd)"""
    w, s, _ = emu_weights(tt)
    wn = (w / s[None]).astype(f64)                                              # (n, B, H W)
    B, C = g.shape[:2]
    hw = tt.Hi * tt.Wi
    part = (wn[:, :, None, :] * g.reshape(B, C, -1).astype(f64)[None]).astype(f32)   # (n, B, C, H W)
    key = (np.arange(B).reshape(1, B, 1, 1) * C + np.arange(C).reshape(1, 1, C, 1)) * hw + tt.off[:, :, None, :]
    p, k = part.ravel(), np.broadcast_to(key, part.shape).ravel()
    perm = np.argsort(k, kind="stable")
    p, k = p[perm], k[perm]
    start = np.r_[0, np.flatnonzero(np.diff(k)) + 1]
    rank = np.arange(k.size) - np.repeat(start, np.diff(np.r_[start, k.size]))   # position of a partial in its element
    out = np.zeros(B * C * hw, f32)
    for j in range(int(rank.max()) + 1):
        sel = rank == j
        out[k[sel]] = round16(out[k[sel]] + p[sel], kind)
    return out.reshape(B, C, tt.Hi, tt.Wi)


def _flow16(kind):
    """the caller's fp32 flow rounded to 16-bit before the taps: fails the fp32 bound of grad_input2"""
    a, in2, g = case16(kind, "iid", 4, 1, seed=1)
    return plain_checks(kind, a, in2, g, 4, 1, "seq", taps_from=round16(in2, kind))["gin2"]


def _gin1_adds16(kind):
    a, in2, g = case16(kind, "iid", 4, 1, seed=1)
    r = rr.resample2d(a, in2, 4, 1, g)
    u, eta = rr.unit(f32)
    tt = rr.Resample2d(in2, 4, 1, *a.shape[2:], trunc=True)
    return check16("gin1 16-bit adds", scatter16(tt, g, kind), r["gin1"], rr.bound_in1(r["gin1"], r["mags_in1"], u, eta), kind)


def _gin2_16(kind):
    a, in2, g = case16(kind, "iid", 4, 1, seed=1)
    r = rr.resample2d(a, in2, 4, 1, g)
    u, eta = rr.unit(f32)
    y = round16(emu_in2_16(r["taps"], a, g), kind)
    return ref64.check("gin2 16-bit", y, r["gin2"], rr.bound_in2(r["gin2"], r["mags_in2"], u, eta))


def _cos_fault(fault, kind):
    """TS = 1.  stats16: the backward reads (v.t, |v|, |t|) rounded to 16-bit -> grad_input2; v16: the cosine of the
    16-bit-rounded warped values (resample2d, then cosine_similarity, in 16-bit storage) -> stats"""
    a, in2, t, gc, ks, dil, c = cos16(kind)
    u, eta = rr.unit(f32)
    v = emu_fwd(c["taps"], a)
    if fault == "v16":
        v = round16(v, kind)

    def csum(x):
        acc = np.zeros(x[:, 0].shape, f32)
        for ch in range(x.shape[1]):
            acc = acc + x[:, ch]
        return acc
    dot, nv, nt = csum(v * t), np.sqrt(csum(v * v)), np.sqrt(csum(t * t))
    if fault == "v16":
        return ref64.check("stats over 16-bit v", np.stack([dot, nv, nt], 1), c["stats"], rr.bound_stats(c, u, eta))
    dot, nv, nt = (round16(x, kind) for x in (dot, nv, nt))
    e = f32(EPS)
    aa, bb = np.maximum(nv, e), np.maximum(nt, e)
    with np.errstate(divide="ignore", invalid="ignore"):
        k1 = gc / (aa * bb)
        k2v = np.where(nv > e, (gc * dot) / (((aa * aa) * bb) * nv), f32(0)).astype(f32)
    gv = (k1[:, None] * t - k2v[:, None] * v).reshape(v.shape[0], v.shape[1], -1)
    taps = gather(c["taps"], a)
    D = np.zeros((c["taps"].n,) + gv[:, 0].shape, f32)
    for ch in range(gv.shape[1]):
        D = D + gv[None, :, ch] * taps[:, :, ch]
    return ref64.check("gin2 from 16-bit stats", emu_store(c["taps"], D), c["gin2"],
                       rr.bound_in2(c["gin2"], c["mags_in2"], u, eta))


FAULTS = {
    "flow rounded to 16-bit before the taps": _flow16,
    "grad_input1 summed with 16-bit adds": _gin1_adds16,
    "grad_input2 stored in 16-bit": _gin2_16,
    "stats stored in 16-bit before the backward": lambda k: _cos_fault("stats16", k),
    "cosine over 16-bit-rounded warped values": lambda k: _cos_fault("v16", k),
}


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("fault", sorted(FAULTS))
def test_injected_16bit_fault_fails_its_bound(fault, kind):
    worst, msg = FAULTS[fault](kind)
    assert msg is not None, f"{fault} ({kind}): worst |err|/bound {worst:.3g} stays within the bound"
