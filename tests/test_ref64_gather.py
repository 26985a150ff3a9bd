"""CPU checks of ref64_gather: the fp64 reference with fp64 tap selection against the oracle's fp64 local attention and
block_extractor, and the fp32 / fp64 bounds against the oracle's results and numpy emulations of the kernels' exact
operation order (they pass), and against injected faults (they fail)."""
import numpy as np
import pytest

import ref64
import ref64_gather as rg
from test_ref64 import FLOWS
from test_ref64 import make_flow as make_flow32

f32, f64 = np.float32, np.float64
DTYPES = {"fp32": f32, "fp64": f64}


def make_flow(kind, rng, B, H, W, k, A):
    """test_ref64.make_flow in the kernel's type A.  fp64: "irregular" places flows whose fp64 taps are not consecutive,
    and the other non-integral kinds get full fp64 mantissas (a jitter below 10^-2), so that fp64 tap selection differs
    from fp32's"""
    if kind == "irregular" and A == f64:
        f = rng.uniform(-3, 3, (B, 2, H, W))
        for i, (x, v) in enumerate(rg.irregular_flow_values(range(2, W - 2, 3), k, rng, f64).items()):
            f[:, 0, (5 * i) % H, x] = v
        return f
    f = make_flow32(kind, rng, B, H, W, k)
    if A == f64 and kind not in ("zero", "int"):
        return f.astype(f64) + rng.uniform(-1e-2, 1e-2, f.shape)
    return f.astype(A)


LOGITS = ["normal", "peaked", "flat"]


def make_logits(family, rng, B, k, H, W):
    """N(0, 2); peaked: one logit per pixel 40 above the rest (100 in every third pixel, where fp32's exp of the others
    underflows into the subnormals); flat: all equal"""
    lg = 2 * rng.standard_normal((B, k * k, H, W))
    if family == "peaked":
        t = rng.integers(0, k * k, (B, 1, H, W))
        up = np.where(np.arange(H * W).reshape(H, W) % 3 == 0, 100.0, 40.0)
        np.put_along_axis(lg, t, np.take_along_axis(lg, t, 1) * 0 + lg.max(1, keepdims=True) + up, 1)
    elif family == "flat":
        lg = np.full((B, k * k, H, W), 0.75)
    return lg


def inputs(B, C, Hs, Ws, H, W, k, kind, seed, A, logits="normal"):
    rng = np.random.default_rng(seed)
    s = rng.standard_normal((B, C, Hs, Ws)).astype(A)
    f = make_flow(kind, rng, B, H, W, k, A).astype(A)
    lg = make_logits(logits, rng, B, k, H, W).astype(A)
    g = rng.standard_normal((B, C, H, W)).astype(A)
    return s, f, lg, g


def magnitude_close(y, ref, mag, rel):
    err = np.abs(np.asarray(y, f64) - ref)
    worst = float((err / (rel * (mag + np.abs(ref)) + 1e-300)).max())
    assert worst <= 1.0, worst


def shape(k, i):
    """B, C, Hs, Ws, H, W: the source larger than the flow field, or smaller, in turn"""
    return (1, 5, 14, 17, 11, 13) if (k + i) % 2 else (2, 3, 9, 10, 11, 13)


# ---------------------------------------------------------------------------------------- reference vs oracle fp64
@pytest.mark.parametrize("k", range(1, 10))
def test_reference_matches_oracle_fp64(oracle_lib, k):
    for i, kind in enumerate(FLOWS):
        B, C, Hs, Ws, H, W = shape(k, i)
        s, f, lg, g = inputs(B, C, Hs, Ws, H, W, k, kind, 100 * k + i, f64)
        la = rg.LocalAttn(f, lg, k, Hs, Ws, f64)
        out, mags = la.fwd(s)
        oout, oprobs = oracle_lib.local_attn_fwd(s, f, lg, k, return_probs=True)
        magnitude_close(oout, out, mags["M"], 1e-12)
        magnitude_close(oprobs, la.probs(), 1.0, 1e-12)
        r = la.bwd(s, g)
        ogs, ogf, ogl = oracle_lib.local_attn_bwd(s, f, lg, g, k)
        magnitude_close(ogs, r["gs"], r["Mgs"], 1e-12)
        magnitude_close(ogl, r["gl"], la.probs() * (r["D"] + r["PD"]), 1e-12)
        magnitude_close(ogf, r["gf"], r["Mgf"], 1e-12)
        gb = np.random.default_rng(k + i).standard_normal((B, C, k * H, k * W))
        be = rg.BlockExtract(s, f, k, gb, f64)
        assert np.array_equal(oracle_lib.block_extract_fwd(s, f, k), be.r["out"])   # 4 products and 3 adds, same order
        obs, obf = oracle_lib.block_extract_bwd(s, f, gb, k)
        magnitude_close(obs, be.r["gs"], be.r["Mgs"], 1e-12)
        magnitude_close(obf, be.r["gf"], be.r["Mgf"], 1e-12)


@pytest.mark.parametrize("k", [2, 3, 5, 8, 9])
@pytest.mark.parametrize("dt", sorted(DTYPES))
def test_irregular_flows_are_irregular(dt, k):
    """the irregular flows of each type select non-consecutive taps in that type, and the other type's do not in it"""
    A, other = DTYPES[dt], (f64 if DTYPES[dt] == f32 else f32)
    f = make_flow("irregular", np.random.default_rng(k), 1, 11, 29, k, A)
    assert (~ref64.Taps(f, k, 11, 29, A).regular).sum() >= 5
    assert ref64.Taps(f.astype(other), k, 11, 29, other).regular.mean() > 0.5


# --------------------------------------------------------------------------------------------- kernel emulation
def emu_softmax(lg, A, fault=None):
    """pixel_softmax (local_attn_pixel.cuh:19-35) in A: (k^2, B, H W)"""
    B, KK = lg.shape[:2]
    l = np.asarray(lg, A).reshape(B, KK, -1).transpose(1, 0, 2)
    m = l.max(0)
    e = np.exp((l - m).astype(A)).astype(A)
    s = np.zeros(m.shape, A)
    low = e.argmin(0)
    for t in range(KK):
        s = s + (np.where(low == t, A(0), e[t]) if fault == "drop_smallest" else e[t])
    return e * (A(1) / s)


def emu_axis(fl, k, coord, dim, A, fault=None):
    """axis_tap (common.cuh:52-64) for the k taps of every pixel: lo, hi, fl (int) and wlo, whi in A, each (k, B, H W)"""
    B = fl.shape[0]
    half = (k - 1) // 2 if fault == "half_offset" else k // 2
    off = (np.arange(k) - half).astype(A).reshape(k, 1, 1)
    d = (np.asarray(fl, A).reshape(1, B, -1) + off) + np.asarray(coord, A).reshape(1, 1, -1)
    fd = np.floor(d)
    lo = np.clip(fd.astype(np.int64), 0, dim - 1)
    hi = np.clip((fd + A(1)).astype(np.int64), 0, dim - 1)
    return lo, hi, fd.astype(np.int64), (A(1) - (d - fd)).astype(A), (d - fd).astype(A)


def emu_taps(f, k, Hs, Ws, A, fault=None):
    H, W = f.shape[2:]
    ys, xs = np.divmod(np.arange(H * W), W)
    TA = f32 if fault == "taps_fp32" else A
    ty = emu_axis(f[:, 1], k, ys, Hs, TA, fault)
    tx = emu_axis(f[:, 0], k, xs, Ws, TA, fault)
    cast = lambda t: t[:3] + tuple(w.astype(A) for w in t[3:])
    return cast(ty), cast(tx)


def collapsed(ty, tx, k):
    """(B, H W): the K = 2..5 instances take the collapsed window where both axes' taps are consecutive"""
    if not 2 <= k <= 5:
        return np.zeros(ty[2].shape[1:], bool)
    st = np.arange(k).reshape(k, 1, 1)
    return np.all(ty[2] == ty[2][:1] + st, 0) & np.all(tx[2] == tx[2][:1] + st, 0)


def emu_fwd(s, f, lg, k, A, fault=None):
    """k_local_attn_fwd (local_attn.cu:31-117) in A, operation by operation (without FMA contraction).
    -> out [B, C, H, W], probs [B, k^2, H, W]"""
    B, C, Hs, Ws = s.shape
    H, W = f.shape[2:]
    KK = k * k
    p = emu_softmax(lg, A, fault)
    (ylo, yhi, yfl, ywl, ywh), (xlo, xhi, xfl, xwl, xwh) = emu_taps(f, k, Hs, Ws, A, fault)
    S = np.asarray(s, A).reshape(B, C, -1)
    val = lambda pos: np.take_along_axis(S, pos[:, None, :], 2)
    inv = A(1) / A(KK)
    acc = np.zeros((B, C, H * W), A)
    for i in range(k - 1 if fault == "drop_row" else k):
        for j in range(k):
            v = np.zeros_like(acc)
            v = v + (xwl[j] * ywl[i])[:, None] * val(ylo[i] * Ws + xlo[j])
            v = v + (xwh[j] * ywl[i])[:, None] * val(ylo[i] * Ws + xhi[j])
            v = v + (xwl[j] * ywh[i])[:, None] * val(yhi[i] * Ws + xlo[j])
            v = v + (xwh[j] * ywh[i])[:, None] * val(yhi[i] * Ws + xhi[j])
            acc = acc + p[i * k + j][:, None] * v
    acc = acc * inv
    reg = collapsed((ylo, yhi, yfl), (xlo, xhi, xfl), k)
    if reg.any():
        K1 = k + 1
        Wc = [np.zeros(reg.shape, A) for _ in range(K1 * K1)]
        for i in range(k):
            for j in range(k):
                pij = p[i * k + j]
                Wc[i * K1 + j] = Wc[i * K1 + j] + pij * (xwl[j] * ywl[i])
                Wc[i * K1 + j + 1] = Wc[i * K1 + j + 1] + pij * (xwh[j] * ywl[i])
                Wc[(i + 1) * K1 + j] = Wc[(i + 1) * K1 + j] + pij * (xwl[j] * ywh[i])
                Wc[(i + 1) * K1 + j + 1] = Wc[(i + 1) * K1 + j + 1] + pij * (xwh[j] * ywh[i])
        cx = [np.clip(xfl[0] + r, 0, Ws - 1) for r in range(K1)]
        cy = [np.clip(yfl[0] + r, 0, Hs - 1) * Ws for r in range(K1)]
        a2 = np.zeros_like(acc)
        for r in range(K1):
            for q in range(K1):
                a2 = a2 + Wc[r * K1 + q][:, None] * val(cy[r] + cx[q])
        acc = np.where(reg[:, None], a2 * inv, acc)
    if fault == "ragged_last":              # the last channel of the last (ragged) slice is never written
        acc[:, C - 1] = 0
    return acc.reshape(B, C, H, W), p.transpose(1, 0, 2).reshape(B, KK, H, W)


def tap_backward(ty, tx, i, j, pij, scale, qLT, qRT, qLB, qRB):
    """tap_backward (local_attn_pixel.cuh:66-73) in A -> dp, d gfx, d gfy"""
    (_, _, _, ywl, ywh), (_, _, _, xwl, xwh) = ty, tx
    yl, yh, xl, xh = ywl[i], ywh[i], xwl[j], xwh[j]
    dp = scale * (yl * (xl * qLT + xh * qRT) + yh * (xl * qLB + xh * qRB))
    gy = pij * ((((-xl) * qLT - xh * qRT) + xl * qLB) + xh * qRB)
    gx = pij * ((((-yl) * qLT - yh * qLB) + yl * qRT) + yh * qRB)
    return dp, gx, gy


def emu_bwd(s, f, lg, g, k, A, order="seq", init=None, fault=None, drop=None):
    """k_local_attn_bwd (local_attn.cu:129-238) in A, operation by operation, with grad_source's partials added in the
    given order (seq, rev or shuffle) onto init[0] (or zeros).  drop = flat index of one partial to lose.
    -> gs, gf, gl; with fault == "partials" the partials (values, flat indices) instead"""
    B, C, Hs, Ws = s.shape
    H, W = f.shape[2:]
    N, KK, P = H * W, k * k, Hs * Ws
    p = emu_softmax(lg, A)
    ty, tx = emu_taps(f, k, Hs, Ws, A)
    (ylo, yhi, yfl, ywl, ywh), (xlo, xhi, xfl, xwl, xwh) = ty, tx
    S = np.asarray(s, A).reshape(B, C, -1)
    G = np.asarray(g, A).reshape(B, C, -1)
    inv = A(1) / A(KK)
    scale = {"kk_twice": inv * inv, "kk_never": A(1)}.get(fault, inv)
    reg = collapsed((ylo, yhi, yfl), (xlo, xhi, xfl), k)
    cidx = (np.arange(B)[:, None, None] * C + np.arange(C)[None, :, None]) * P       # (B, C, 1)
    vals, idx = [], []

    def scatter(v, pos, where):
        """v (B, C, N) partials at source positions pos (B, N) of the pixels where (B, N) takes this path"""
        w = np.broadcast_to(where[:, None], v.shape)
        vals.append(v[w])
        idx.append(np.broadcast_to(cidx + pos[:, None], v.shape)[w])

    def dots(pos):
        q = np.zeros((B, N), A)
        for c in range(C):
            q = q + G[:, c] * np.take_along_axis(S[:, c], pos, 1)
        return q

    dp = np.zeros((KK, B, N), A)
    gfx, gfy = np.zeros((B, N), A), np.zeros((B, N), A)
    lit = ~reg
    for i in range(k):
        for j in range(k):
            pos = [ylo[i] * Ws + xlo[j], ylo[i] * Ws + xhi[j], yhi[i] * Ws + xlo[j], yhi[i] * Ws + xhi[j]]
            wts = [xwl[j] * ywl[i], xwh[j] * ywl[i], xwl[j] * ywh[i], xwh[j] * ywh[i]]
            pij = p[i * k + j] * scale
            q = [dots(ps) for ps in pos]
            gp = G * pij[:, None]
            for ps, w in zip(pos, wts):
                scatter(gp * w[:, None], ps, lit)
            d, gx, gy = tap_backward(ty, tx, i, j, pij, scale, *q)
            dp[i * k + j] = np.where(lit, d, 0)
            gfx, gfy = np.where(lit, gfx + gx, gfx), np.where(lit, gfy + gy, gfy)
    if reg.any():
        K1 = k + 1
        Wc = [np.zeros((B, N), A) for _ in range(K1 * K1)]
        for i in range(k):
            for j in range(k):
                pij = p[i * k + j] * scale
                Wc[i * K1 + j] = Wc[i * K1 + j] + pij * (xwl[j] * ywl[i])
                Wc[i * K1 + j + 1] = Wc[i * K1 + j + 1] + pij * (xwh[j] * ywl[i])
                Wc[(i + 1) * K1 + j] = Wc[(i + 1) * K1 + j] + pij * (xwl[j] * ywh[i])
                Wc[(i + 1) * K1 + j + 1] = Wc[(i + 1) * K1 + j + 1] + pij * (xwh[j] * ywh[i])
        cx = [np.clip(xfl[0] + r, 0, Ws - 1) for r in range(K1)]
        cy = [np.clip(yfl[0] + r, 0, Hs - 1) * Ws for r in range(K1)]
        Q = [[dots(cy[r] + cx[c]) for c in range(K1)] for r in range(K1)]
        for r in range(K1):
            for c in range(K1):
                scatter(G * Wc[r * K1 + c][:, None], cy[r] + cx[c], reg)
        rx, ry = np.zeros((B, N), A), np.zeros((B, N), A)
        for i in range(k):
            for j in range(k):
                d, gx, gy = tap_backward(ty, tx, i, j, p[i * k + j] * scale, scale, Q[i][j], Q[i][j + 1], Q[i + 1][j],
                                         Q[i + 1][j + 1])
                dp[i * k + j] = np.where(reg, d, dp[i * k + j])
                rx, ry = rx + gx, ry + gy
        gfx, gfy = np.where(reg, rx, gfx), np.where(reg, ry, gfy)
    v, ix = np.concatenate(vals), np.concatenate(idx)
    if fault == "partials":
        return v, ix
    dot = np.zeros((B, N), A)
    for t in range(KK):
        dot = dot + p[t] * dp[t]
    gl = p * (dp - dot)
    gf = np.stack([gfy, gfx] if fault == "swap_axes" else [gfx, gfy], 1)
    gs = np.zeros(B * C * P, A)
    if init is not None and fault != "ignore_init":
        gs += np.broadcast_to(np.asarray(init[0], A), (B, C, Hs, Ws)).ravel()
        gf = np.asarray(init[1], A).reshape(B, 2, N) + gf
        gl = np.asarray(init[2], A).reshape(B, KK, N).transpose(1, 0, 2) + gl
    if drop is not None:
        v, ix = np.delete(v, drop), np.delete(ix, drop)
    perm = {"seq": np.arange(v.size), "rev": np.arange(v.size)[::-1],
            "shuffle": np.random.default_rng(0).permutation(v.size)}[order]
    np.add.at(gs, ix[perm], v[perm])
    return (gs.reshape(B, C, Hs, Ws), gf.reshape(B, 2, H, W), gl.transpose(1, 0, 2).reshape(B, KK, H, W))


def emu_be_bwd(s, f, g, k, A, slices, order="seq", init=None, fault=None):
    """k_block_extract_bwd (block_extract.cu:60-115) in A: grad_flow summed per slice (i, j outer, channels inner),
    slices == 1: one read-modify-write, else one atomic add per slice in the given order; grad_source partials
    (g wx) wy in the given order.  fault == "one_slice": only the last slice's partial reaches grad_flow"""
    B, C, Hs, Ws = s.shape
    H, W = f.shape[2:]
    N, P = H * W, Hs * Ws
    (ylo, yhi, _, ywl, ywh), (xlo, xhi, _, xwl, xwh) = emu_taps(f, k, Hs, Ws, A)
    S = np.asarray(s, A).reshape(B, C, -1)
    G6 = np.asarray(g, A).reshape(B, C, H, k, W, k)
    cps = -(-C // slices)
    part = []
    vals, idx = [], []
    cidx = (np.arange(B)[:, None] * C) * P
    for s0 in range(0, C, cps):
        gx, gy = np.zeros((B, N), A), np.zeros((B, N), A)
        for i in range(k):
            for j in range(k):
                pos = [ylo[i] * Ws + xlo[j], ylo[i] * Ws + xhi[j], yhi[i] * Ws + xlo[j], yhi[i] * Ws + xhi[j]]
                for c in range(s0, min(C, s0 + cps)):
                    gg = G6[:, c, :, i, :, j].reshape(B, N)
                    v = [np.take_along_axis(S[:, c], ps, 1) for ps in pos]
                    for ps, (wa, wb) in zip(pos, [(xwl, ywl), (xwh, ywl), (xwl, ywh), (xwh, ywh)]):
                        vals.append(((gg * wa[j]) * wb[i]).ravel())
                        idx.append((cidx + c * P + ps).ravel())
                    xl, xh, yl, yh = xwl[j], xwh[j], ywl[i], ywh[i]
                    gy = gy + gg * ((((-xl) * v[0] - xh * v[1]) + xl * v[2]) + xh * v[3])
                    gx = gx + gg * ((((-yl) * v[0] - yh * v[2]) + yl * v[1]) + yh * v[3])
        part.append(np.stack([gx, gy], 1))
    gf = np.zeros((B, 2, N), A) if init is None else np.asarray(init[1], A).reshape(B, 2, N).copy()
    if fault == "one_slice":
        part = part[-1:]
    ordr = {"seq": range(len(part)), "rev": range(len(part) - 1, -1, -1),
            "shuffle": np.random.default_rng(1).permutation(len(part))}[order]
    for n in ordr:
        gf = gf + part[n]
    gs = np.zeros(B * C * P, A)
    if init is not None:
        gs += np.broadcast_to(np.asarray(init[0], A), (B, C, Hs, Ws)).ravel()
    v, ix = np.concatenate(vals), np.concatenate(idx)
    perm = {"seq": np.arange(v.size), "rev": np.arange(v.size)[::-1],
            "shuffle": np.random.default_rng(2).permutation(v.size)}[order]
    np.add.at(gs, ix[perm], v[perm])
    return gs.reshape(B, C, Hs, Ws), gf.reshape(B, 2, H, W)


# ----------------------------------------------------------------------------------------------- the checks
def check_all(la, s, g, y_fwd=None, y_bwd=None, C=None, init=None, prev=None, mask=None, y_blend=None):
    """-> {name: (worst, message)} of the given forward (out, probs) and backward (gs, gf, gl) results"""
    res = {}
    if y_fwd is not None:
        out, mags = la.fwd(s)
        res["out"] = ref64.check("out", y_fwd[0], out, la.bound_out(mags))
        res["probs"] = ref64.check("probs", y_fwd[1], la.probs(), la.bound_probs())
        if y_blend is not None:
            rb, _ = ref64.blend_ref(out, mags["M"], prev, mask)
            res["blend"] = ref64.check("blend", y_blend, rb, la.bound_blend(rb, mags, prev, mask))
    if y_bwd is not None:
        r = la.bwd(s, g)
        i0, i1, i2 = (0.0, 0.0, 0.0) if init is None else (np.asarray(x, f64) for x in init)
        res["grad_source"] = ref64.check("grad_source", y_bwd[0], r["gs"] + i0, la.bound_gs(r, i0))
        res["grad_flow"] = ref64.check("grad_flow", y_bwd[1], r["gf"] + i1, la.bound_gf(r, C, i1))
        res["grad_logits"] = ref64.check("grad_logits", y_bwd[2], r["gl"] + i2, la.bound_gl(r, C, i2))
    return res


def assert_ok(res):
    for name, (worst, msg) in res.items():
        assert msg is None, msg


@pytest.mark.parametrize("k", range(1, 10))
@pytest.mark.parametrize("dt", sorted(DTYPES))
def test_oracle_within_bounds(oracle_lib, dt, k):
    """the oracle sums in the reference's order (block tensor, then avg_pool; g / k^2 before the products)"""
    A = DTYPES[dt]
    for i, kind in enumerate(["smooth", "border", "irregular", "span3"]):
        B, C, Hs, Ws, H, W = shape(k, i)
        s, f, lg, g = inputs(B, C, Hs, Ws, H, W, k, kind, 10 * k + i, A, LOGITS[i % 3])
        la = rg.LocalAttn(f, lg, k, Hs, Ws, A)
        ofwd = oracle_lib.local_attn_fwd(s, f, lg, k, return_probs=True)
        assert_ok(check_all(la, s, g, ofwd, oracle_lib.local_attn_bwd(s, f, lg, g, k), C))
        gb = np.random.default_rng(i).standard_normal((B, C, k * H, k * W)).astype(A)
        be = rg.BlockExtract(s, f, k, gb, A)
        obs, obf = oracle_lib.block_extract_bwd(s, f, gb, k)
        assert ref64.check("be gs", obs, be.r["gs"], be.bound_gs())[1] is None
        assert ref64.check("be gf", obf, be.r["gf"], be.bound_gf())[1] is None


EMU_KINDS = ["smooth", "iid", "border", "outside", "irregular"]


@pytest.mark.parametrize("k", range(1, 10))
@pytest.mark.parametrize("dt", sorted(DTYPES))
def test_emulation_within_bounds(dt, k):
    """the kernels' operation order (collapsed window for k = 2..5, literal path otherwise and for irregular pixels),
    three scatter orders, accumulate onto a non-zero buffer, the fused blend; both block_extractor grad_flow paths"""
    A = DTYPES[dt]
    worst = {}
    for i, kind in enumerate(EMU_KINDS):
        B, C, Hs, Ws, H, W = shape(k, i)
        s, f, lg, g = inputs(B, C, Hs, Ws, H, W, k, kind, 7 * k + i, A, LOGITS[i % 3])
        la = rg.LocalAttn(f, lg, k, Hs, Ws, A)
        rng = np.random.default_rng(i)
        prev, mask = rng.standard_normal((B, C, H, W)).astype(A), rng.uniform(0, 1, (B, 1, H, W)).astype(A)
        out, probs = emu_fwd(s, f, lg, k, A)
        blend = prev * (A(1) - mask) + out * mask
        res = check_all(la, s, g, (out, probs), None, C, prev=prev.astype(f64), mask=mask.astype(f64), y_blend=blend)
        order = ["seq", "rev", "shuffle"][i % 3]
        res.update(check_all(la, s, g, None, emu_bwd(s, f, lg, g, k, A, order), C))
        init = (A(0.5), rng.standard_normal(f.shape).astype(A), rng.standard_normal(lg.shape).astype(A))
        acc = check_all(la, s, g, None, emu_bwd(s, f, lg, g, k, A, order, init=init), C, init=init)
        res.update({n + " accumulate": v for n, v in acc.items()})
        gb = rng.standard_normal((B, C, k * H, k * W)).astype(A)
        be = rg.BlockExtract(s, f, k, gb, A)
        ib = (rng.standard_normal(s.shape).astype(A), rng.standard_normal(f.shape).astype(A))
        for slices in (1, 2, C):
            bs, bf = emu_be_bwd(s, f, gb, k, A, slices, order)
            res[f"be gs slices={slices}"] = ref64.check("be gs", bs, be.r["gs"], be.bound_gs())
            res[f"be gf slices={slices}"] = ref64.check("be gf", bf, be.r["gf"], be.bound_gf())
            bs, bf = emu_be_bwd(s, f, gb, k, A, slices, order, init=ib)
            res[f"be gf slices={slices} accumulate"] = ref64.check("be gf", bf, be.r["gf"] + ib[1], be.bound_gf(ib[1]))
            res[f"be gs slices={slices} accumulate"] = ref64.check("be gs", bs, be.r["gs"] + ib[0], be.bound_gs(ib[0]))
        assert_ok(res)
        for n, (w, _) in res.items():
            worst[n] = max(worst.get(n, 0.0), w)
    # not vacuous: the forward and the scatter come within a factor of 1000 of their bounds (worst-case sums with
    # gamma's 4x headroom, against rounding that grows about as the square root of the number of terms)
    assert worst["out"] > 1e-3 and worst["grad_source"] > 1e-3, worst


# --------------------------------------------------------------------------------------------------- faults
def flat(name, A, y, ref):
    """would test_gpu_parity's flat tolerances (t = 1e-5 fp32, 1e-12 fp64; test_local_attn_vs_oracle,
    test_block_extractor_vs_oracle) accept y?"""
    t = 1e-5 if A == f32 else 1e-12
    rtol, atol = {"out": (t, t), "grad_source": (10 * t, 10 * t), "grad_flow": (100 * t, 100 * t),
                  "grad_logits": (100 * t, 10 * t), "be gf": (2 * t, 2 * t * max(1.0, float(np.abs(ref).max())))}[name]
    return bool((np.abs(np.asarray(y, f64) - ref) <= atol + rtol * np.abs(ref)).all())


def fault_fwd(fault, k, A=f32, kind="smooth", C=5):
    s, f, lg, g = inputs(1, C, 14, 17, 11, 13, k, kind, 3, A)
    la = rg.LocalAttn(f, lg, k, 14, 17, A)
    y = emu_fwd(s, f, lg, k, A, fault)[0]
    out, mags = la.fwd(s)
    return ref64.check("out", y, out, la.bound_out(mags)), flat("out", A, y, out)


def fault_bwd(fault, output, k=3, A=f32, init=None, drop=None):
    s, f, lg, g = inputs(1, 5, 14, 17, 11, 13, k, "smooth", 4, A)
    la = rg.LocalAttn(f, lg, k, 14, 17, A)
    ys = dict(zip(["grad_source", "grad_flow", "grad_logits"],
                  emu_bwd(s, f, lg, g, k, A, init=init, fault=fault, drop=drop)))
    res = check_all(la, s, g, None, tuple(ys.values()), 5, init=init)
    r = la.bwd(s, g)
    key = {"grad_source": "gs", "grad_flow": "gf", "grad_logits": "gl"}[output]
    ref = r[key] + (0.0 if init is None else np.asarray(init[["gs", "gf", "gl"].index(key)], f64))
    return res[output], flat(output, A, ys[output], ref)


def fault_small_partial():
    """one grad_source partial of size ~3e-6 is lost (a partial added to the wrong buffer, or a lost atomic)"""
    s, f, lg, g = inputs(1, 5, 14, 17, 11, 13, 3, "smooth", 4, f32)
    v, _ = emu_bwd(s, f, lg, g, 3, f32, fault="partials")
    drop = int(np.argmin(np.abs(np.abs(v) - 3e-6)))
    return fault_bwd(None, "grad_source", drop=drop)


def fault_be_one_slice():
    B, C, Hs, Ws, H, W, k = 1, 6, 14, 17, 11, 13, 3
    s, f, _, _ = inputs(B, C, Hs, Ws, H, W, k, "smooth", 5, f32)
    gb = np.random.default_rng(5).standard_normal((B, C, k * H, k * W)).astype(f32)
    be = rg.BlockExtract(s, f, k, gb, f32)
    y = emu_be_bwd(s, f, gb, k, f32, 3, fault="one_slice")[1]
    return ref64.check("be gf", y, be.r["gf"], be.bound_gf()), flat("be gf", f32, y, be.r["gf"])


INIT = (f32(0.5), np.full((1, 2, 11, 13), -0.25, f32), np.full((1, 9, 11, 13), 0.125, f32))

# name -> (the fault's check, whether test_gpu_parity's flat tolerances accept the faulty result).  Only the small lost
# partial passes them; of the faults they reject, the dropped row (k >= 7), the ignored accumulate buffer and the ragged
# last slice are in cases test_gpu_parity never ran.
FAULTS = {
    "dropped last tap row, k = 7": (lambda: fault_fwd("drop_row", 7), False),
    "i - (k-1)/2 for even k": (lambda: fault_fwd("half_offset", 4), False),
    "inv_kk twice in the backward": (lambda: fault_bwd("kk_twice", "grad_logits"), False),
    "inv_kk never in the backward": (lambda: fault_bwd("kk_never", "grad_flow"), False),
    "softmax's smallest term dropped": (lambda: fault_fwd("drop_smallest", 3, kind="iid"), False),
    "fp32 taps in an fp64 kernel": (lambda: fault_fwd("taps_fp32", 3, A=f64), False),
    "last channel of a ragged slice skipped": (lambda: fault_fwd("ragged_last", 9, C=3), False),
    "one atomic partial dropped": (fault_small_partial, True),
    "exchanged grad_flow axes": (lambda: fault_bwd("swap_axes", "grad_flow"), False),
    "accumulate ignores the buffer": (lambda: fault_bwd("ignore_init", "grad_logits", init=INIT), False),
    "block_extractor grad_flow of one slice only": (fault_be_one_slice, False),
}


@pytest.mark.parametrize("fault", sorted(FAULTS))
def test_injected_fault_fails_its_bound(fault):
    check, flat_accepts = FAULTS[fault]
    (worst, msg), accepted = check()
    assert msg is not None, f"{fault}: worst |err|/bound {worst:.3g} stays within the bound"
    assert accepted == flat_accepts, (fault, accepted)


# ------------------------------------------------------------------------------------------------ host mirror
def test_launch_slices_mirror():
    """what the GPU cases rely on: C = 1 one slice, small images C >= 2 several, ragged last slices for C = 3 and 130,
    and one slice once the pixels alone fill the machine"""
    assert rg.launch_slices(300, 1, 128, 132) == (1, 1)
    assert rg.launch_slices(300, 48, 128, 132) == (24, 2)
    assert rg.launch_slices(300, 3, 128, 132) == (2, 2)             # 2 + 1
    assert rg.launch_slices(300, 130, 128, 132) == (44, 3)          # 43 x 3 + 1
    assert rg.launch_slices(128 * 4 * 132 * 16, 64, 128, 132) == (1, 64)
    assert rg.launch_slices(128 * 4 * 114 * 16, 64, 128, 132)[0] == 2
