"""fp16 twins of the tile kernels' emulations and bounds (ref64, test_ref64): the tensor-core local-attention kernels in
fp16 storage (k_local_attn_fwd_tc*<..., __half>, k_local_attn_bwd_tc<..., __half>).

fp16 differs from bf16 in range, not only in precision.  A window weight p w / k^2 below 2^-14 is subnormal in fp16 and
rounds with an absolute error of up to ETA_W = 2^-25, which is not a multiple of its own size.  ref64's tile bounds add
their absolute floor eta once per output, so they do not cover that: the bounds here carry one ETA_W per non-zero weight,
times the magnitude it multiplies (A = |W|_0 |S| forward, |W|_0^T |G| for grad_source, |W|_0 the 0/1 pattern of the
collapsed window).
"""
import numpy as np

import ref64
import ref64_det

# half the spacing of fp16's subnormals: the largest rounding error of any weight that is stored as a subnormal
ETA_W = 2.0 ** -25


def round_fp16(x):
    """round to nearest even fp16, subnormals included (through fp32, as __float2half_rn of an fp32 value), as fp64"""
    return ref64.round_fp16(x)


def sps_round16(w):
    w = w.copy()
    w.data = round_fp16(w.data)
    return w


def w_fp16(la):
    """the tile kernels' collapsed windows in fp16: every summed weight rounded to fp16 once"""
    return [sps_round16(w) for w in la.W]


def pattern(la):
    """|W|_0 per image: 1 where the collapsed window has a non-zero weight"""
    out = []
    for w in la.W:
        p = w.copy()
        p.data = (p.data != 0).astype(np.float64)
        out.append(p)
    return out


def weight_mag_fwd(la, s):
    """A = |W|_0 |S|: the source magnitudes the forward's weights multiply, one per non-zero weight"""
    t = la.taps
    return la._apply(pattern(la), np.abs(np.asarray(s, np.float64)), (t.H, t.W))


def weight_mag_gs(la, g):
    """|W|_0^T |G|: the grad_out magnitudes each grad_source element's weights multiply"""
    t = la.taps
    return la._apply([p.T.tocsr() for p in pattern(la)], np.abs(np.asarray(g, np.float64)), (t.Hs, t.Ws))


def groups(t):
    """pixel indices of every 16x8 group, row-major per image"""
    ys, xs = np.divmod(np.arange(t.H * t.W), t.W)
    gid = (ys // ref64.GH) * ((t.W + ref64.GW - 1) // ref64.GW) + xs // ref64.GW
    return [np.flatnonzero(gid == i) for i in range(int(gid.max()) + 1)]


def tile_fwd16(la, s, mats=None):
    """the tile forward in fp16: fp16 window, exact sums (the fp32 accumulators are inside FP32_SLACK), one fp16 store"""
    mats = w_fp16(la) if mats is None else mats
    t = la.taps
    return round_fp16(la._apply(mats, s, (t.H, t.W)))


def tile_bwd_gs16(la, g, rng, drop=None):
    """grad_source of the fp16 tile backward: per group an fp16-rounded partial (sum of fp16 window x grad_out), added with
    one fp16 rounding per add in a shuffled group order inside the image, summed exactly and rounded once on the border
    (k_fold_border).  drop = (b, group, positions) loses those adds."""
    t = la.taps
    B, C = g.shape[:2]
    acc = np.zeros((B, t.Hs * t.Ws, C))
    border = ref64.border_mask(t.Hs, t.Ws).ravel()
    gr = groups(t)
    for b in range(B):
        edge = np.zeros((t.Hs * t.Ws, C))
        wb = sps_round16(la.W[b])
        G = np.asarray(g[b], np.float64).reshape(C, -1).T
        for gi in rng.permutation(len(gr)):
            rows = wb[gr[gi]]
            cols = np.unique(rows.indices)
            if drop is not None and drop[0] == b and drop[1] == gi:
                cols = np.setdiff1d(cols, drop[2])
            raw = rows[:, cols].T @ G[gr[gi]]
            inner = ~border[cols]
            acc[b, cols[inner]] = round_fp16(acc[b, cols[inner]] + round_fp16(raw[inner]))
            edge[cols[~inner]] += raw[~inner]
        acc[b, border] = round_fp16(acc[b, border] + edge[border])
    return acc.transpose(0, 2, 1).reshape(B, C, t.Hs, t.Ws)


# ----------------------------------------------------------------------------------------------------------- bounds
# u, eta = ref64.storage("fp16").  A / Ags: weight_mag_fwd / weight_mag_gs.

def bound_out_tile16(r, M, A, u, eta):
    """tile forward in fp16: the fp16 window (u of each normal weight, u M; ETA_W of each subnormal one, ETA_W A), the fp32
    accumulation (FP32_SLACK M) and one fp16 store (u |r + error| + eta; the 1.01 pays for u of the error terms)"""
    return 1.01 * (u * (np.abs(r) + M) + ETA_W * A) + ref64.FP32_SLACK * M + eta


def bound_out_tile16_blend(r, M, Mattn, Aattn, u, eta):
    """tile forward with blend: the window terms scale with the attention part only (Mattn = m W|S|, Aattn = m A); M =
    ref64.blend_ref's magnitude"""
    return 1.01 * (u * (np.abs(r) + Mattn) + ETA_W * Aattn) + ref64.FP32_SLACK * M + eta


def bound_gs_tile16(Mgs, Ags, n_adds, u, eta, init=0.0):
    """tile backward grad_source in fp16: per element n_adds roundings of the running sum (<= Mgs + |init|), each u of it
    plus eta (subnormal sums), and as many fp16 roundings of a group's partial (u Mgs in total, eta each); the fp16 window
    (u Mgs + ETA_W Ags); fp32 MMA accumulation of the partials (FP32_SLACK Mgs)"""
    return u * (n_adds + 2) * (Mgs + np.abs(init)) + ETA_W * Ags + ref64.FP32_SLACK * Mgs + (2 * n_adds + 1) * eta


def bound_gs_tile16_det(r, Mgs, Ags, E, n, u, eta):
    """deterministic tile backward in fp16 (k_local_attn_bwd_tc<K, CN, true, __half>): ref64_det.bound_gs_tile (fp16 window
    u Mgs, the fp32 GEMM sums, quantisation, int64 -> double, one rounding) plus the subnormal weights' ETA_W Ags"""
    return ref64_det.bound_gs_tile(r, Mgs, E, n, u, eta) + 1.01 * ETA_W * Ags
