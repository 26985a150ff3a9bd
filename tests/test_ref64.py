"""CPU: the fp64 reference (ref64) against the fp32 oracle, and its 16-bit error bounds against numpy emulations of the
kernels' roundings: correct arithmetic must pass, plausible kernel bugs must not."""
import numpy as np
import pytest

import ref64
from test_gpu_parity import _flow, _irregular_flow_values
from test_gpu_tile_masks import _mask_flow

FLOWS = ["smooth", "iid", "border", "zero", "int", "rows", "halves", "outside", "span3", "irregular"]


def make_flow(kind, rng, B, H, W, k):
    if kind in ("rows", "halves", "outside", "span3"):
        return _mask_flow(kind, rng, B, H, W)
    if kind == "irregular":
        f = rng.uniform(-3, 3, (B, 2, H, W)).astype(np.float32)
        for i, (x, v) in enumerate(_irregular_flow_values(range(2, W - 2, 3), k, rng).items()):
            f[:, 0, (5 * i) % H, x] = v
        return f
    return _flow(rng, kind, B, H, W).astype(np.float32)


def bf16(a):
    return ref64.round_bf16(a).astype(np.float32)


def inputs(B, C, Hs, Ws, H, W, k, kind, seed):
    rng = np.random.default_rng(seed)
    s = bf16(rng.standard_normal((B, C, Hs, Ws)))
    f = make_flow(kind, rng, B, H, W, k)
    lg = bf16(2 * rng.standard_normal((B, k * k, H, W)))
    g = bf16(rng.standard_normal((B, C, H, W)))
    return s, f, lg, g


def close(a, ref, mag, rel=2.0 ** -18):
    """fp32 accuracy scaled by the magnitude (the oracle sums in fp32)"""
    err = np.abs(np.asarray(a, np.float64) - ref)
    assert float((err - rel * (mag + np.abs(ref)) - 1e-30).max()) <= 0, float(err.max())


@pytest.mark.parametrize("k", [1, 2, 3, 4, 5, 6])
@pytest.mark.parametrize("kind", FLOWS)
def test_ref64_matches_oracle(oracle_lib, kind, k):
    B, C, Hs, Ws, H, W = (1, 8, 22, 29, 17, 23) if k % 2 else (2, 5, 17, 23, 17, 23)   # source larger than the flow, or not
    s, f, lg, g = inputs(B, C, Hs, Ws, H, W, k, kind, seed=11 * k + len(kind))
    la = ref64.LocalAttn(f, lg, k, Hs, Ws)
    out, M = la.fwd(s)
    oout, oprobs = oracle_lib.local_attn_fwd(s, f, lg, k, return_probs=True)
    close(oout, out, M)
    close(oprobs, la.probs(), 1.0)
    r = la.bwd(s, g)
    ogs, ogf, ogl = oracle_lib.local_attn_bwd(s, f, lg, g, k)
    close(ogs, r["gs"], r["Mgs"])
    close(ogl, r["gl"], la.probs() * (r["D"] + r["PD"]))
    close(ogf, r["gf"], r["Mgf"])
    if kind == "irregular" and k > 1:       # one tap per axis is always consecutive
        assert not la.taps.regular.all()


def test_block_extract_ref64_matches_oracle(oracle_lib):
    for kind, k in (("smooth", 3), ("border", 4), ("irregular", 5)):
        s, f, _, _ = inputs(1, 6, 15, 19, 11, 13, k, kind, seed=k)
        g = bf16(np.random.default_rng(k).standard_normal((1, 6, k * 11, k * 13)))
        r = ref64.block_extract(s, f, k, g)
        close(oracle_lib.block_extract_fwd(s, f, k), r["out"], r["M"])
        ogs, ogf = oracle_lib.block_extract_bwd(s, f, g, k)
        close(ogs, r["gs"], r["Mgs"])
        close(ogf, r["gf"], r["Mgf"], rel=2.0 ** -16)


# ------------------------------------------------------------------------------------------- emulated kernels
def w_bf16(la):
    """the tile kernels' collapsed windows: every summed weight rounded to bf16 once"""
    return [sps_round(w) for w in la.W]


def sps_round(w):
    w = w.copy()
    w.data = ref64.round_bf16(w.data)
    return w


def tile_fwd(la, s, mats=None):
    mats = w_bf16(la) if mats is None else mats
    t = la.taps
    return ref64.round_bf16(la._apply(mats, s, (t.H, t.W)))


def groups(t):
    """pixel indices of every 16x8 group, row-major per image"""
    ys, xs = np.divmod(np.arange(t.H * t.W), t.W)
    gid = (ys // ref64.GH) * ((t.W + ref64.GW - 1) // ref64.GW) + xs // ref64.GW
    return [np.flatnonzero(gid == i) for i in range(int(gid.max()) + 1)]


def tile_bwd_gs(la, g, rng, drop=None):
    """grad_source of the tile backward: per group a bf16-rounded partial (fp64 sum of bf16 window x grad_out), added
    with one bf16 rounding per add in a shuffled group order inside the image, summed exactly and rounded once on the
    border.  drop = (b, group, positions) loses those adds."""
    t = la.taps
    B, C = g.shape[:2]
    acc = np.zeros((B, t.Hs * t.Ws, C))
    border = ref64.border_mask(t.Hs, t.Ws).ravel()
    gr = groups(t)
    for b in range(B):
        edge = np.zeros((t.Hs * t.Ws, C))
        wb = sps_round(la.W[b])
        G = np.asarray(g[b], np.float64).reshape(C, -1).T
        for gi in rng.permutation(len(gr)):
            rows = wb[gr[gi]]
            cols = np.unique(rows.indices)
            if drop is not None and drop[0] == b and drop[1] == gi:
                cols = np.setdiff1d(cols, drop[2])
            raw = rows[:, cols].T @ G[gr[gi]]
            inner = ~border[cols]
            acc[b, cols[inner]] = ref64.round_bf16(acc[b, cols[inner]] + ref64.round_bf16(raw[inner]))
            edge[cols[~inner]] += raw[~inner]
        acc[b, border] = ref64.round_bf16(acc[b, border] + edge[border])
    return acc.transpose(0, 2, 1).reshape(B, C, t.Hs, t.Ws)


SHAPE = (1, 64, 24, 40, 24, 40)


@pytest.fixture(scope="module")
def case5():
    B, C, Hs, Ws, H, W = SHAPE
    s, f, lg, g = inputs(B, C, Hs, Ws, H, W, 5, "smooth", seed=5)
    la = ref64.LocalAttn(f, lg, 5, Hs, Ws)
    out, M = la.fwd(s)
    return dict(s=s, f=f, lg=lg, g=g, la=la, out=out, M=M, r=la.bwd(s, g))


def fwd_ok(y, c):
    return ref64.check("out", y, c["out"], ref64.bound_out_tile(c["out"], c["M"], ref64.U_BF16, ref64.ETA_BF16))


def test_bounds_accept_emulated_tile_forward(case5):
    worst, msg = fwd_ok(tile_fwd(case5["la"], case5["s"]), case5)
    assert msg is None, msg
    assert worst > 0.1          # the bound is not vacuous


def test_bounds_accept_emulated_tile_backward_grad_source(case5):
    c = case5
    gs = tile_bwd_gs(c["la"], c["g"], np.random.default_rng(0))
    bound = ref64.bound_gs_tile(c["r"]["Mgs"], c["r"]["n_adds"][:, None], ref64.U_BF16, ref64.ETA_BF16)
    assert ref64.assert_within("grad_source", gs, c["r"]["gs"], bound) > 0.05


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_bounds_accept_single_rounding_gather(case5, dt):
    import ref64_gather
    c = case5
    u, eta = ref64.storage(dt)
    rnd = ref64.round_bf16 if dt == "bf16" else ref64.round_fp16
    g32 = ref64_gather.LocalAttn(c["f"], c["lg"], 5, SHAPE[2], SHAPE[3], np.float32)
    out, mags = g32.fwd(c["s"])
    r = g32.bwd(c["s"], c["g"])
    p = g32.probs()
    b = lambda y, e32: ref64.bound_gather16(y, e32, u, eta)
    worst = [ref64.assert_within("out", rnd(out), out, b(out, g32.bound_out(mags))),
             ref64.assert_within("probs", rnd(p), p, b(p, g32.bound_probs())),
             ref64.assert_within("gs", rnd(r["gs"]), r["gs"], b(r["gs"], g32.bound_gs(r))),
             ref64.assert_within("gl", rnd(r["gl"]), r["gl"], b(r["gl"], g32.bound_gl(r, 64))),
             ref64.assert_within("gf", rnd(r["gf"]), r["gf"], b(r["gf"], g32.bound_gf(r, 64)))]
    assert min(worst) > 0.3


# ------------------------------------------------------------------------------------------- injected faults
def rebuilt(la, edit):
    """a copy of la's windows with tap arrays edited by edit(taps), rebuilt"""
    import copy
    lb = copy.deepcopy(la)
    edit(lb.taps)
    lb.taps.build()
    lb.build()
    return lb


def flat_accepts(y, ref):
    return bool(np.abs(y - ref).max() <= 1e-2)


def reject(name, y, ref, bound, report):
    _, msg = ref64.check(name, y, ref, bound)
    report[name] = flat_accepts(y, ref)
    assert msg is not None, f"{name}: fault not detected"


@pytest.fixture(scope="module")
def report():
    r = {}
    yield r
    print("\nfaults the flat 1e-2 tolerance accepts:", sorted(n for n, ok in r.items() if ok))


def test_bounds_reject_forward_faults(case5, report):
    c = case5
    la, s = c["la"], c["s"]
    t = la.taps
    mats = w_bf16(la)
    bound = ref64.bound_out_tile(c["out"], c["M"], ref64.U_BF16, ref64.ETA_BF16)

    # a 16-pixel group row loses one source row of its window (row mask wrong): group row y = 9, pixels x 16..31
    m = mats[0].tolil()
    pix = 9 * t.W + np.arange(16, 32)
    y0 = int(t.pos[0, 0, 0, 0, pix[0]] // t.Ws) + 1
    for n in pix:
        for col in list(m.rows[n]):
            if col // t.Ws == y0:
                m[n, col] = 0
    reject("row_mask", tile_fwd(la, s, [m.tocsr()]), c["out"], bound, report)

    # one pixel loses its rightmost window column
    m = mats[0].tolil()
    n = 12 * t.W + 20
    right = max(col % t.Ws for col in m.rows[n])
    for col in list(m.rows[n]):
        if col % t.Ws == right:
            m[n, col] = 0
    reject("window_column", tile_fwd(la, s, [m.tocsr()]), c["out"], bound, report)

    # a border-folded weight lands one position inside the image: pixel (3, 0), whose window folds onto column 0
    m = mats[0].tolil()
    n = 3 * t.W
    for col in [cc for cc in m.rows[n] if cc % t.Ws == 0]:
        m[n, col + 1] += m[n, col]
        m[n, col] = 0
    reject("border_fold", tile_fwd(la, s, [m.tocsr()]), c["out"], bound, report)

    # wlo and whi swapped on the x axis of one pixel
    def swap(tp):
        lo, hi = tp.tx[3].copy(), tp.tx[4].copy()
        tp.tx[3][:, 0, 7, 9], tp.tx[4][:, 0, 7, 9] = hi[:, 0, 7, 9], lo[:, 0, 7, 9]
    reject("wlo_whi_swap", tile_fwd(la, s, w_bf16(rebuilt(la, swap))), c["out"], bound, report)

    # the ragged last group is dropped (W = 40: the last group column holds 8 pixels)
    y = tile_fwd(la, s)
    y[:, :, 16:24, 32:40] = 0
    reject("ragged_group", y, c["out"], bound, report)


def test_bounds_reject_second_channel_pass_dropped(report):
    """C = 512: the backward's second 256-channel pass is lost for one group, so that group's dot products miss half the
    channels"""
    B, C, Hs, Ws, H, W = 1, 512, 16, 32, 16, 32
    s, f, lg, g = inputs(B, C, Hs, Ws, H, W, 3, "smooth", seed=9)
    la = ref64.LocalAttn(f, lg, 3, Hs, Ws)
    r = la.bwd(s, g)
    half = la.bwd(s[:, :256], g[:, :256])
    gl = r["gl"].copy()
    gl[:, :, 8:16, 16:32] = half["gl"][:, :, 8:16, 16:32]
    bound = ref64.bound_gl(r["gl"], la.probs(), r["D"], r["PD"], C, ref64.U_BF16, ref64.ETA_BF16)
    assert ref64.assert_within("gl", ref64.round_bf16(r["gl"]), r["gl"], bound) < 1
    reject("second_pass", ref64.round_bf16(gl), r["gl"], bound, report)


def test_bounds_reject_backward_faults(case5, report):
    c = case5
    la, r = c["la"], c["r"]
    t = la.taps
    bgs = ref64.bound_gs_tile(r["Mgs"], r["n_adds"][:, None], ref64.U_BF16, ref64.ETA_BF16)
    # one group's grad_source adds for one step (16 positions of a source row in its footprint) are lost
    col = int(la.W[0][groups(t)[7]].indices.min())
    step = col + np.arange(16)
    gs = tile_bwd_gs(la, c["g"], np.random.default_rng(1), drop=(0, 7, step))
    reject("lost_step", gs, r["gs"], bgs, report)

    # one tap's dp is taken off the wrong corner (RT's dot product in place of LT's) for one pixel
    q = r["q"].copy()
    q[0, 2, 1, 0, 300] = q[0, 2, 1, 1, 300]
    bad = la.grads_from_q(q)
    bgl = ref64.bound_gl(r["gl"], la.probs(), r["D"], r["PD"], 64, ref64.U_BF16, ref64.ETA_BF16)
    reject("dp_corner", ref64.round_bf16(bad["gl"]), r["gl"], bgl, report)

    # one corner term of grad_flow has its sign flipped: tap (2, 1), corner LB of the y gradient, pixel 300
    pij = la.p[0, 2 * 5 + 1].ravel()[300] / 25
    gf = r["gf"].copy()
    gf[0, 1].ravel()[300] -= 2 * pij * t.wx[0][1, 0, 300] * r["q"][0, 2, 1, 2, 300]
    bgf = ref64.bound_gf(r["gf"], r["Mgf"], 64)
    assert ref64.assert_within("gf", r["gf"].astype(np.float32), r["gf"], bgf) < 1
    reject("gf_sign", gf, r["gf"], bgf, report)
