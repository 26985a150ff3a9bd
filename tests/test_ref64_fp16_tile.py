"""CPU: the fp16 tile bounds (ref64_tile16) against numpy emulations of the fp16 tile kernels' roundings, subnormal weights
included: correct arithmetic must pass with a non-vacuous margin, the injected faults of test_ref64 must not."""
import numpy as np
import pytest

import ref64
import ref64_tile16 as T16
from test_ref64 import make_flow

U, ETA = ref64.storage("fp16")
SHAPE = (1, 64, 24, 40, 24, 40)


def inputs16(B, C, Hs, Ws, H, W, k, kind, seed):
    rng = np.random.default_rng(seed)
    f16 = lambda a: T16.round_fp16(a).astype(np.float32)
    s = f16(rng.standard_normal((B, C, Hs, Ws)))
    f = make_flow(kind, rng, B, H, W, k)
    lg = f16(2 * rng.standard_normal((B, k * k, H, W)))
    g = f16(rng.standard_normal((B, C, H, W)))
    return s, f, lg, g


@pytest.fixture(scope="module", params=[3, 5])
def case(request):
    k = request.param
    B, C, Hs, Ws, H, W = SHAPE
    s, f, lg, g = inputs16(B, C, Hs, Ws, H, W, k, "smooth", seed=5 + k)
    la = ref64.LocalAttn(f, lg, k, Hs, Ws)
    out, M = la.fwd(s)
    return dict(k=k, s=s, g=g, la=la, out=out, M=M, A=T16.weight_mag_fwd(la, s), r=la.bwd(s, g), Ags=T16.weight_mag_gs(la, g))


def fwd_bound(c):
    return T16.bound_out_tile16(c["out"], c["M"], c["A"], U, ETA)


def gs_bound(c):
    return T16.bound_gs_tile16(c["r"]["Mgs"], c["Ags"], c["r"]["n_adds"][:, None], U, ETA)


def test_windows_hold_subnormal_weights(case):
    """the case exercises what the per-weight term is for: some window weights are fp16 subnormals"""
    w = np.concatenate([m.data for m in case["la"].W])
    assert ((np.abs(w) < 2.0 ** -14) & (w != 0)).sum() > 100


def test_bounds_accept_emulated_fp16_tile_forward(case):
    worst = ref64.assert_within("out fp16", T16.tile_fwd16(case["la"], case["s"]), case["out"], fwd_bound(case))
    assert worst > 0.1          # the bound is not vacuous


def test_bounds_accept_emulated_fp16_tile_backward_grad_source(case):
    gs = T16.tile_bwd_gs16(case["la"], case["g"], np.random.default_rng(0))
    assert ref64.assert_within("grad_source fp16", gs, case["r"]["gs"], gs_bound(case)) > 0.1


def test_det_bound_accepts_exact_sums_of_fp16_windows(case):
    """the deterministic fp16 tile backward: the fp16 window, exact sums, one fp16 rounding"""
    import ref64_det as D
    c = case
    la, k = c["la"], c["k"]
    t = la.taps
    exact = la._apply([m.T.tocsr() for m in T16.w_fp16(la)], c["g"], (t.Hs, t.Ws))
    E = np.asarray(D.la_exponents(c["g"], t.H, t.W, k), np.float64).reshape(-1, 1, 1, 1)
    bound = T16.bound_gs_tile16_det(c["r"]["gs"], c["r"]["Mgs"], c["Ags"], E, D.n_partials_la(t.H, t.W, k), U, ETA)
    assert ref64.assert_within("grad_source det fp16", T16.round_fp16(exact), c["r"]["gs"], bound) > 0.1


def test_bounds_reject_dropped_window_row(case):
    """a 16-pixel group row loses one source row of its window: group row y = 9, pixels x 16..31"""
    la, s = case["la"], case["s"]
    t = la.taps
    m = T16.w_fp16(la)[0].tolil()
    pix = 9 * t.W + np.arange(16, 32)
    y0 = int(t.pos[0, 0, 0, 0, pix[0]] // t.Ws) + 1
    for n in pix:
        for col in list(m.rows[n]):
            if col // t.Ws == y0:
                m[n, col] = 0
    _, msg = ref64.check("row_mask fp16", T16.tile_fwd16(la, s, [m.tocsr()]), case["out"], fwd_bound(case))
    assert msg is not None, "dropped window row not detected"


def test_bounds_reject_lost_add(case):
    """one group's grad_source adds for one step (16 positions of a source row in its footprint) are lost"""
    la = case["la"]
    col = int(la.W[0][T16.groups(la.taps)[7]].indices.min())
    gs = T16.tile_bwd_gs16(la, case["g"], np.random.default_rng(1), drop=(0, 7, col + np.arange(16)))
    _, msg = ref64.check("lost_step fp16", gs, case["r"]["gs"], gs_bound(case))
    assert msg is not None, "lost add not detected"
