"""GPU (-m gpu): the deterministic backward mode against the fp64 reference (ref64), element by element, with the bounds
of ref64_det.py, on the shapes and flows of test_gpu_lowp_bounds.py (local attention, block_extract) and
test_gpu_patch_conv.py (patch convolution).  Prints the largest |err|/bound per output and path."""
import numpy as np
import pytest
import torch

import ref64
import ref64_det as D
from test_gpu_lowp_bounds import CASES, case_id, host, make
from test_gpu_patch_conv import CASES as PC_CASES, case_id as pc_case_id, make as pc_make, reference as pc_reference

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
CL = torch.channels_last
WORST = {}


def within(row, y, ref, bound, **mags):
    r = ref64.assert_within(row, host(y) if torch.is_tensor(y) else y, ref, bound, **mags)
    WORST[row] = max(WORST.get(row, 0.0), r)


@pytest.fixture(scope="module", autouse=True)
def worst_ratios():
    yield
    print("\nlargest |err|/bound per output and path (deterministic mode):")
    for row in sorted(WORST):
        print(f"  {row:48s} {WORST[row]:.3f}")


@pytest.fixture(scope="module")
def G():
    import gfla_b200
    from gfla_b200 import _lib
    _lib.check(_lib.lib().gfla_device_check(), "device check")
    return gfla_b200


@pytest.fixture
def det():
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)


def _per_image(E, ndim):
    return np.asarray(E, np.float64).reshape((-1,) + (1,) * (ndim - 1))


def check_la(la, r, gs, gf, gl, C, row, gs_bound):
    u, eta = ref64.storage("bf16")
    within(f"grad_source {row}", gs, r["gs"], gs_bound, Mgs=r["Mgs"])
    within(f"grad_logits {row}", gl, r["gl"], ref64.bound_gl(r["gl"], la.probs(), r["D"], r["PD"], C, u, eta), D=r["D"],
           PD=r["PD"])
    within(f"grad_flow {row}", gf, r["gf"], ref64.bound_gf(r["gf"], r["Mgf"], C), Mgf=r["Mgf"])


@pytest.mark.parametrize("k", [3, 5])
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_tile_backward_det_bounds(G, det, case, k):
    F_ = G.functional
    (B, C, Hs, Ws, H, W), kind = case
    s, f, lg, g = make(B, C, Hs, Ws, H, W, k, kind, seed=3 * sum(case[0]) + k + len(kind))
    s, g = s.contiguous(memory_format=CL), g.contiguous(memory_format=CL)
    la = ref64.LocalAttn(host(f), host(lg), k, Hs, Ws)
    r = la.bwd(host(s), host(g))
    u, eta = ref64.storage("bf16")
    E = _per_image(D.la_exponents(host(g), H, W, k), 4)
    bound = D.bound_gs_tile(r["gs"], r["Mgs"], E, D.n_partials_la(H, W, k), u, eta)
    gs, gf, gl = F_.local_attn_bwd(s, f, lg, g, k, algo="tile")
    check_la(la, r, gs, gf, gl, C, "tile bwd det", bound)
    # today's bf16 bound for the same outputs: without the quantisation term (below 2^-40 of M_b), the deterministic bound
    # is tighter wherever a partial lands (the per-partial and per-add bf16 roundings are gone)
    old = ref64.bound_gs_tile(r["Mgs"], r["n_adds"][:, None], u, eta)
    rounding = D.bound_gs_tile(r["gs"], r["Mgs"], E, 0, u, eta)
    touched = r["Mgs"] > 0
    assert (rounding <= old)[touched].all()
    if kind in ("smooth", "span3"):
        gs, gf, gl = F_.local_attn_bwd(s.contiguous(), f, lg, g.contiguous(), k, algo="auto")
        assert gs.is_contiguous()
        check_la(la, r, gs, gf, gl, C, "tile bwd det nchw auto", bound)


# fp64 is not listed: ref64's taps and weights are fp32 arithmetic (ref64.Taps), which the fp64 kernel does not do; the
# fp64 path is checked by fp64 gradcheck and bit for bit in test_gpu_deterministic.py
@pytest.mark.parametrize("dt", ["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("k", [3, 4, 5])
def test_gather_backward_det_bounds(G, det, dt, k):
    F_ = G.functional
    B, C, Hs, Ws, H, W = 2, 48, 23, 29, 23, 29
    tdt = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}[dt]
    u, eta = (D.U_FP32, 0.0) if dt == "fp32" else ref64.storage(dt)
    for kind in ("smooth", "border", "irregular"):
        s, f, lg, g = make(B, C, Hs, Ws, H, W, k, kind, seed=7 * k + len(kind) + len(dt), dt="bf16")
        s, lg, g = s.to(tdt), lg.to(tdt), g.to(tdt)
        la = ref64.LocalAttn(host(f), host(lg), k, Hs, Ws)
        r = la.bwd(host(s), host(g))
        E = _per_image(D.la_exponents(host(g), H, W, k), 4)
        gs, gf, gl = F_.local_attn_bwd(s, f, lg, g, k, algo="gather")
        assert gs.dtype == s.dtype
        within(f"grad_source gather det {dt}", gs, r["gs"],
               D.bound_gs_gather(r["gs"], r["Mgs"], E, D.n_partials_la(H, W, k), u, eta), Mgs=r["Mgs"])


@pytest.mark.parametrize("flow_dt", ["fp32", "storage"])
@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_block_extract_det_bounds(G, det, dt, flow_dt):
    F_ = G.functional
    B, C, Hs, Ws, H, W, k = 2, 16, 13, 17, 11, 15, 3
    tdt = {"bf16": torch.bfloat16, "fp16": torch.float16}[dt]
    fdt = torch.float32 if flow_dt == "fp32" else tdt
    u, eta = ref64.storage(dt)
    for kind in ("smooth", "border"):
        s, f, _, _ = make(B, C, Hs, Ws, H, W, k, kind, seed=len(kind) + len(dt), dt=dt, flow_dt=fdt)
        g = torch.randn(B, C, k * H, k * W, device=DEV).to(tdt)
        r = ref64.block_extract(host(s), host(f), k, host(g))
        E = _per_image(D.be_exponents(host(g), k, H, W), 4)
        gs, gf = F_.block_extract_bwd(s, f, g, k)
        assert gs.dtype == s.dtype and gf.dtype == f.dtype
        within(f"block_extract grad_source det {dt}", gs, r["gs"], D.bound_be_gs(r["gs"], r["Mgs"], E, 4 * k * k * H * W, u, eta),
               Mgs=r["Mgs"])
        fu, feta = (0.0, 0.0) if flow_dt == "fp32" else (u, eta)
        within(f"block_extract grad_flow det {dt} flow {flow_dt}", gf, r["gf"],
               ref64.bound_be_gf(r["gf"], r["Mgf"], k * k * C, fu, feta), Mgf=r["Mgf"])


@pytest.mark.parametrize("case", PC_CASES, ids=pc_case_id)
def test_patch_conv_det_bounds(G, det, case):
    from test_patch_conv_ref import N_OUT, bound_gf
    (B, C, Hs, Ws, H, W), kind, k = case
    s, f, w, g = pc_make(B, C, Hs, Ws, H, W, k, kind, seed=C + H + k)
    r = pc_reference(G, s, f, w, g, k)
    u, eta = ref64.storage("bf16")
    Es, Ew = D.pc_exponents(host(g), host(w), host(s), k, H, W, N_OUT)
    gs, gf, gw = G.functional.patch_conv_bwd(s, f, w, g, k)
    within("patch_conv grad_source det", host(gs), r["gs"],
           D.bound_pc_gs(r["gs"], r["Mgs"], _per_image(Es, 4), 4 * k * k * H * W, N_OUT, u, eta), Mgs=r["Mgs"])
    within("patch_conv grad_flow det", host(gf), r["gf"], bound_gf(r["gf"], r["Mgf"], C, k), Mgf=r["Mgf"])
    ngroups = B * ((W + 15) // 16) * ((H + 7) // 8)
    per_slice = min(256, ngroups)            # PCW_DET_GROUPS groups of 128 pixels per fixed-point partial
    n_slices = (ngroups + per_slice - 1) // per_slice
    within("patch_conv grad_weight det", host(gw), r["gw"],
           D.bound_pc_gw(r["gw"], r["Mgw"], Ew, n_slices, 128 * per_slice, u, eta), Mgw=r["Mgw"])
