"""GPU (-m gpu): the tensor-core tile kernels in fp16 storage against the fp64 reference (ref64), element by element, with
the fp16 bounds of ref64_tile16 (a per-weight term for subnormal window weights), on the shapes and flows of
test_gpu_lowp_bounds.py; the kernels fp16 calls launch; an Inf in grad_out; and the deterministic fp16 tile backward
(repeats, per image, batch halves, SM count, within its bound).  Prints the largest |err|/bound per output and path."""
import numpy as np
import pytest
import torch

import ref64
import ref64_det as D
import ref64_tile16 as T16
from kernel_names import kernel_names
from test_gpu_deterministic import check_r1_r2, la_inputs, same
from test_gpu_lowp_bounds import CASES, case_id, host, make

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
CL = torch.channels_last
U, ETA = ref64.storage("fp16")
WORST = {}


def within(row, y, ref, bound, **mags):
    r = ref64.assert_within(row, host(y) if torch.is_tensor(y) else y, ref, bound, **mags)
    WORST[row] = max(WORST.get(row, 0.0), r)


@pytest.fixture(scope="module", autouse=True)
def worst_ratios():
    yield
    print("\nlargest |err|/bound per output and path (fp16 tile kernels):")
    for row in sorted(WORST):
        print(f"  {row:44s} {WORST[row]:.3f}")


@pytest.fixture(scope="module")
def F_():
    import gfla_b200
    from gfla_b200 import _lib
    _lib.check(_lib.lib().gfla_device_check(), "device check")
    return gfla_b200.functional


@pytest.fixture
def det():
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)


@pytest.mark.parametrize("k", [3, 5])
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_tile_forward_fp16(F_, case, k):
    (B, C, Hs, Ws, H, W), kind = case
    s, f, lg, _ = make(B, C, Hs, Ws, H, W, k, kind, seed=sum(case[0]) + k + len(kind), dt="fp16")
    la = ref64.LocalAttn(host(f), host(lg), k, Hs, Ws)
    r, M = la.fwd(host(s))
    A = T16.weight_mag_fwd(la, host(s))
    bound = T16.bound_out_tile16(r, M, A, U, ETA)
    for layout in ("nhwc", "nchw") if Ws % 8 == 0 else ("nhwc",):      # the planar tile kernel needs Ws % 8 == 0
        src = s.contiguous(memory_format=CL) if layout == "nhwc" else s
        out, probs = F_.local_attn_fwd(src, f, lg, k, return_probs=True, algo="tile")
        assert out.dtype == torch.float16 and probs.dtype == torch.float16
        within(f"out tile fwd fp16 {layout}", out, r, bound, M=M, A=A)
        within("probs tile fwd fp16", probs, la.probs(), ref64.bound_probs(la.probs(), U, ETA))
    if kind in ("smooth", "outside"):       # the fused blend, same kernel
        m = torch.rand(B, 1, H, W, device=DEV).half()
        prev = torch.randn(B, C, H, W, device=DEV).half().contiguous(memory_format=CL)
        out = F_.local_attn_blend_fwd(s.contiguous(memory_format=CL), f, lg, prev, m, k, algo="tile")
        rb, Mb = ref64.blend_ref(r, M, host(prev), host(m))
        within("out tile blend fp16", out, rb, T16.bound_out_tile16_blend(rb, Mb, M * host(m), A * host(m), U, ETA), M=Mb)


def check_bwd16(la, r, gs, gf, gl, C, row, gs_bound, init=(0.0, 0.0, 0.0)):
    assert gs.dtype == torch.float16 and gl.dtype == torch.float16 and gf.dtype == torch.float32
    within(f"grad_source {row}", gs, r["gs"] + init[0], gs_bound, Mgs=r["Mgs"], n_adds=r["n_adds"][:, None])
    within(f"grad_logits {row}", gl, r["gl"] + init[2],
           ref64.bound_gl(r["gl"] + init[2], la.probs(), r["D"], r["PD"], C, U, ETA, init=init[2]), D=r["D"], PD=r["PD"])
    within(f"grad_flow {row}", gf, r["gf"] + init[1], ref64.bound_gf(r["gf"] + init[1], r["Mgf"], C, init=init[1]),
           Mgf=r["Mgf"])


@pytest.mark.parametrize("k", [3, 5])
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_tile_backward_fp16(F_, case, k):
    """the default tile backward (NHWC, and planar callers through the re-layout), then the deterministic one on the same
    inputs and reference"""
    (B, C, Hs, Ws, H, W), kind = case
    s, f, lg, g = make(B, C, Hs, Ws, H, W, k, kind, seed=3 * sum(case[0]) + k + len(kind), dt="fp16")
    s, g = s.contiguous(memory_format=CL), g.contiguous(memory_format=CL)
    la = ref64.LocalAttn(host(f), host(lg), k, Hs, Ws)
    r = la.bwd(host(s), host(g))
    Ags = T16.weight_mag_gs(la, host(g))
    bound = T16.bound_gs_tile16(r["Mgs"], Ags, r["n_adds"][:, None], U, ETA)
    gs, gf, gl = F_.local_attn_bwd(s, f, lg, g, k, algo="tile")
    check_bwd16(la, r, gs, gf, gl, C, "tile bwd fp16", bound)
    if kind in ("smooth", "span3"):     # planar callers: relayout to channels-last, the tile kernel, relayout back
        gs, gf, gl = F_.local_attn_bwd(s.contiguous(), f, lg, g.contiguous(), k, algo="auto")
        assert gs.is_contiguous()
        check_bwd16(la, r, gs, gf, gl, C, "tile bwd fp16 nchw auto", bound)
    # deterministic mode: fixed-point sums of the fp16 window's partials, rounded once
    E = np.asarray(D.la_exponents(host(g), H, W, k), np.float64).reshape(-1, 1, 1, 1)
    det_bound = T16.bound_gs_tile16_det(r["gs"], r["Mgs"], Ags, E, D.n_partials_la(H, W, k), U, ETA)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        gs, gf, gl = F_.local_attn_bwd(s, f, lg, g, k, algo="tile")
    finally:
        torch.use_deterministic_algorithms(prev)
    check_bwd16(la, r, gs, gf, gl, C, "tile bwd fp16 det", det_bound)


@pytest.mark.parametrize("k", [3, 5])
@pytest.mark.parametrize("kind", ["halves", "span3", "irregular"])
def test_tile_backward_fp16_accumulate(F_, kind, k):
    """accumulate = 1 through the raw ABI: the gradients are added into what the buffers hold"""
    from gfla_b200 import _lib
    from gfla_b200.functional import ALGO, _dt, _p, _stream
    B, C, Hs, Ws, H, W = 1, 256, 19, 45, 19, 45
    s, f, lg, g = make(B, C, Hs, Ws, H, W, k, kind, seed=101 + k, dt="fp16")
    s, g = s.contiguous(memory_format=CL), g.contiguous(memory_format=CL)
    init = (0.5, -0.25, 0.125)
    gs = torch.full(s.shape, init[0], device=DEV, dtype=torch.float16).contiguous(memory_format=CL)
    gf = torch.full(f.shape, init[1], device=DEV, dtype=torch.float32)
    gl = torch.full(lg.shape, init[2], device=DEV, dtype=torch.float16)
    _lib.check(_lib.lib().gfla_local_attn_bwd(_p(s), _p(f), _p(lg), _p(g), _p(gs), _p(gf), _p(gl), B, C, Hs, Ws, H, W, k,
                                              _dt(s), _dt(f), _lib.GFLA_NHWC, 1, ALGO["tile"], _stream(s)), "local_attn_bwd")
    la = ref64.LocalAttn(host(f), host(lg), k, Hs, Ws)
    r = la.bwd(host(s), host(g))
    Ags = T16.weight_mag_gs(la, host(g))
    check_bwd16(la, r, gs, gf, gl, C, "tile bwd fp16 accumulate",
                T16.bound_gs_tile16(r["Mgs"], Ags, r["n_adds"][:, None], U, ETA, init=init[0]), init=init)


_FP16_INPUTS = """
from gfla_b200 import functional as F_
CL = torch.channels_last
s = torch.randn(2, 256, 32, 32, device="cuda").half()
f = torch.rand(2, 2, 32, 32, device="cuda") * 8 - 4
lg = torch.randn(2, 25, 32, 32, device="cuda").half()
g = torch.randn(2, 256, 32, 32, device="cuda").half()
sc, gc = s.contiguous(memory_format=CL), g.contiguous(memory_format=CL)
"""


def test_fp16_calls_launch_the_tile_kernels(F_, tmp_path):
    """algo="auto" on fp16: the planar and channels-last forward and the backward are the fp16 tile instances, never the
    CUDA-core gather kernels (profiled in a child process: kernel_names.py)"""
    names = kernel_names(_FP16_INPUTS + """
NAMES = profiled(lambda: (F_.local_attn_fwd(s, f, lg, 5), F_.local_attn_fwd(sc, f, lg, 5),
                          F_.local_attn_bwd(sc, f, lg, gc, 5), F_.local_attn_bwd(s, f, lg, g, 5)))
""", tmp_path)
    half = [n for n in names if "__half" in n]
    assert any("k_local_attn_fwd_tc<" in n for n in half), names
    assert any("k_local_attn_fwd_tc_cl<" in n for n in half), names
    assert any("k_local_attn_bwd_tc<" in n for n in half), names
    assert not [n for n in names if "gfla::k_local_attn_fwd<" in n or "gfla::k_local_attn_bwd<" in n], names


def test_inf_in_grad_out_reaches_grad_source(F_):
    """an Inf in one image's grad_out (what GradScaler watches for) leaves that image's grad_source not all finite and
    the other images' finite"""
    s, f, lg, g = make(3, 256, 16, 16, 16, 16, 5, "smooth", seed=2, dt="fp16")
    s, g = s.contiguous(memory_format=CL), g.contiguous(memory_format=CL)
    g[1, 7, 3, 4] = float("inf")
    gs, _, _ = F_.local_attn_bwd(s, f, lg, g, 5, algo="tile")
    assert not torch.isfinite(gs[1]).all()
    assert torch.isfinite(gs[0]).all() and torch.isfinite(gs[2]).all()


# ---------------------------------------------------------------------------------------------- deterministic mode
@pytest.mark.parametrize("cl", [True, False], ids=["nhwc", "nchw"])
@pytest.mark.parametrize("C", [64, 128, 256, 512])
@pytest.mark.parametrize("k", [3, 5])
def test_det_fp16_tile_backward_repeats_and_is_per_image(F_, det, k, C, cl):
    args = la_inputs(3, C, 21, 27, 19, 23, k, dtype=torch.float16, cl=cl, seed=k + C)
    check_r1_r2(lambda s, f, l, g: F_.local_attn_bwd(s, f, l, g, k), args, ((1, 1, 1, 1), (1, 1, 1)))


def test_det_fp16_runs_the_deterministic_tile_instance(F_, tmp_path):
    names = kernel_names(_FP16_INPUTS + """
torch.use_deterministic_algorithms(True)
NAMES = profiled(lambda: F_.local_attn_bwd(sc, f, lg, gc, 5))
""", tmp_path)
    assert [n for n in names if "k_local_attn_bwd_tc<5, 256, true, __half>" in n], names
    assert not [n for n in names if "gfla::k_local_attn_bwd<" in n], names


def test_det_fp16_full_size_batch_halves(F_, det):
    """cfg2 in fp16: the B=16 backward equals its two B=8 halves bit for bit"""
    s, f, l, g = la_inputs(16, 256, 256, 256, 256, 256, 5, dtype=torch.float16, seed=6)
    full = F_.local_attn_bwd(s, f, l, g, 5)
    for h in range(2):
        part = F_.local_attn_bwd(s[8 * h:8 * h + 8], f[8 * h:8 * h + 8], l[8 * h:8 * h + 8], g[8 * h:8 * h + 8], 5)
        for x, y in zip(full, part):
            assert same(x[8 * h:8 * h + 8], y)


_OTHER_SM_COUNT = r"""
import sys, torch
import gfla_b200
from gfla_b200 import functional as F_
torch.use_deterministic_algorithms(True)
gen = torch.Generator().manual_seed(12)
s = torch.randn(4, 128, 96, 96, generator=gen).to("cuda", torch.float16).contiguous(memory_format=torch.channels_last)
f = (torch.randn(4, 2, 96, 96, generator=gen) * 2).to("cuda")
lg = torch.randn(4, 25, 96, 96, generator=gen).to("cuda", torch.float16)
g = torch.randn(4, 128, 96, 96, generator=gen).to("cuda", torch.float16).contiguous(memory_format=torch.channels_last)
torch.save([t.cpu() for t in F_.local_attn_bwd(s, f, lg, g, 5)], sys.argv[1])
"""


def test_det_fp16_does_not_depend_on_the_sm_count(F_, tmp_path):
    import os
    import subprocess
    import sys
    from conftest import ROOT
    res = {}
    for n in ("114", "132", "66"):
        path = tmp_path / f"sm{n}.pt"
        subprocess.run([sys.executable, "-c", _OTHER_SM_COUNT, str(path)], cwd=ROOT, env=dict(os.environ, GFLA_SM_COUNT=n),
                       check=True)
        res[n] = torch.load(path)
    for n in ("132", "66"):
        for x, y in zip(res["114"], res[n]):
            assert same(x, y), n
