"""GPU (-m gpu): every 16-bit path of the fused local-attention op and of block_extractor against the fp64 reference
(ref64), element by element, with bounds derived from what each kernel rounds (DESIGN.md section 6).  Stricter than the
flat 1e-2 of the other tests: a kernel that drops a window row, a tap or an atomic add fails here even when the values
it gets wrong are small."""
import numpy as np
import pytest
import torch

import ref64
import ref64_gather
from test_ref64 import make_flow

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
TDT = {"bf16": torch.bfloat16, "fp16": torch.float16}
WORST = {}


def host(t):
    return np.ascontiguousarray(t.detach().double().cpu().numpy())


def within(row, y, ref, bound, **mags):
    r = ref64.assert_within(row, host(y) if torch.is_tensor(y) else y, ref, bound, **mags)
    WORST[row] = max(WORST.get(row, 0.0), r)


@pytest.fixture(scope="module", autouse=True)
def worst_ratios():
    yield
    print("\nlargest |err|/bound per output and path:")
    for row in sorted(WORST):
        print(f"  {row:40s} {WORST[row]:.3f}")


@pytest.fixture(scope="module")
def F_():
    import gfla_b200
    from gfla_b200 import _lib
    _lib.check(_lib.lib().gfla_device_check(), "device check")
    return gfla_b200.functional


def make(B, C, Hs, Ws, H, W, k, kind, seed, dt="bf16", flow_dt=torch.float32):
    rng = np.random.default_rng(seed)
    s = torch.from_numpy(rng.standard_normal((B, C, Hs, Ws)).astype(np.float32)).to(DEV).to(TDT[dt])
    f = torch.from_numpy(make_flow(kind, rng, B, H, W, k)).to(DEV).to(flow_dt)
    lg = torch.from_numpy((2 * rng.standard_normal((B, k * k, H, W))).astype(np.float32)).to(DEV).to(TDT[dt])
    g = torch.from_numpy(rng.standard_normal((B, C, H, W)).astype(np.float32)).to(DEV).to(TDT[dt])
    return s, f, lg, g


KINDS = ["smooth", "iid", "border", "zero", "int", "rows", "halves", "outside", "span3", "irregular"]
SHAPES = [                              # B, C, Hs, Ws, H, W; the flow kinds each shape runs with
    ((2, 64, 21, 37, 21, 37), KINDS),                                   # ragged H and W
    ((1, 128, 24, 40, 24, 40), KINDS),
    ((1, 256, 19, 48, 19, 48), KINDS),                                  # ragged H, planar-capable
    ((1, 512, 16, 32, 16, 32), KINDS),                                  # two 256-channel passes of the backward
    ((1, 64, 26, 40, 19, 27), KINDS),                                   # source larger than the flow field
    ((2, 64, 72, 136, 72, 136), ["smooth", "iid", "rows", "irregular"]),   # 162 groups: more than the H100's 132 SMs
]
CASES = [(shape, kind) for shape, kinds in SHAPES for kind in kinds]


def case_id(c):
    return "x".join(map(str, c[0])) + "-" + c[1]


@pytest.mark.parametrize("k", [3, 5])
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_tile_forward_bf16(F_, case, k):
    (B, C, Hs, Ws, H, W), kind = case
    s, f, lg, _ = make(B, C, Hs, Ws, H, W, k, kind, seed=sum(case[0]) + k + len(kind))
    la = ref64.LocalAttn(host(f), host(lg), k, Hs, Ws)
    r, M = la.fwd(host(s))
    u, eta = ref64.storage("bf16")
    bound = ref64.bound_out_tile(r, M, u, eta)
    for layout in ("nhwc", "nchw") if Ws % 8 == 0 else ("nhwc",):      # the planar tile kernel needs Ws % 8 == 0
        src = s.contiguous(memory_format=torch.channels_last) if layout == "nhwc" else s
        out, probs = F_.local_attn_fwd(src, f, lg, k, return_probs=True, algo="tile")
        within(f"out tile fwd {layout}", out, r, bound, M=M)
        within("probs tile fwd", probs, la.probs(), ref64.bound_probs(la.probs(), u, eta))
    if kind in ("smooth", "outside"):       # the fused blend, same kernel
        m = torch.rand(B, 1, H, W, device=DEV).bfloat16()
        prev = torch.randn(B, C, H, W, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)
        out = F_.local_attn_blend_fwd(s.contiguous(memory_format=torch.channels_last), f, lg, prev, m, k, algo="tile")
        rb, Mb = ref64.blend_ref(r, M, host(prev), host(m))
        within("out tile blend", out, rb, ref64.bound_out_tile_blend(rb, Mb, M * host(m), u, eta), M=Mb)


def check_bwd(la, r, gs, gf, gl, C, row, gs_bound, init=(0.0, 0.0, 0.0)):
    u, eta = ref64.storage("bf16")
    within(f"grad_source {row}", gs, r["gs"] + init[0], gs_bound, Mgs=r["Mgs"], n_adds=r["n_adds"][:, None])
    within(f"grad_logits {row}", gl, r["gl"] + init[2],
           ref64.bound_gl(r["gl"] + init[2], la.probs(), r["D"], r["PD"], C, u, eta, init=init[2]), D=r["D"], PD=r["PD"])
    within(f"grad_flow {row}", gf, r["gf"] + init[1], ref64.bound_gf(r["gf"] + init[1], r["Mgf"], C, init=init[1]),
           Mgf=r["Mgf"])


@pytest.mark.parametrize("k", [3, 5])
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_tile_backward_bf16(F_, case, k):
    (B, C, Hs, Ws, H, W), kind = case
    s, f, lg, g = make(B, C, Hs, Ws, H, W, k, kind, seed=3 * sum(case[0]) + k + len(kind))
    s, g = s.contiguous(memory_format=torch.channels_last), g.contiguous(memory_format=torch.channels_last)
    la = ref64.LocalAttn(host(f), host(lg), k, Hs, Ws)
    r = la.bwd(host(s), host(g))
    u, eta = ref64.storage("bf16")
    gs, gf, gl = F_.local_attn_bwd(s, f, lg, g, k, algo="tile")
    check_bwd(la, r, gs, gf, gl, C, "tile bwd", ref64.bound_gs_tile(r["Mgs"], r["n_adds"][:, None], u, eta))
    if kind in ("smooth", "span3"):     # planar callers: relayout to channels-last, the tile kernel, relayout back
        gs, gf, gl = F_.local_attn_bwd(s.contiguous(), f, lg, g.contiguous(), k, algo="auto")
        assert gs.is_contiguous()
        check_bwd(la, r, gs, gf, gl, C, "tile bwd nchw auto", ref64.bound_gs_tile(r["Mgs"], r["n_adds"][:, None], u, eta))


@pytest.mark.parametrize("k", [3, 5])
@pytest.mark.parametrize("kind", ["halves", "span3", "irregular"])
def test_tile_backward_bf16_accumulate(F_, kind, k):
    """accumulate = 1 through the raw ABI: the gradients are added into what the buffers hold"""
    from gfla_b200 import _lib
    from gfla_b200.functional import ALGO, _dt, _p, _stream
    B, C, Hs, Ws, H, W = 1, 256, 19, 45, 19, 45
    s, f, lg, g = make(B, C, Hs, Ws, H, W, k, kind, seed=101 + k)
    s, g = s.contiguous(memory_format=torch.channels_last), g.contiguous(memory_format=torch.channels_last)
    init = (0.5, -0.25, 0.125)
    gs = torch.full(s.shape, init[0], device=DEV, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
    gf = torch.full(f.shape, init[1], device=DEV, dtype=torch.float32)
    gl = torch.full(lg.shape, init[2], device=DEV, dtype=torch.bfloat16)
    _lib.check(_lib.lib().gfla_local_attn_bwd(_p(s), _p(f), _p(lg), _p(g), _p(gs), _p(gf), _p(gl), B, C, Hs, Ws, H, W, k,
                                              _dt(s), _dt(f), _lib.GFLA_NHWC, 1, ALGO["tile"], _stream(s)), "local_attn_bwd")
    la = ref64.LocalAttn(host(f), host(lg), k, Hs, Ws)
    r = la.bwd(host(s), host(g))
    u, eta = ref64.storage("bf16")
    check_bwd(la, r, gs, gf, gl, C, "tile bwd accumulate",
              ref64.bound_gs_tile(r["Mgs"], r["n_adds"][:, None], u, eta, init=init[0]), init=init)


@pytest.mark.parametrize("k", range(1, 10))
@pytest.mark.parametrize("flow_dt", ["fp32", "storage"])
@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_gather_16bit(F_, dt, flow_dt, k):
    """the CUDA-core kernels in 16-bit storage: the fp32 kernels' arithmetic on the widened values (their ref64_gather
    bound, which grows with k and C) and one rounding per output (the backward runs on fp32 copies); with an fp32 flow and
    with a flow in the storage dtype"""
    B, C, Hs, Ws, H, W = 2, 48, 23, 29, 23, 29
    fdt = torch.float32 if flow_dt == "fp32" else TDT[dt]
    u, eta = ref64.storage(dt)
    b = lambda y, e32: ref64.bound_gather16(y, e32, u, eta)
    for kind in ("smooth", "border", "irregular") if k > 1 else ("smooth", "border"):   # one tap: always regular
        s, f, lg, g = make(B, C, Hs, Ws, H, W, k, kind, seed=7 * k + len(kind) + len(dt), dt=dt, flow_dt=fdt)
        la = ref64_gather.LocalAttn(host(f), host(lg), k, Hs, Ws, np.float32)
        r, mags = la.fwd(host(s))
        out, probs = F_.local_attn_fwd(s, f, lg, k, return_probs=True, algo="gather")
        within(f"out gather {dt}", out, r, b(r, la.bound_out(mags)), M=mags["M"])
        within(f"probs gather {dt}", probs, la.probs(), b(la.probs(), la.bound_probs()))
        m = torch.rand(B, 1, H, W, device=DEV).to(TDT[dt])
        prev = torch.randn(B, C, H, W, device=DEV).to(TDT[dt])
        rb, Mb = ref64.blend_ref(r, mags["M"], host(prev), host(m))
        within(f"out gather blend {dt}", F_.local_attn_blend_fwd(s, f, lg, prev, m, k, algo="gather"), rb,
               b(rb, la.bound_blend(rb, mags, host(prev), host(m))), M=Mb)
        rr = la.bwd(host(s), host(g))
        gs, gf, gl = F_.local_attn_bwd(s, f, lg, g, k, algo="gather")
        assert gs.dtype == s.dtype and gf.dtype == f.dtype and gl.dtype == lg.dtype
        within(f"grad_source gather {dt}", gs, rr["gs"], b(rr["gs"], la.bound_gs(rr)), Mgs=rr["Mgs"])
        within(f"grad_logits gather {dt}", gl, rr["gl"], b(rr["gl"], la.bound_gl(rr, C)), D=rr["D"], PD=rr["PD"])
        fu, feta = (0.0, 0.0) if flow_dt == "fp32" else (u, eta)
        within(f"grad_flow gather {dt} flow {flow_dt}", gf, rr["gf"], ref64.bound_gather16(rr["gf"], la.bound_gf(rr, C), fu, feta),
               Mgf=rr["Mgf"])


@pytest.mark.parametrize("flow_dt", ["fp32", "storage"])
@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_block_extract_16bit(F_, dt, flow_dt):
    B, C, Hs, Ws, H, W, k = 2, 16, 13, 17, 11, 15, 3
    fdt = torch.float32 if flow_dt == "fp32" else TDT[dt]
    u, eta = ref64.storage(dt)
    for kind in ("smooth", "border"):
        s, f, _, _ = make(B, C, Hs, Ws, H, W, k, kind, seed=len(kind) + len(dt), dt=dt, flow_dt=fdt)
        g = torch.randn(B, C, k * H, k * W, device=DEV).to(TDT[dt])
        be = ref64_gather.BlockExtract(host(s), host(f), k, host(g), np.float32)
        r = be.r
        out = F_.block_extract_fwd(s, f, k)
        within(f"block_extract fwd {dt}", out, r["out"], ref64.bound_gather16(r["out"], be.bound_out(), u, eta), M=r["M"])
        gs, gf = F_.block_extract_bwd(s, f, g, k)
        assert gs.dtype == s.dtype and gf.dtype == f.dtype
        within(f"block_extract grad_source {dt}", gs, r["gs"], ref64.bound_gather16(r["gs"], be.bound_gs(), u, eta),
               Mgs=r["Mgs"])
        fu, feta = (0.0, 0.0) if flow_dt == "fp32" else (u, eta)
        within(f"block_extract grad_flow {dt} flow {flow_dt}", gf, r["gf"],
               ref64.bound_gather16(r["gf"], be.bound_gf(), fu, feta), Mgf=r["Mgf"])
