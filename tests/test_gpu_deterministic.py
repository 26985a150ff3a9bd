"""GPU (-m gpu): the backward passes under torch.use_deterministic_algorithms(True) (csrc/det_accum.cuh).

  * R1: two calls give bitwise-equal outputs (compared as integer views of the storage) for the tile backward (NHWC and
    the NCHW route), the gather backward in every dtype, block_extract, patch_conv and accumulate=1 through the ABI;
  * R2: every per-image output of bwd(x)[b] equals bwd(x[b:b+1])[0] and bwd(x.flip(0))[B-1-b], bit for bit;
  * the results agree with the default (flag off) path; a non-finite grad_out makes only its own image NaN;
  * the deterministic kernel instances are what runs under the flag; resample2d raises (warns with warn_only);
  * ExtractorAttn's gradients repeat bit for bit, and BlockExtractor / LocalAttnFunction pass fp64 gradcheck.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
CL = torch.channels_last


@pytest.fixture(scope="module")
def G():
    import gfla_b200
    from gfla_b200 import _lib
    _lib.check(_lib.lib().gfla_device_check(), "device check")
    return gfla_b200


@pytest.fixture
def det():
    """deterministic mode on for the test; the previous setting (and warn_only) restored whatever happens"""
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)


_INT = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}


def bits(t):
    t = t.detach()
    return t.contiguous(memory_format=CL if t.dim() == 4 and not t.is_contiguous() else torch.contiguous_format).view(
        _INT[t.element_size()])


def same(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def la_inputs(B, C, Hs, Ws, H, W, k, dtype=torch.bfloat16, flow_dtype=torch.float32, cl=True, seed=0, flow="smooth"):
    g = torch.Generator(device="cpu").manual_seed(seed)
    s = torch.randn(B, C, Hs, Ws, generator=g)
    if flow == "smooth":
        f = torch.randn(B, 2, H, W, generator=g) * 3.0
    elif flow == "corner":            # every window folded onto the top-left corner
        f = torch.full((B, 2, H, W), -1e4)
    else:                             # irregular taps: fractions that straddle an integer after rounding
        f = torch.randn(B, 2, H, W, generator=g) * 2.0 + 1e-7
    lg = torch.randn(B, k * k, H, W, generator=g)
    go = torch.randn(B, C, H, W, generator=g)
    fmt = CL if cl else torch.contiguous_format
    return (s.to(DEV, dtype).contiguous(memory_format=fmt), f.to(DEV, flow_dtype), lg.to(DEV, dtype),
            go.to(DEV, dtype).contiguous(memory_format=fmt))


def check_r1_r2(fn, args, per_image):
    """fn(*args) -> tuple of outputs; per_image: which of the args / outputs have a batch axis"""
    a = fn(*args)
    b = fn(*args)
    for x, y in zip(a, b):
        assert same(x, y)
    B = args[0].shape[0]
    flip = fn(*[t.flip(0).contiguous(memory_format=CL if t.dim() == 4 and not t.is_contiguous() else torch.contiguous_format)
                if pi else t for t, pi in zip(args, per_image[0])])
    for i in (0, B - 1):
        one = fn(*[t[i:i + 1] if pi else t for t, pi in zip(args, per_image[0])])
        for o, (x, xo, xf) in enumerate(zip(a, one, flip)):
            if per_image[1][o]:
                assert same(x[i:i + 1], xo), (o, i)
                assert same(x[i], xf[B - 1 - i]), (o, i)
    return a


# ---------------------------------------------------------------------------------------------- local attention
@pytest.mark.parametrize("cl", [True, False], ids=["nhwc", "nchw"])
@pytest.mark.parametrize("C", [64, 128, 256, 512])
@pytest.mark.parametrize("k", [3, 5])
def test_tile_backward_repeats_and_is_per_image(G, det, k, C, cl):
    F_ = G.functional
    args = la_inputs(3, C, 21, 27, 19, 23, k, cl=cl, seed=k + C)
    gs, gf, gl = check_r1_r2(lambda s, f, l, g: F_.local_attn_bwd(s, f, l, g, k), args, ((1, 1, 1, 1), (1, 1, 1)))
    torch.use_deterministic_algorithms(False)
    rs, rf, rl = F_.local_attn_bwd(*args, k)
    # the default path rounds every partial to bf16: agree within a few bf16 ulps of the gradient's scale
    scale = rs.float().abs().amax()
    assert (gs.float() - rs.float()).abs().max() <= 2 ** -6 * scale
    assert torch.equal(gf, rf) and torch.equal(gl, rl)


@pytest.mark.parametrize("flow", ["corner", "irregular"])
def test_tile_backward_pileup_and_irregular_flows_are_per_image(G, det, flow):
    F_ = G.functional
    args = la_inputs(3, 256, 24, 40, 24, 40, 5, seed=3, flow=flow)
    check_r1_r2(lambda s, f, l, g: F_.local_attn_bwd(s, f, l, g, 5, algo="tile"), args, ((1, 1, 1, 1), (1, 1, 1)))


def test_tile_backward_more_groups_than_sms(G, det):
    F_ = G.functional
    args = la_inputs(2, 64, 150, 130, 147, 133, 3, seed=9)
    check_r1_r2(lambda s, f, l, g: F_.local_attn_bwd(s, f, l, g, 3), args, ((1, 1, 1, 1), (1, 1, 1)))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("k", [3, 4])
def test_gather_backward_repeats_and_is_per_image(G, det, k, dtype):
    F_ = G.functional
    fdt = torch.float64 if dtype == torch.float64 else torch.float32
    args = la_inputs(3, 24, 13, 17, 11, 15, k, dtype=dtype, flow_dtype=fdt, cl=False, seed=k)
    gs, gf, gl = check_r1_r2(lambda s, f, l, g: F_.local_attn_bwd(s, f, l, g, k, algo="gather"), args, ((1, 1, 1, 1), (1, 1, 1)))
    torch.use_deterministic_algorithms(False)
    ref = F_.local_attn_bwd(*[t.double() for t in args], k, algo="gather")[0]
    tol = {torch.float64: 1e-12, torch.float32: 1e-5, torch.bfloat16: 2 ** -7, torch.float16: 2 ** -10}[dtype]
    assert (gs.double() - ref).abs().max() <= tol * ref.abs().amax() + 1e-30


def test_accumulate_through_the_abi(G, det):
    from gfla_b200 import _lib
    F_ = G.functional
    s, f, l, g = la_inputs(2, 64, 16, 16, 16, 16, 5, seed=4)
    base = [torch.randn(s.shape, device=DEV).bfloat16().contiguous(memory_format=CL), torch.randn_like(f),
            torch.randn_like(l)]
    B, C, Hs, Ws = s.shape
    nb = _lib.lib().gfla_local_attn_bwd_det_workspace_bytes(B, C, Hs, Ws, 16, 16, 5)
    outs = []
    for _ in range(2):
        gs, gf, gl = [t.clone() for t in base]
        ws = torch.empty(nb, dtype=torch.uint8, device=DEV)
        _lib.check(_lib.lib().gfla_local_attn_bwd_det(*[t.data_ptr() for t in (s, f, l, g, gs, gf, gl)], B, C, Hs, Ws, 16, 16, 5,
                                                      _lib.GFLA_BF16, _lib.GFLA_F32, _lib.GFLA_NHWC, 1, 0, ws.data_ptr(), nb,
                                                      torch.cuda.current_stream().cuda_stream), "det")
        outs.append((gs, gf, gl))
    for x, y in zip(*outs):
        assert same(x, y)
    d = F_.local_attn_bwd(s, f, l, g, 5)
    assert torch.allclose(outs[0][0].float(), base[0].float() + d[0].float(), rtol=2 ** -7, atol=2 ** -7)


def test_non_finite_grad_out_poisons_only_its_image(G, det):
    F_ = G.functional
    s, f, l, g = la_inputs(3, 256, 16, 16, 16, 16, 5, seed=5)
    clean = F_.local_attn_bwd(s, f, l, g, 5)
    g2 = g.clone()
    g2[1, 7, 3, 4] = float("inf")
    gs, _, _ = F_.local_attn_bwd(s, f, l, g2, 5)
    assert torch.isnan(gs[1]).all()
    assert same(gs[0], clean[0][0]) and same(gs[2], clean[0][2])
    z = torch.zeros_like(g)
    assert (F_.local_attn_bwd(s, f, l, z, 5)[0] == 0).all()


def test_full_size_batch_halves(G, det):
    """cfg2: the B=16 backward equals the two B=8 halves bit for bit (the batch-sharding property)"""
    F_ = G.functional
    s, f, l, g = la_inputs(16, 256, 256, 256, 256, 256, 5, seed=6)
    full = F_.local_attn_bwd(s, f, l, g, 5)
    for h in range(2):
        part = F_.local_attn_bwd(s[8 * h:8 * h + 8], f[8 * h:8 * h + 8], l[8 * h:8 * h + 8], g[8 * h:8 * h + 8], 5)
        for x, y in zip(full, part):
            assert same(x[8 * h:8 * h + 8], y)


# ---------------------------------------------------------------------------------------------- block_extract, patch_conv
@pytest.mark.parametrize("dtype,flow_dtype", [(torch.float32, torch.float32), (torch.bfloat16, torch.float32),
                                              (torch.bfloat16, torch.bfloat16), (torch.float16, torch.float16)])
def test_block_extract_backward_repeats_and_is_per_image(G, det, dtype, flow_dtype):
    F_ = G.functional
    gen = torch.Generator().manual_seed(1)
    B, C, Hs, Ws, Hf, Wf, k = 3, 40, 14, 10, 9, 11, 3
    s = torch.randn(B, C, Hs, Ws, generator=gen).to(DEV, dtype)
    f = (torch.randn(B, 2, Hf, Wf, generator=gen) * 2).to(DEV, flow_dtype)
    g = torch.randn(B, C, k * Hf, k * Wf, generator=gen).to(DEV, dtype)
    gs, gf = check_r1_r2(lambda s_, f_, g_: F_.block_extract_bwd(s_, f_, g_, k), (s, f, g), ((1, 1, 1), (1, 1)))
    torch.use_deterministic_algorithms(False)
    rs, rf = F_.block_extract_bwd(s, f, g, k)
    assert torch.allclose(gs.float(), rs.float(), rtol=2 ** -6, atol=2 ** -6 * rs.float().abs().max().item())
    assert torch.allclose(gf.float(), rf.float(), rtol=2 ** -6, atol=2 ** -6 * rf.float().abs().max().item())


def test_patch_conv_backward_repeats_and_is_per_image(G, det):
    F_ = G.functional
    gen = torch.Generator().manual_seed(2)
    B, C, Hs, Ws, H, W, k = 3, 128, 13, 21, 11, 19, 5
    s = torch.randn(B, C, Hs, Ws, generator=gen).to(DEV, torch.bfloat16).contiguous(memory_format=CL)
    f = (torch.randn(B, 2, H, W, generator=gen) * 2).to(DEV)
    w = (torch.randn(128, C, k, k, generator=gen) / 40).to(DEV, torch.bfloat16)
    g = torch.randn(B, 128, H, W, generator=gen).to(DEV, torch.bfloat16).contiguous(memory_format=CL)
    gs, gf, gw = check_r1_r2(lambda s_, f_, g_: F_.patch_conv_bwd(s_, f_, w, g_, k), (s, f, g), ((1, 1, 1), (1, 1, 0)))
    torch.use_deterministic_algorithms(False)
    rs, rf, rw = F_.patch_conv_bwd(s, f, w, g, k)
    # grad_flow is written once per pixel on both paths, but the two kernel instances may contract differently
    assert torch.allclose(gf, rf, rtol=1e-5, atol=1e-5 * rf.abs().max().item())
    for x, y in ((gs, rs), (gw, rw)):
        assert (x.float() - y.float()).abs().max() <= 2 ** -7 * y.float().abs().max()


# ---------------------------------------------------------------------------------------------- routing
def _kernel_names(fn, witness, tries=3):
    """kernel names of one profiled call of fn, from the first of up to `tries` sessions that recorded this library's
    kernels at all (witness): a profiler session late in a long test process can miss them and is then repeated"""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(tries):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = [e.key for e in prof.key_averages()]
        if any(witness in n for n in names):
            break
    return names


def test_flag_selects_the_deterministic_instances(G):
    F_ = G.functional
    args = la_inputs(2, 256, 32, 32, 32, 32, 5, seed=7)
    prev = torch.are_deterministic_algorithms_enabled()
    try:
        torch.use_deterministic_algorithms(True)
        on = _kernel_names(lambda: F_.local_attn_bwd(*args, 5), "k_local_attn_bwd_tc")
        torch.use_deterministic_algorithms(False)
        off = _kernel_names(lambda: F_.local_attn_bwd(*args, 5), "k_local_attn_bwd_tc")
    finally:
        torch.use_deterministic_algorithms(prev)
    tile = lambda names, d: [n for n in names if "k_local_attn_bwd_tc<5, 256, " + d in n]
    assert tile(on, "true") and not tile(on, "false"), on
    assert any("k_fx_narrow" in n for n in on) and not any("k_fold_border" in n for n in on)
    assert tile(off, "false") and not tile(off, "true") and any("k_fold_border" in n for n in off), off
    assert not any("k_fx_" in n for n in off)


def _routing_cases(G):
    F_ = G.functional
    gen = torch.Generator().manual_seed(3)
    s32 = torch.randn(2, 16, 12, 12, generator=gen).to(DEV)
    f32 = (torch.randn(2, 2, 12, 12, generator=gen) * 2).to(DEV)
    l32 = torch.randn(2, 9, 12, 12, generator=gen).to(DEV)
    g32 = torch.randn(2, 16, 12, 12, generator=gen).to(DEV)
    gbe = torch.randn(2, 16, 36, 36, generator=gen).to(DEV)
    sp = torch.randn(2, 128, 16, 16, generator=gen).to(DEV, torch.bfloat16).contiguous(memory_format=CL)
    fp = (torch.randn(2, 2, 16, 16, generator=gen) * 2).to(DEV)
    wp = (torch.randn(128, 128, 3, 3, generator=gen) / 30).to(DEV, torch.bfloat16)
    gp = torch.randn(2, 128, 16, 16, generator=gen).to(DEV, torch.bfloat16).contiguous(memory_format=CL)
    return {
        "k_local_attn_bwd<": lambda: F_.local_attn_bwd(s32, f32, l32, g32, 3, algo="gather"),
        "k_block_extract_bwd<": lambda: F_.block_extract_bwd(s32, f32, gbe, 3),
        "k_patch_conv_bwd_tc<": lambda: F_.patch_conv_bwd(sp, fp, wp, gp, 3),
        "k_patch_conv_wgrad_tc<": lambda: F_.patch_conv_bwd(sp, fp, wp, gp, 3),
    }


@pytest.mark.parametrize("kern", ["k_local_attn_bwd<", "k_block_extract_bwd<", "k_patch_conv_bwd_tc<", "k_patch_conv_wgrad_tc<"])
def test_flag_selects_the_deterministic_instances_of_every_path(G, kern):
    fn = _routing_cases(G)[kern]
    prev = torch.are_deterministic_algorithms_enabled()
    try:
        torch.use_deterministic_algorithms(True)
        on = [n for n in _kernel_names(fn, kern) if kern in n]
        torch.use_deterministic_algorithms(False)
        off = [n for n in _kernel_names(fn, kern) if kern in n]
    finally:
        torch.use_deterministic_algorithms(prev)
    assert on and all("true>" in n for n in on), on
    assert off and all("false>" in n for n in off), off


_OTHER_SM_COUNT = r"""
import sys, torch
import gfla_b200
from gfla_b200 import functional as F_
torch.use_deterministic_algorithms(True)
gen = torch.Generator().manual_seed(11)
out = {}
s = torch.randn(4, 128, 128, 128, generator=gen).to("cuda", torch.bfloat16).contiguous(memory_format=torch.channels_last)
f = (torch.randn(4, 2, 128, 128, generator=gen) * 2).to("cuda")
w = (torch.randn(128, 128, 5, 5, generator=gen) / 80).to("cuda", torch.bfloat16)
g = torch.randn(4, 128, 128, 128, generator=gen).to("cuda", torch.bfloat16).contiguous(memory_format=torch.channels_last)
out["pc"] = [t.cpu() for t in F_.patch_conv_bwd(s, f, w, g, 5)]
sb = torch.randn(4, 64, 40, 40, generator=gen).to("cuda")
fb = (torch.randn(4, 2, 40, 40, generator=gen) * 2).to("cuda")
gb = torch.randn(4, 64, 120, 120, generator=gen).to("cuda")
out["be"] = [t.cpu() for t in F_.block_extract_bwd(sb, fb, gb, 3)]
lg = torch.randn(4, 25, 128, 128, generator=gen).to("cuda", torch.bfloat16)
out["la"] = [t.cpu() for t in F_.local_attn_bwd(s, f, lg, g, 5)]
torch.save(out, sys.argv[1])
"""


def test_results_do_not_depend_on_the_sm_count(G, tmp_path):
    """GFLA_SM_COUNT gives the launch heuristics another H100 variant's SM count (the patch convolution's weight-gradient
    slices and block_extract's channel slices follow it in the default mode): the deterministic results stay the same"""
    import os
    import subprocess
    import sys
    from conftest import ROOT
    res = {}
    for n in ("114", "132", "66"):
        path = tmp_path / f"sm{n}.pt"
        env = dict(os.environ, GFLA_SM_COUNT=n)
        subprocess.run([sys.executable, "-c", _OTHER_SM_COUNT, str(path)], cwd=ROOT, env=env, check=True)
        res[n] = torch.load(path)
    for n in ("132", "66"):
        for key in res["114"]:
            for x, y in zip(res["114"][key], res[n][key]):
                assert same(x, y), (n, key)


def test_resample2d_backward_raises_or_warns(G, det):
    gen = torch.Generator().manual_seed(0)
    x = torch.randn(1, 3, 8, 8, generator=gen).to(DEV).requires_grad_()
    fl = torch.randn(1, 2, 8, 8, generator=gen).to(DEV)
    out = G.Resample2d(4, 1)(x, fl)
    with pytest.raises(RuntimeError, match="does not have a deterministic implementation"):
        out.sum().backward()
    torch.use_deterministic_algorithms(True, warn_only=True)
    out = G.Resample2d(4, 1)(x, fl)
    with pytest.warns(UserWarning, match="does not have a deterministic implementation"):
        out.sum().backward()


# ---------------------------------------------------------------------------------------------- modules
def test_extractor_attn_gradients_repeat(G, det):
    from gfla_b200.extractor_attn import ExtractorAttn
    torch.manual_seed(0)
    m = ExtractorAttn(256, 5, softmax=True).to(DEV).to(torch.bfloat16).to(memory_format=CL)
    gen = torch.Generator().manual_seed(1)
    src = torch.randn(2, 256, 24, 24, generator=gen).to(DEV, torch.bfloat16).contiguous(memory_format=CL)
    tgt = torch.randn(2, 256, 24, 24, generator=gen).to(DEV, torch.bfloat16).contiguous(memory_format=CL)
    flow = (torch.randn(2, 2, 24, 24, generator=gen) * 2).to(DEV)

    def run():
        xs = [t.clone().requires_grad_() for t in (src, tgt, flow)]
        m.zero_grad(set_to_none=True)
        m(*xs).float().square().sum().backward()
        return [x.grad for x in xs] + [p.grad for p in m.parameters()]

    a, b = run(), run()
    for x, y in zip(a, b):
        assert same(x, y)
    torch.use_deterministic_algorithms(False)
    c = run()
    for x, y in zip(a, c):
        assert torch.allclose(x.float(), y.float(), rtol=5e-2, atol=5e-2 * y.float().abs().max().item())


def test_gradcheck_under_the_flag(G, det):
    from gfla_b200.extractor_attn import LocalAttnFunction
    torch.manual_seed(0)
    s = torch.rand(4, 6, 14, 10, dtype=torch.float64, device=DEV, requires_grad=True)
    f = (torch.rand(4, 2, 14, 10, dtype=torch.float64, device=DEV) * 1.8).requires_grad_()
    assert torch.autograd.gradcheck(lambda a, b: G.BlockExtractor(3)(a, b), (s, f), eps=1e-6, atol=1e-5)
    lg = torch.rand(4, 9, 14, 10, dtype=torch.float64, device=DEV, requires_grad=True)
    assert torch.autograd.gradcheck(lambda a, b, c: LocalAttnFunction.apply(a, b, c, 3), (s, f, lg), eps=1e-6, atol=1e-5)
