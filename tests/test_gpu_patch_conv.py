"""GPU (-m gpu): the patch-convolution kernels (csrc/patch_conv_tc.cu) behind gfla_b200.patch_conv and ExtractorAttn's
source-half conv, against the fp64 reference of tests/test_patch_conv_ref.py, element by element:

  * the gathered operand is bit-identical to block_extract_fwd's bf16 block tensor;
  * forward, grad_source, grad_flow and grad_weight lie within their rounding bounds over ragged shapes, C = 64..512,
    source sizes other than the flow's, more pixel groups than SMs and every flow kind; grad_flow is deterministic;
  * planar callers get what channels-last callers get; calls the kernels do not serve get the literal composition;
  * ExtractorAttn in bf16 channels-last runs the new kernels and no block_extract kernel, and one patch_conv
    forward+backward needs a fraction of one block tensor in transient memory.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import ref64
from test_patch_conv_ref import N_OUT, bound_gf, bound_gs, bound_gw, bound_out, conv_blocks, patch_ref
from test_ref64 import FLOWS, make_flow

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
CL = torch.channels_last
KINDS = ["smooth", "iid", "border", "zero", "int", "rows", "halves", "outside", "span3", "irregular"]


def host(t):
    return np.ascontiguousarray(t.detach().double().cpu().numpy())


@pytest.fixture(scope="module")
def G():
    import gfla_b200
    from gfla_b200 import _lib
    _lib.check(_lib.lib().gfla_device_check(), "device check")
    return gfla_b200


def make(B, C, Hs, Ws, H, W, k, kind, seed, n=N_OUT):
    rng = np.random.default_rng(seed)
    s = torch.from_numpy(rng.standard_normal((B, C, Hs, Ws)).astype(np.float32)).to(DEV).bfloat16().contiguous(memory_format=CL)
    f = torch.from_numpy(make_flow(kind, rng, B, H, W, k)).to(DEV)
    w = torch.from_numpy((rng.standard_normal((n, C, k, k)) / np.sqrt(C * k * k)).astype(np.float32)).to(DEV).bfloat16()
    g = torch.from_numpy(rng.standard_normal((B, n, H, W)).astype(np.float32)).to(DEV).bfloat16().contiguous(memory_format=CL)
    return s, f, w, g


# --------------------------------------------------------------------------------------------- 1. gathered operand
@pytest.mark.parametrize("kind", FLOWS)
@pytest.mark.parametrize("k", [3, 4, 5])
def test_gathered_operand_is_bit_identical_to_block_extract(G, k, kind):
    """a weight whose rows are one-hots over 128 distinct (tap, channel) pairs, covering every tap and both 64-channel
    chunks, makes out[:, n] the block tensor at that tap and channel, bit for bit"""
    B, C, Hs, Ws, H, W = 2, 128, 13, 21, 11, 19
    s, f, _, _ = make(B, C, Hs, Ws, H, W, k, kind, seed=k)
    kk = k * k
    taps = [n % kk for n in range(N_OUT)]
    chans = [((n // kk) % 2) * 64 + 3 * (n // kk) + (n % kk) % 5 for n in range(N_OUT)]
    assert len(set(zip(taps, chans))) == N_OUT and set(taps) == set(range(kk)) and {c // 64 for c in chans} == {0, 1}
    w = torch.zeros(N_OUT, C, k, k, device=DEV, dtype=torch.bfloat16)
    for n, (t, c) in enumerate(zip(taps, chans)):
        w[n, c, t // k, t % k] = 1.0
    out = G.functional.patch_conv_fwd(s, f, w, k)
    blk = G.functional.block_extract_fwd(s.contiguous(), f, k).view(B, C, H, k, W, k)
    want = torch.stack([blk[:, c, :, t // k, :, t % k] for t, c in zip(taps, chans)], 1)
    assert torch.equal(out.contiguous().view(torch.int16), want.contiguous().view(torch.int16))


# ------------------------------------------------------------------------------------------ 2./3. forward, backward
SHAPES = [                              # B, C, Hs, Ws, H, W; the flow kinds each shape runs with; the k values
    ((2, 64, 21, 37, 21, 37), KINDS, (3, 5)),                           # ragged H and W
    ((1, 128, 24, 40, 24, 40), KINDS, (3, 4, 5)),
    ((1, 256, 19, 48, 19, 48), ["smooth", "iid", "border", "outside"], (3, 5)),
    ((1, 512, 16, 32, 16, 32), ["smooth", "irregular"], (3,)),
    ((1, 64, 26, 40, 19, 27), KINDS, (3, 5)),                           # source larger than the flow field
    ((2, 64, 72, 136, 72, 136), ["smooth", "iid"], (3,)),               # 162 pixel groups: more than the H100's 132 SMs
]
CASES = [(shape, kind, k) for shape, kinds, ks in SHAPES for kind in kinds for k in ks]


def case_id(c):
    return "x".join(map(str, c[0])) + f"-{c[1]}-k{c[2]}"


def reference(G, s, f, w, g, k):
    blk = G.functional.block_extract_fwd(s.contiguous(), f, k)          # bf16: the operand the kernels gather
    return patch_ref(host(s), host(f).astype(np.float32), host(w), k, None if g is None else host(g), block=host(blk))


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_forward_and_backward_within_bounds(G, case):
    (B, C, Hs, Ws, H, W), kind, k = case
    s, f, w, g = make(B, C, Hs, Ws, H, W, k, kind, seed=C + H + k)
    r = reference(G, s, f, w, g, k)
    out = G.functional.patch_conv_fwd(s, f, w, k)
    assert out.is_contiguous(memory_format=CL)
    ref64.assert_within("out", host(out), r["out"], bound_out(r["out"], r["M"], C, k), M=r["M"])
    gs, gf, gw = G.functional.patch_conv_bwd(s, f, w, g, k)
    ref64.assert_within("grad_source", host(gs), r["gs"], bound_gs(r["gs"], r["Mgs"], r["n"]), Mgs=r["Mgs"])
    ref64.assert_within("grad_flow", host(gf), r["gf"], bound_gf(r["gf"], r["Mgf"], C, k), Mgf=r["Mgf"])
    ref64.assert_within("grad_weight", host(gw), r["gw"], bound_gw(r["gw"], r["Mgw"], B * H * W), Mgw=r["Mgw"])
    _, gf2, _ = G.functional.patch_conv_bwd(s, f, w, g, k)
    assert torch.equal(gf, gf2)                     # grad_flow is written once per pixel, without atomics


@pytest.mark.parametrize("kind", ["smooth", "iid", "border", "outside"])
def test_backward_accumulates_through_the_abi(G, kind):
    """accumulate = 1 adds all three gradients into the caller's fp32 buffers"""
    from gfla_b200 import _lib
    B, C, Hs, Ws, H, W, k = 2, 128, 21, 37, 17, 29, 3
    s, f, w, g = make(B, C, Hs, Ws, H, W, k, kind, seed=5)
    r = reference(G, s, f, w, g, k)
    gs0 = torch.randn(B, Hs, Ws, C, device=DEV)
    gf0 = torch.randn(B, 2, H, W, device=DEV)
    gw0 = torch.randn(N_OUT, k, k, C, device=DEV)
    gs, gf, gw = gs0.clone(), gf0.clone(), gw0.clone()
    wp = w.permute(0, 2, 3, 1).contiguous()
    st = torch.cuda.current_stream().cuda_stream
    _lib.check(_lib.lib().gfla_patch_conv_bwd(s.data_ptr(), f.data_ptr(), wp.data_ptr(), g.data_ptr(), gs.data_ptr(), gf.data_ptr(),
                                              gw.data_ptr(), B, C, Hs, Ws, H, W, k, N_OUT, _lib.GFLA_BF16, _lib.GFLA_F32,
                                              _lib.GFLA_NHWC, 1, st), "patch_conv_bwd")
    i_s, i_w = host(gs0.permute(0, 3, 1, 2)), host(gw0.permute(0, 3, 1, 2))
    ref64.assert_within("grad_source (acc)", host(gs.permute(0, 3, 1, 2)), r["gs"] + i_s,
                        bound_gs(r["gs"], r["Mgs"], r["n"], u=0.0, eta=0.0, init=i_s))
    ref64.assert_within("grad_flow (acc)", host(gf), r["gf"] + host(gf0), bound_gf(r["gf"], r["Mgf"], C, k, init=host(gf0)))
    ref64.assert_within("grad_weight (acc)", host(gw.permute(0, 3, 1, 2)), r["gw"] + i_w,
                        bound_gw(r["gw"], r["Mgw"], B * H * W, u=0.0, eta=0.0, init=i_w))


# --------------------------------------------------------------------------------------------------- 4. layouts
@pytest.mark.parametrize("k", [3, 4])
def test_planar_caller_matches_channels_last(G, k):
    s, f, w, g = make(2, 128, 20, 30, 18, 27, k, "smooth", seed=9)
    sp = s.contiguous()
    out_cl = G.patch_conv(s, f, w, k)
    out_p = G.patch_conv(sp, f, w, k)
    assert out_p.is_contiguous() and out_cl.is_contiguous(memory_format=CL)
    assert torch.equal(out_p, out_cl)
    grads = []
    for src, go in ((s, g), (sp, g.contiguous())):
        src = src.detach().requires_grad_()
        fl, wt = f.clone().requires_grad_(), w.clone().requires_grad_()
        G.patch_conv(src, fl, wt, k).backward(go)
        grads.append((src.grad, fl.grad, wt.grad))
    (gs_cl, gf_cl, gw_cl), (gs_p, gf_p, gw_p) = grads
    assert gs_p.is_contiguous() and gs_cl.is_contiguous(memory_format=CL)
    assert torch.equal(gf_p, gf_cl)         # written without atomics
    # grad_source and grad_weight are fp32 sums of reductions in whatever order they land, rounded to bf16 once: a
    # different order may move a value across a rounding boundary (one bf16 ulp, 2^-7 relative at most)
    for a, b in ((gs_p, gs_cl), (gw_p, gw_cl)):
        a, b = a.double(), b.double()
        assert ((a - b).abs() <= 2.0 ** -7 * b.abs() + 1e-6 * b.abs().max()).all()


# -------------------------------------------------------------------------------------------------- 5. fallback
@pytest.mark.parametrize("variant", ["fp32", "fp16", "C48", "N64"])
def test_unserved_calls_run_the_composition(G, variant):
    """the same value bit for bit; the same gradients up to the order of the composition's own atomic adds
    (block_extract_bwd's scatter, cuDNN's weight gradient)"""
    k = 3
    C, n, dt = {"fp32": (64, 128, torch.float32), "fp16": (64, 128, torch.float16), "C48": (48, 128, torch.bfloat16),
                "N64": (64, 64, torch.bfloat16)}[variant]
    s, f, w, g = make(2, C, 15, 22, 13, 20, k, "smooth", seed=1, n=n)
    s, w, g = s.to(dt).contiguous(), w.to(dt), g.to(dt).contiguous()
    res = []
    for fn in (lambda a, b, c: G.patch_conv(a, b, c, k),
               lambda a, b, c: F.conv2d(G.BlockExtractor(k)(a, b), c, None, stride=k)):
        a, b, c = (t.clone().requires_grad_() for t in (s, f, w))
        out = fn(a, b, c)
        out.backward(g)
        res.append((out, a.grad, b.grad, c.grad))
    assert torch.equal(res[0][0], res[1][0])
    for x, y in zip(res[0][1:], res[1][1:]):
        x, y = x.double(), y.double()
        assert (x - y).abs().max().item() <= 1e-2 * y.abs().max().item()


# ---------------------------------------------------------------------------------------------------- 6. module
WITNESS = "k_local_attn_fwd_tc"     # a library kernel every ExtractorAttn step launches, whichever conv path it takes


def _kernel_names(fn, tries=3):
    """names of the kernels one profiled call of fn launched, from the first of up to `tries` profiling sessions that
    recorded this library's kernels at all (WITNESS).  Late in a long test process, every other session has been seen
    to return torch's own kernels but none launched from libgfla_warp.so, with the next session complete again; such a
    session says nothing about which kernels ran, so it is repeated rather than judged."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(tries):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = [e.key for e in prof.key_averages()]
        if any(WITNESS in n for n in names):
            break
    return names


@pytest.fixture
def _no_tf32():
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = old


@pytest.mark.parametrize("level", [(256, 32, 3), (128, 64, 5)])
def test_extractor_attn_uses_the_patch_conv_kernels(G, level, _no_tf32):
    C, S, k = level
    torch.manual_seed(C + k)
    m = G.ExtractorAttn(C, k, softmax=True).to(DEV).bfloat16().to(memory_format=CL)
    src = torch.randn(2, C, S, S, device=DEV).bfloat16().contiguous(memory_format=CL)
    tgt = torch.randn(2, C, S, S, device=DEV).bfloat16().contiguous(memory_format=CL)
    flow = (torch.rand(2, 2, S, S, device=DEV) * 6 - 3).bfloat16()
    conv1, conv2 = m.fully_connect_layer[0], m.fully_connect_layer[2]
    w_src = conv1.weight[:, C:]

    def step():
        a, fl = src.clone().requires_grad_(), flow.clone().requires_grad_()
        m(a, tgt, fl).float().mean().backward()
    names = _kernel_names(step)
    for kern in ("k_patch_conv_fwd_tc", "k_patch_conv_bwd_tc", "k_patch_conv_wgrad_tc", "k_local_attn_fwd_tc", "k_local_attn_bwd_tc"):
        assert any(kern in n for n in names), (kern, names)
    assert not [n for n in names if "k_block_extract_fwd" in n or "k_block_extract_bwd" in n]
    m.zero_grad()

    # the source half inside the module: within the forward bound of the fp64 conv of the bf16 block tensor
    with torch.no_grad():
        x = G.patch_conv(src, flow, w_src, k)
        r = reference(G, src, flow.float(), w_src, None, k)
        ref64.assert_within("source half", host(x), r["out"], bound_out(r["out"], r["M"], C, k))
        # logits: the fused module against the materialised composition, which differs only in that source half (both
        # round it to bf16 and then run the same bf16 ops): the difference of the source halves (both within the bound)
        # passes through the bf16 sum with the target half, the LeakyReLU (1-Lipschitz) and the 1x1 conv
        lf, _ = m._logits(src, tgt, flow)
        lm, blk = m._logits(src, tgt, flow, materialise=True)
        assert blk is not None
        xm = F.conv2d(blk, w_src, None, stride=k)
        lo, hi = k // 2, k - 1 - k // 2
        xt = F.conv2d(F.pad(tgt, (lo, hi, lo, hi), mode="replicate"), conv1.weight[:, :C], conv1.bias)
        u = ref64.U_BF16
        dx = 2 * bound_out(r["out"], r["M"], C, k) + 2 * u * (np.abs(host(xm)) + np.abs(host(xt)))
        w2 = np.abs(host(conv2.weight)[:, :, 0, 0])
        h = np.abs(host(F.leaky_relu(xm + xt, 0.01)))
        bound = (np.einsum("on,bnhw->bohw", w2, dx + 2 * u * h) + 2 * ref64.gamma(N_OUT) * np.einsum("on,bnhw->bohw", w2, h)
                 + 2 * u * np.abs(host(lm)) + ref64.ETA_BF16)
        ref64.assert_within("logits", host(lf), host(lm), bound)

    # gradients of the whole module: fused against the materialised composition (the reference ExtractorAttn chain)
    grads = {}
    for mat in (False, True):
        a, fl = src.clone().requires_grad_(), flow.clone().requires_grad_()
        m.zero_grad()
        if mat:
            logits, blk = m._logits(a, tgt, fl, materialise=True)
        else:
            logits, _ = m._logits(a, tgt, fl)
        out = G.local_attention(a, fl, logits, k)
        out.float().square().mean().backward()
        grads[mat] = (a.grad.float(), fl.grad.float(), conv1.weight.grad.float())
    for name, x_f, x_m in zip(("source", "flow", "conv1.weight"), grads[False], grads[True]):
        err, ref = (x_f - x_m).norm().item(), x_m.norm().item()
        assert err <= 2e-2 * ref, (name, err, ref)


def test_pose_generator_bf16_runs_no_block_extract():
    import bench_models
    if bench_models.reference_root() is None:
        pytest.skip("baseline/_ref snapshot of the reference generators not present")
    from test_gpu_models import _build, _pose_inputs
    net = _build(bench_models, "fused", "pose", torch.bfloat16, cl=True)
    x = _pose_inputs(2, torch.bfloat16, CL)

    def step():
        img, flows, masks = net(*x)
        img.float().mean().backward()
    names = _kernel_names(step)
    assert any("k_patch_conv_fwd_tc" in n for n in names) and any("k_patch_conv_bwd_tc" in n for n in names), names
    assert not [n for n in names if "k_block_extract_fwd" in n or "k_block_extract_bwd" in n]


# ---------------------------------------------------------------------------------------------------- 7. memory
def test_transient_memory_is_a_fraction_of_one_block_tensor(G):
    B, C, S, k = 8, 128, 64, 5
    s, f, w, g = make(B, C, S, S, S, S, k, "smooth", seed=2)
    s.requires_grad_()
    f.requires_grad_()
    w.requires_grad_()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = G.patch_conv(s, f, w, k)
    out.backward(g)
    torch.cuda.synchronize()
    kept = sum(t.numel() * t.element_size() for t in (out, s.grad, f.grad, w.grad))
    rise = torch.cuda.max_memory_allocated() - base - kept
    block = B * C * k * S * k * S * 2
    assert rise < block / 4, (rise, block)
