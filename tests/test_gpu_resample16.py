"""GPU (-m gpu): resample2d and the fused resample2d -> cosine op on bf16 / fp16 feature maps (k_resample2d16_*,
csrc/resample2d.cu).  A 16-bit call computes what the fp32 kernels compute on the widened inputs and rounds each 16-bit
output once: out, cos and grad_target are compared with the narrowed fp32 results bit for bit, grad_input2 and the stats
(fp32) bit for bit, and grad_input1 (an fp32 atomic scatter, rounded once) against the 16-bit bound of the fp64 reference
(ref64_resample16).  Then the modules, PerceptualCorrectness in a bf16 pipeline, and the deterministic mode."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import ref64_resample as rr
from ref64_resample16 import check16, round16
from test_gpu_resample_bounds import COS, DILS, KS, SHAPES, cases, cos_inputs
from test_ref64_resample import make_in2

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
EPS = 1e-8
KINDS = {"bf16": torch.bfloat16, "fp16": torch.float16}
WORST = {}


def cu(a, dt=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    return t if dt is None else t.to(dt)


def host(t):
    return t.detach().float().cpu().numpy().astype(np.float64)


def within(row, y, ref, b32, kind):
    worst, msg = check16(row, host(y), ref, b32, kind)
    assert msg is None, msg
    WORST[row] = max(WORST.get(row, 0.0), worst)


@pytest.fixture(scope="module", autouse=True)
def worst_ratios():
    yield
    print("\nlargest |err|/bound per output and path:")
    for row in sorted(WORST):
        print(f"  {row:44s} {WORST[row]:.3f}")


@pytest.fixture(scope="module")
def F_():
    import gfla_b200
    from gfla_b200 import _lib
    _lib.check(_lib.lib().gfla_device_check(), "device check")
    return gfla_b200.functional


# --------------------------------------------------------------------------------------------------- resample2d
@pytest.mark.parametrize("dil", DILS)
@pytest.mark.parametrize("ks", KS)
@pytest.mark.parametrize("kind", sorted(KINDS))
def test_resample2d16_equals_narrowed_fp32(F_, kind, ks, dil):
    dt = KINDS[kind]
    u, eta = rr.unit(np.float32)
    for flow, a, in2, g in cases(np.float32, ks, dil):
        a16, g16, t2 = cu(a, dt), cu(g, dt), cu(in2)
        out = F_.resample2d_fwd(a16, t2, ks, dil)
        assert out.dtype == dt
        assert torch.equal(out, F_.resample2d_fwd(a16.float(), t2, ks, dil).to(dt)), (flow, ks, dil)
        g1, g2 = F_.resample2d_bwd(a16, t2, g16, ks, dil)
        assert g1.dtype == dt and g2.dtype == torch.float32
        assert torch.equal(g2, F_.resample2d_bwd(a16.float(), t2, g16.float(), ks, dil)[1]), (flow, ks, dil)
        r = rr.resample2d(host(a16), in2, ks, dil, host(g16))
        path = "shuffle" if rr.fast_warps(in2, ks, dil, *a.shape[2:]).all() else "per tap/mixed"
        within(f"grad_in1 {kind} {path}", g1, r["gin1"], rr.bound_in1(r["gin1"], r["mags_in1"], u, eta), kind)


def test_cases_cover_both_grad_input1_paths():
    fast = [rr.fast_warps(in2, ks, 1, *a.shape[2:]).all() for ks in (2, 4) for _, a, in2, _ in cases(np.float32, ks, 1)]
    assert any(fast) and not all(fast), fast


@pytest.mark.parametrize("ks", [4, 6])
@pytest.mark.parametrize("kind", sorted(KINDS))
def test_resample2d16_backward_accumulates(F_, kind, ks):
    """accumulate = 1 through the C ABI: grad_input2 equals the fp32 kernel's accumulation bit for bit, grad_input1 (fp32
    atomics) stays within the fp32 bound around reference + initial value"""
    from gfla_b200 import _lib
    from gfla_b200.functional import _dt, _p, _stream
    dt = KINDS[kind]
    u, eta = rr.unit(np.float32)
    B, C, Hi, Wi, H, W = SHAPES[1]
    rng = np.random.default_rng(ks)
    in2 = make_in2("smooth", rng, B, H, W, Hi, Wi, 2.0, np.float32)
    a16, g16, t2 = cu(rng.standard_normal((B, C, Hi, Wi)), dt), cu(rng.standard_normal((B, C, H, W)), dt), cu(in2)
    i1, i2 = cu(rng.standard_normal((B, C, Hi, Wi)).astype(np.float32)), cu(rng.standard_normal(in2.shape).astype(np.float32))
    g1, g2 = i1.clone(), i2.clone()
    _lib.check(_lib.lib().gfla_resample2d16_bwd(_p(a16), _p(t2), _p(g16), _p(g1), _p(g2), B, C, Hi, Wi, H, W, ks, 1, _dt(a16), 1,
                                                _stream(a16)), "resample2d16_bwd")
    a32, go32, r1, r2 = a16.float(), g16.float(), i1.clone(), i2.clone()
    _lib.check(_lib.lib().gfla_resample2d_bwd(_p(a32), _p(t2), _p(go32), _p(r1), _p(r2), B, C, Hi, Wi, H, W, ks, 1, _lib.GFLA_F32, 1,
                                              _stream(a16)), "resample2d_bwd")
    assert torch.equal(g2, r2)
    r = rr.resample2d(host(a16), in2, ks, 1, host(g16))
    init = host(i1)
    ref = r["gin1"] + init
    err = np.abs(host(g1) - ref) / rr.bound_in1(ref, r["mags_in1"], u, eta, init)
    assert err.max() <= 1.0, err.max()


# ------------------------------------------------------------------------------------------------ fused cosine
# Runs in a fresh process per SM count (sm_count() is read once per process): every COS case in bf16 and fp16 against the
# fp32 kernels on the widened inputs, accumulate = 1 through the ABI, and one profiled forward + backward of a C < 64 case
# and a C >= 64 case (with 100000 SMs: the TS = 1 and the TS = 4 instances in one session).
_RUN = r"""
import sys
import numpy as np
import torch
import gfla_b200
from gfla_b200 import _lib
from gfla_b200.functional import _dt, _p, _stream
F = gfla_b200.functional
L = _lib.lib()
z = np.load(sys.argv[1])
out = {}
host = lambda t: t.detach().float().cpu().numpy()
eq = lambda a, b: np.array(bool(torch.equal(a, b)))
for kind, dt in (("bf16", torch.bfloat16), ("fp16", torch.float16)):
    for key in sorted({k.split("/")[1] for k in z.files if k.startswith(kind + "/")}):
        k = f"{kind}/{key}"
        a, t, gc = (torch.from_numpy(z[f"{k}/{n}"]).cuda().to(dt) for n in ("a", "t", "gc"))
        in2 = torch.from_numpy(z[f"{k}/in2"]).cuda()
        ks, dil = (int(v) for v in z[f"{k}/ks_dil"])
        B, C, Hi, Wi = a.shape
        H, W = in2.shape[2:]
        cos, st = F.resample2d_cosine_fwd(a, in2, t, ks, dil, 1e-8)
        cos32, st32 = F.resample2d_cosine_fwd(a.float(), in2, t.float(), ks, dil, 1e-8)
        out[k + "/cos_eq"], out[k + "/stats_eq"] = eq(cos, cos32.to(dt)), eq(st, st32)
        out[k + "/dtypes"] = np.array(cos.dtype == dt and st.dtype == torch.float32)
        g1, g2, g3 = F.resample2d_cosine_bwd(a, in2, t, st, gc, ks, dil, 1e-8, need_input1=True, need_target=True)
        _, r2, r3 = F.resample2d_cosine_bwd(a.float(), in2, t.float(), st32, gc.float(), ks, dil, 1e-8, need_target=True)
        out[k + "/gin2_eq"], out[k + "/gt_eq"] = eq(g2, r2), eq(g3, r3.to(dt))
        out[k + "/gin1"] = host(g1)
        # accumulate = 1: grad_in2 and grad_target added into non-zero buffers, grad_target widened, added, rounded once
        rng = np.random.default_rng(0)
        i2 = torch.from_numpy(rng.standard_normal(in2.shape).astype(np.float32)).cuda()
        it = torch.from_numpy(rng.standard_normal(t.shape).astype(np.float32)).cuda().to(dt)
        a2, at = i2.clone(), it.clone()
        _lib.check(L.gfla_resample2d16_cosine_bwd(_p(a), _p(in2), _p(t), _p(st), _p(gc), None, _p(a2), None, _p(at), B, C, Hi, Wi,
                                                  H, W, ks, dil, 1e-8, _dt(a), 1, _stream(a)), "resample2d16_cosine_bwd")
        b2, bt = i2.clone(), it.float()
        a32, t32, gc32 = a.float(), t.float(), gc.float()       # kept alive until the kernel has run
        _lib.check(L.gfla_resample2d_cosine_bwd(_p(a32), _p(in2), _p(t32), _p(st32), _p(gc32), None, _p(b2), None, _p(bt), B, C, Hi,
                                                Wi, H, W, ks, dil, 1e-8, _lib.GFLA_F32, 1, _stream(a)), "resample2d_cosine_bwd")
        torch.cuda.synchronize()
        out[k + "/acc_gin2_eq"], out[k + "/acc_gt_eq"] = eq(a2, b2), eq(at, bt.to(dt))
keys = [str(v) for v in z["profile_keys"]]
if keys:
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):                                    # a session that recorded none of this library's kernels is repeated
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for key in keys:
                a, t, gc = (torch.from_numpy(z[f"bf16/{key}/{n}"]).cuda().bfloat16() for n in ("a", "t", "gc"))
                in2 = torch.from_numpy(z[f"bf16/{key}/in2"]).cuda()
                ks, dil = (int(v) for v in z[f"bf16/{key}/ks_dil"])
                cos, st = F.resample2d_cosine_fwd(a, in2, t, ks, dil, 1e-8)
                F.resample2d_cosine_bwd(a, in2, t, st, gc, ks, dil, 1e-8)
            torch.cuda.synchronize()
        names = [e.key for e in prof.key_averages()]
        if any("k_resample2d16_cos" in n for n in names):
            break
    out["kernel_names"] = np.array(names)
np.savez(sys.argv[2], **out)
"""


def cos_inputs16(i, kind):
    """test_gpu_resample_bounds' cosine case i with source, target and grad_cos rounded to the 16-bit type"""
    a, in2, t, gc, ks, dil = cos_inputs(i, np.float32)
    return round16(a, kind), in2, round16(t, kind), round16(gc, kind), ks, dil


@pytest.fixture(scope="module")
def cos_runs(tmp_path_factory):
    from conftest import ROOT
    d = tmp_path_factory.mktemp("cos16")
    inp = {}
    for kind in KINDS:
        for i in range(len(COS)):
            a, in2, t, gc, ks, dil = cos_inputs16(i, kind)
            k = f"{kind}/c{i}"
            inp.update({f"{k}/a": a, f"{k}/in2": in2, f"{k}/t": t, f"{k}/gc": gc, f"{k}/ks_dil": np.array([ks, dil])})
    res = {}
    for sm in (1, 100000):
        inp["profile_keys"] = np.array(["c0", "c1"] if sm == 100000 else [])
        src, dst = d / f"in_{sm}.npz", d / f"out_{sm}.npz"
        np.savez(src, **inp)
        subprocess.run([sys.executable, "-c", _RUN, str(src), str(dst)], cwd=ROOT, env=dict(os.environ, GFLA_SM_COUNT=str(sm)),
                       check=True)
        res[sm] = dict(np.load(dst))
    return res


def test_cosine16_both_slicings_ran(cos_runs):
    assert rr.cos_slices(*(COS[0][i] for i in (0, 1, 4, 5)), COS[0][6], 100000) == 1
    assert rr.cos_slices(*(COS[1][i] for i in (0, 1, 4, 5)), COS[1][6], 100000) == 4
    names = [str(n) for n in cos_runs[100000]["kernel_names"]]
    for n in ("k_resample2d16_cos_fwd<__nv_bfloat16, 2, 1>", "k_resample2d16_cos_bwd<__nv_bfloat16, 2, 1>",
              "k_resample2d16_cos_fwd<__nv_bfloat16, 1, 4>", "k_resample2d16_cos_bwd<__nv_bfloat16, 1, 4>"):
        assert any(n in m for m in names), (n, names)


@pytest.mark.parametrize("i", range(len(COS)))
@pytest.mark.parametrize("kind", sorted(KINDS))
def test_cosine16_equals_narrowed_fp32(cos_runs, kind, i):
    a, in2, t, gc, ks, dil = cos_inputs16(i, kind)
    u, eta = rr.unit(np.float32)
    c = rr.cosine(a, in2, t, ks, dil, EPS, gc)
    for sm, res in cos_runs.items():
        k = f"{kind}/c{i}"
        for what in ("dtypes", "cos_eq", "stats_eq", "gin2_eq", "gt_eq", "acc_gin2_eq", "acc_gt_eq"):
            assert bool(res[f"{k}/{what}"]), (what, kind, i, sm)
        TS = rr.cos_slices(*(COS[i][j] for j in (0, 1, 4, 5)), ks, sm)
        worst, msg = check16(f"cos grad_in1 {kind} TS={TS}", res[f"{k}/gin1"], c["gin1"],
                             rr.bound_in1(c["gin1"], c["mags_in1"], u, eta), kind)
        assert msg is None, msg
        WORST[f"cos grad_in1 {kind} TS={TS}"] = max(WORST.get(f"cos grad_in1 {kind} TS={TS}", 0.0), worst)


# ------------------------------------------------------------------------------------------------------- modules
def _module_inputs(feat, flow_dt, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    src = torch.randn(2, 24, 20, 36, device=DEV, generator=g).to(feat)
    tgt = torch.randn(2, 24, 16, 40, device=DEV, generator=g).to(feat)
    flow = (torch.rand(2, 2, 16, 40, device=DEV, generator=g) * 6 - 3).to(flow_dt)
    return src.requires_grad_(), tgt.requires_grad_(), flow.requires_grad_()


COMBOS = [(torch.bfloat16, torch.bfloat16), (torch.bfloat16, torch.float32), (torch.float16, torch.float16),
          (torch.float16, torch.float32), (torch.float32, torch.bfloat16)]


@pytest.mark.parametrize("feat,flow_dt", COMBOS, ids=lambda d: str(d).split(".")[-1])
def test_modules_keep_dtypes_and_match_functional(F_, feat, flow_dt):
    import gfla_b200
    ks, sigma = 4, 2.0
    src, tgt, flow = _module_inputs(feat, flow_dt)
    in2 = torch.cat([flow.detach().float(), torch.full((2, 1, 16, 40), sigma, device=DEV)], 1)
    # Resample2d
    out = gfla_b200.Resample2d(ks, 1, sigma)(src, flow)
    assert out.dtype == feat and torch.equal(out, F_.resample2d_fwd(src.detach(), in2, ks, 1))
    go = torch.randn_like(out)
    out.backward(go)
    r1, r2 = F_.resample2d_bwd(src.detach(), in2, go, ks, 1)
    assert src.grad.dtype == feat and flow.grad.dtype == flow_dt
    assert torch.equal(flow.grad, r2[:, :2].to(flow_dt))
    u, eta = rr.unit(np.float32)
    # grad_input1 is an atomic scatter: compare against the bound, not bit for bit
    r = rr.resample2d(host(src), host(in2).astype(np.float32), ks, 1, host(go))
    kind = "fp16" if feat == torch.float16 else "bf16"
    b32 = rr.bound_in1(r["gin1"], r["mags_in1"], u, eta)
    if feat == torch.float32:
        assert (np.abs(host(src.grad) - r["gin1"]) <= b32).all()
    else:
        within(f"module grad_in1 {kind}", src.grad, r["gin1"], b32, kind)
    # Resample2dCosine
    src.grad = flow.grad = None
    cos = gfla_b200.Resample2dCosine(ks, 1, sigma)(src, flow, tgt)
    c_ref, st = F_.resample2d_cosine_fwd(src.detach(), in2, tgt.detach(), ks, 1, 1e-8)
    assert cos.dtype == feat and torch.equal(cos, c_ref)
    gc = torch.randn_like(cos)
    cos.backward(gc)
    _, c2, ct = F_.resample2d_cosine_bwd(src.detach(), in2, tgt.detach(), st, gc, ks, 1, 1e-8, need_target=True)
    assert src.grad.dtype == feat and tgt.grad.dtype == feat and flow.grad.dtype == flow_dt
    assert torch.equal(flow.grad, c2[:, :2].to(flow_dt)) and torch.equal(tgt.grad, ct)


# ------------------------------------------------------------------------------------------- the loss, bf16 pipeline
class VGGLayers(torch.nn.Module):
    """torchvision's VGG19 features (random weights) -> {'relu1_1', 'relu2_1', 'relu3_1', 'relu4_1'}, frozen like the
    reference's VGG19; `cast`: the dtype the features are handed on in"""
    CUTS = {"relu1_1": 1, "relu2_1": 6, "relu3_1": 11, "relu4_1": 20}

    def __init__(self, features, cast=None):
        super().__init__()
        self.features, self.cast = features, cast

    def forward(self, x):
        out, h = {}, x.to(next(self.features.parameters()).dtype)
        for i, layer in enumerate(self.features[:21]):
            h = layer(h)
            for name, cut in self.CUTS.items():
                if i == cut:
                    out[name] = h if self.cast is None else h.to(self.cast)
        return out


def _vgg():
    import torchvision
    torch.manual_seed(0)
    f = torchvision.models.vgg19(weights=None).features.to(DEV).eval()
    for p in f.parameters():
        p.requires_grad_(False)
    return f


def _loss(vgg, imgs, flows):
    import gfla_b200
    return gfla_b200.PerceptualCorrectness(vgg=vgg)(imgs[0], imgs[1], flows, [2, 1])


def _images(dt):
    g = torch.Generator(device=DEV).manual_seed(3)
    return [torch.rand(2, 3, 64, 96, device=DEV, generator=g).to(dt) for _ in range(2)]


def _flows(dt):
    """at the feature resolution of relu3_1 and relu2_1 (F.interpolate is then the identity); displacements of up to 8 pixels
    move the loss well away from its floor, where a relative comparison means something"""
    g = torch.Generator(device=DEV).manual_seed(4)
    return [(torch.rand(2, 2, h, w, device=DEV, generator=g) * 16 - 8).to(dt).requires_grad_() for h, w in ((16, 24), (32, 48))]


def test_perceptual_correctness_bf16_vgg_bf16_flows():
    from torch.profiler import ProfilerActivity, profile
    feats = _vgg().bfloat16()
    imgs, flows = _images(torch.bfloat16), _flows(torch.bfloat16)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        loss = _loss(VGGLayers(feats), imgs, flows)
        loss.backward()
        torch.cuda.synchronize()
    names = [e.key for e in prof.key_averages()]
    assert any("k_resample2d16_cos_fwd<__nv_bfloat16" in n for n in names), names
    assert any("k_resample2d16_cos_bwd<__nv_bfloat16" in n for n in names), names
    assert torch.isfinite(loss) and all(f.grad is not None and f.grad.dtype == torch.bfloat16 for f in flows)
    # the same loss on fp32 copies of the same bf16-valued features and flows
    flows32 = [f.detach().float().requires_grad_() for f in flows]
    loss32 = _loss(VGGLayers(feats, cast=torch.float32), imgs, flows32)
    loss32.backward()
    assert abs(loss.item() - loss32.item()) <= 1e-2 * abs(loss32.item()), (loss.item(), loss32.item())
    for f, f32 in zip(flows, flows32):
        assert (f.grad.float() - f32.grad).abs().max() <= 1e-2 * f32.grad.abs().max()


def test_perceptual_correctness_fp32_vgg_bf16_flows():
    feats = _vgg()
    imgs, flows = _images(torch.float32), _flows(torch.bfloat16)
    loss = _loss(VGGLayers(feats), imgs, flows)
    loss.backward()
    flows32 = [f.detach().float().requires_grad_() for f in flows]
    loss32 = _loss(VGGLayers(feats), imgs, flows32)
    loss32.backward()
    assert loss.dtype == torch.float32 and torch.equal(loss, loss32)
    for f, f32 in zip(flows, flows32):
        assert f.grad.dtype == torch.bfloat16 and torch.equal(f.grad, f32.grad.to(torch.bfloat16))


# -------------------------------------------------------------------------------------------------- determinism
_DET = r"""
import sys
import torch
sys.path.insert(0, "tests")
from test_gpu_resample16 import VGGLayers, _flows, _images, _loss, _vgg
torch.use_deterministic_algorithms(True)
feats = _vgg().bfloat16()
grads = []
for _ in range(2):
    flows = _flows(torch.bfloat16)
    _loss(VGGLayers(feats), _images(torch.bfloat16), flows).backward()
    grads.append([f.grad for f in flows])
assert all(torch.equal(a, b) for a, b in zip(*grads))
print("identical")
"""


def test_deterministic_mode_16bit():
    import gfla_b200
    from conftest import ROOT
    src, _, flow = _module_inputs(torch.bfloat16, torch.bfloat16)
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        out = gfla_b200.Resample2d(4, 1, 2.0)(src, flow)
        with pytest.raises(RuntimeError, match="does not have a deterministic implementation"):
            out.backward(torch.ones_like(out))
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)
    # the loss's backward (flow gradient only, no scatter) runs under the flag; cuBLAS's bmm needs its workspace setting,
    # which is read when cuBLAS starts: a fresh process
    r = subprocess.run([sys.executable, "-c", _DET], cwd=ROOT, env=dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8"),
                       capture_output=True, text=True)
    assert r.returncode == 0 and "identical" in r.stdout, r.stdout + r.stderr
