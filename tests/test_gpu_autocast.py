"""GPU (-m gpu): torch.autocast("cuda") on the fused ops.

  * ExtractorAttn with fp32 parameters and channels-last fp32 inputs, under autocast bf16 and fp16, at the two attention
    levels of the pose generator: the output and every gradient equal, bit for bit, the same computation on hand-cast
    inputs (source and logits in the autocast dtype, the flow in fp32, the weights cast where autocast casts them), and
    the tile kernels run (and the patch-convolution kernels, for bf16);
  * one reference PoseGenerator training step under autocast fp16 with a GradScaler, and under autocast bf16: finite,
    every attention level on the tile kernels, and close to the fp32 step;
  * PerceptualCorrectness and MultiAffineRegularizationLoss under both autocast dtypes: finite flow gradients.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from kernel_names import kernel_names

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
CL = torch.channels_last
DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}
TNAME = {torch.bfloat16: "__nv_bfloat16", torch.float16: "__half"}


@pytest.fixture(scope="module")
def G():
    import gfla_b200
    from gfla_b200 import _lib
    _lib.check(_lib.lib().gfla_device_check(), "device check")
    return gfla_b200


@pytest.fixture
def det():
    """bit-for-bit comparisons of gradients need the deterministic backward kernels (the default ones add with atomics)"""
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)


def _hand_cast(G, m, src, tgt, flow, dt):
    """ExtractorAttn.forward (softmax variant) with every cast autocast makes written out: each op casts its own fp32
    inputs, so source is cast once for patch_conv and once for local_attention, and the replicate-padded target is cast
    after the pad (F.pad is not an autocast op)"""
    conv1, act, conv2 = m.fully_connect_layer[0], m.fully_connect_layer[1], m.fully_connect_layer[2]
    k, c = m.kernel_size, src.shape[1]
    x = G.patch_conv(src.to(dt), flow, conv1.weight[:, c:].to(dt), k)
    lo, hi = k // 2, k - 1 - k // 2
    x = x + F.conv2d(F.pad(tgt, (lo, hi, lo, hi), mode="replicate").to(dt), conv1.weight[:, :c].to(dt), conv1.bias.to(dt))
    x = F.conv2d(act(x), conv2.weight.to(dt), conv2.bias.to(dt))
    return G.local_attention(src.to(dt), flow, x, k)


@pytest.mark.parametrize("dt", list(DTYPES), ids=list(DTYPES))
@pytest.mark.parametrize("level", [(256, 32, 3), (128, 64, 5)], ids=["256x32x32-k3", "128x64x64-k5"])
def test_extractor_attn_under_autocast_equals_hand_cast(G, det, level, dt, tmp_path):
    dname = dt
    dt = DTYPES[dt]
    C, S, k = level
    torch.manual_seed(C + k)
    m = G.ExtractorAttn(C, k, softmax=True).to(DEV).to(memory_format=CL)
    gen = torch.Generator().manual_seed(C)
    src = torch.randn(2, C, S, S, generator=gen).to(DEV).contiguous(memory_format=CL)
    tgt = torch.randn(2, C, S, S, generator=gen).to(DEV).contiguous(memory_format=CL)
    flow = (torch.rand(2, 2, S, S, generator=gen) * 6 - 3).to(DEV)

    def run(fn):
        xs = [t.clone().requires_grad_() for t in (src, tgt, flow)]
        m.zero_grad(set_to_none=True)
        out = fn(*xs)
        out.float().square().sum().backward()
        return out.detach(), [x.grad for x in xs] + [p.grad for p in m.parameters()]

    def auto(*xs):
        with torch.autocast("cuda", dtype=dt):
            return m(*xs)

    out_a, grads_a = run(auto)
    out_h, grads_h = run(lambda *xs: _hand_cast(G, m, *xs, dt))
    assert out_a.dtype == dt and torch.equal(out_a, out_h)
    assert len(grads_a) == 7
    for i, (a, h) in enumerate(zip(grads_a, grads_h)):
        assert a is not None and a.dtype == torch.float32, i          # every gradient in its input's own dtype
        assert torch.equal(a, h), i
    # the kernels one autocast training step of the same module launches (profiled in a child process: kernel_names.py)
    names = kernel_names(f"""
import gfla_b200
CL = torch.channels_last
torch.manual_seed({C + k})
m = gfla_b200.ExtractorAttn({C}, {k}, softmax=True).to("cuda").to(memory_format=CL)
x = [torch.randn(2, {C}, {S}, {S}, device="cuda").contiguous(memory_format=CL) for _ in range(2)]
x.append(torch.rand(2, 2, {S}, {S}, device="cuda") * 6 - 3)
x = [t.requires_grad_() for t in x]


def step():
    with torch.autocast("cuda", dtype=torch.{ {"bf16": "bfloat16", "fp16": "float16"}[dname] }):
        out = m(*x)
    out.float().square().sum().backward()


NAMES = profiled(step)
""", tmp_path)
    assert any("k_local_attn_fwd_tc" in n and TNAME[dt] in n for n in names), names
    assert any("k_local_attn_bwd_tc" in n and TNAME[dt] in n for n in names), names
    assert not [n for n in names if "gfla::k_local_attn_fwd<" in n or "gfla::k_local_attn_bwd<" in n], names
    if dt == torch.bfloat16:
        assert any("k_patch_conv_fwd_tc" in n for n in names) and any("k_patch_conv_bwd_tc" in n for n in names), names
    else:       # fp16 patch convolution runs the composition: BlockExtractor and a cuDNN conv
        assert not any("k_patch_conv" in n for n in names) and any("k_block_extract_fwd" in n for n in names), names


def test_extractor_attn_blend_under_autocast(G):
    """the inference blend (mask=, no grad): target and mask follow the attention's dtype"""
    torch.manual_seed(0)
    m = G.ExtractorAttn(128, 5, softmax=True).to(DEV).to(memory_format=CL)
    src = torch.randn(2, 128, 64, 64, device=DEV).contiguous(memory_format=CL)
    tgt = torch.randn(2, 128, 64, 64, device=DEV).contiguous(memory_format=CL)
    flow = torch.rand(2, 2, 64, 64, device=DEV) * 6 - 3
    mask = torch.rand(2, 1, 64, 64, device=DEV)
    for dt in DTYPES.values():
        with torch.no_grad(), torch.autocast("cuda", dtype=dt):
            out = m(src, tgt, flow, mask=mask)
            attn = m(src, tgt, flow)
            probs, res = m.hook_attn_param(src, tgt, flow)
        assert out.dtype == dt and attn.dtype == dt and probs.dtype == dt and res.dtype == dt
        assert torch.equal(res, attn)
        ref = tgt.to(dt).float() * (1 - mask.to(dt).float()) + attn.float() * mask.to(dt).float()
        # the kernel blends in fp32 and rounds once: within one unit of the 16-bit type plus the blend's own rounding
        assert (out.float() - ref).abs().max().item() <= 2 * (2.0 ** -8 if dt == torch.bfloat16 else 2.0 ** -11) * ref.abs().max().item()


# ------------------------------------------------------------------------------------------------------ generator
@pytest.fixture(scope="module")
def BM():
    import bench_models
    if bench_models.reference_root() is None:
        pytest.skip("baseline/_ref snapshot of the reference generators not present")
    return bench_models


@pytest.fixture
def no_tf32():
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


@pytest.mark.parametrize("dt", list(DTYPES), ids=list(DTYPES))
def test_pose_generator_training_step_under_autocast(G, BM, no_tf32, dt, tmp_path):
    dname = dt
    dt = DTYPES[dt]
    Pose, _ = BM.load_generators("fused")
    torch.manual_seed(11)
    net = Pose(**BM.POSE_KW)
    net.init_weights("orthogonal", gain=0.5)
    net = net.to(DEV).to(memory_format=CL)
    gen = torch.Generator(device="cpu").manual_seed(3)
    x = [torch.randn(1, c, 256, 256, generator=gen).to(DEV).contiguous(memory_format=CL) for c in (3, 18, 18)]
    with torch.no_grad():
        img32, _, _ = net(*x)
    opt = torch.optim.SGD(net.parameters(), lr=0.0)
    # a GradScaler for fp16, as the mixed-precision recipe has it; 2^12 instead of the default 2^16 start, which is a guess
    # the scaler lowers by skipping overflowing steps: this test takes one step, and it must not be a skipped one
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 12, enabled=dt == torch.float16)
    with torch.autocast("cuda", dtype=dt):
        img, flows, _ = net(*x)
        loss = img.float().mean() + sum(f.float().pow(2).mean() for f in flows)
    scaler.scale(loss).backward()
    scaler.unscale_(opt)
    assert torch.isfinite(img.float()).all() and torch.isfinite(loss)
    grads = [p.grad for p in net.parameters() if p.grad is not None]
    assert len(grads) > 50 and all(torch.isfinite(g).all() for g in grads)
    # every attention level (ExtractorAttn) runs the local attention on the tile kernels: no gather kernel at all (one
    # autocast step of the same generator, profiled in a child process: kernel_names.py)
    names = kernel_names(f"""
import bench_models
CL = torch.channels_last
Pose, _ = bench_models.load_generators("fused")
torch.manual_seed(11)
net = Pose(**bench_models.POSE_KW)
net.init_weights("orthogonal", gain=0.5)
net = net.to("cuda").to(memory_format=CL)
x = [torch.randn(1, c, 256, 256, device="cuda").contiguous(memory_format=CL) for c in (3, 18, 18)]


def step():
    with torch.autocast("cuda", dtype=torch.{ {"bf16": "bfloat16", "fp16": "float16"}[dname] }):
        img, flows, _ = net(*x)
        loss = img.float().mean() + sum(f.float().pow(2).mean() for f in flows)
    loss.backward()


NAMES = profiled(step)
""", tmp_path)
    assert any("k_local_attn_fwd_tc" in n and TNAME[dt] in n for n in names), names
    assert any("k_local_attn_bwd_tc" in n and TNAME[dt] in n for n in names), names
    assert not [n for n in names if "gfla::k_local_attn_fwd<" in n or "gfla::k_local_attn_bwd<" in n], names
    # Against the fp32 forward: every conv layer on the image's path rounds its input and weight to the 16-bit type (2 u
    # relative) and the instance norms rescale each layer's output, so errors of different layers add up rather than
    # multiply; independent errors add in RMS, sqrt(L) of them for L layers.  The relative RMS error of the image is then
    # about 2 u sqrt(L); the bound allows 4x that for the norms' rescaling of small-variance channels.
    L = sum(isinstance(mod, torch.nn.Conv2d) for mod in net.modules())
    u = 2.0 ** -8 if dt == torch.bfloat16 else 2.0 ** -11
    rel = ((img.float() - img32).norm() / img32.norm()).item()
    assert rel <= 8 * u * math.sqrt(L), (rel, L)


# ------------------------------------------------------------------------------------------------------ losses
@pytest.mark.parametrize("dt", list(DTYPES), ids=list(DTYPES))
def test_losses_under_autocast(G, dt):
    from test_gpu_resample16 import VGGLayers, _vgg
    dt = DTYPES[dt]
    vgg = VGGLayers(_vgg())                      # fp32 weights: autocast runs its convs in dt
    g = torch.Generator(device=DEV).manual_seed(3)
    imgs = [torch.rand(2, 3, 64, 96, device=DEV, generator=g) for _ in range(2)]
    flows = [(torch.rand(2, 2, h, w, device=DEV, generator=g) * 16 - 8).requires_grad_() for h, w in ((16, 24), (32, 48))]
    with torch.autocast("cuda", dtype=dt):
        loss = G.PerceptualCorrectness(vgg=vgg)(imgs[0], imgs[1], flows, [2, 1])
        reg = G.MultiAffineRegularizationLoss({"2": 5, "3": 3})(flows)
    (loss + reg).backward()
    assert torch.isfinite(loss) and torch.isfinite(reg)
    for f in flows:
        assert f.grad is not None and f.grad.dtype == torch.float32 and torch.isfinite(f.grad).all()
