"""GPU (-m gpu): parity against the REFERENCE'S OWN kernels on the GPU box.

Two reference builds travel with the snapshot (git-ignored, built by ``__graft_entry__.build()`` where
/root/reference exists):
  * ``oracle/_ref/libgfla_ref.so``       -- the reference kernel bodies compiled for the host (OpenMP);
  * ``oracle/_ref/libgfla_ref_cuda.so``  -- the same extracted text compiled by nvcc for sm_90a
    (``oracle/ref_cuda*.cu``: plain launchers, no ATen) = "the reference's CUDA kernels, recompiled".
The CUDA build reaches BASELINE.json's full sizes in milliseconds, so the `<5,256>` tile instantiations
that bench.py times are checked here at 256x256, C=256, k=5 -- forward and backward -- against the reference
itself (chunked, because the reference's `int n` overflows above B=5 at this size), not only against
our own kernels.  Tolerances = north_star: 1e-4 fp32, 1e-2 bf16 (absolute, flat).
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CL = torch.channels_last


@pytest.fixture(scope="module")
def RC():
    import oracle.ref_cuda as rc
    if not rc.available():
        pytest.skip("oracle/_ref/libgfla_ref_cuda.so not built (needs /root/reference at build time)")
    return rc


@pytest.fixture(scope="module")
def F_():
    import gfla_b200
    from gfla_b200 import _lib
    _lib.check(_lib.lib().gfla_device_check(), "device check")
    return gfla_b200.functional


def _smooth_flow(B, H, W, amp=8.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    coarse = torch.rand(B, 2, max(H // 16, 2), max(W // 16, 2), generator=g) * 2 * amp - amp
    return torch.nn.functional.interpolate(coarse, size=(H, W), mode="bilinear", align_corners=True).to(DEV).contiguous()


def _inputs(B, C, H, W, k, kind, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    src = torch.randn(B, C, H, W, generator=g).to(DEV)
    logits = torch.randn(B, k * k, H, W, generator=g).to(DEV)
    gout = torch.randn(B, C, H, W, generator=g).to(DEV)
    flow = _smooth_flow(B, H, W, seed=seed) if kind == "smooth" else ((torch.rand(B, 2, H, W, generator=g) * 16 - 8).to(DEV))
    return src, flow, logits, gout


# ----------------------------------------------------------------------------- the checker itself: nvcc build == host build
@pytest.mark.parametrize("k", [3, 4, 5])
def test_refcuda_equals_host_reference(RC, ref_lib, k):
    """same reference text through g++ (no FMA contraction) and through nvcc (FMA contraction on, like the
    reference's own build): equal up to that contraction"""
    rng = np.random.default_rng(k)
    B, C, H, W = 2, 6, 14, 10
    s = rng.standard_normal((B, C, H, W)).astype(np.float32)
    f = rng.uniform(-6, 6, (B, 2, H, W)).astype(np.float32)
    go = rng.standard_normal((B, C, k * H, k * W)).astype(np.float32)
    ts, tf, tg = (torch.from_numpy(a).to(DEV) for a in (s, f, go))
    np.testing.assert_allclose(RC.block_extract_fwd(ts, tf, k).cpu().numpy(), ref_lib.block_extract_fwd(s, f, k), rtol=1e-6, atol=1e-6)
    gs, gf = RC.block_extract_bwd(ts, tf, tg, k)
    rgs, rgf = ref_lib.block_extract_bwd(s, f, go, k)
    np.testing.assert_allclose(gs.cpu().numpy(), rgs, rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(gf.cpu().numpy(), rgf, rtol=1e-4, atol=1e-4)
    x = rng.standard_normal((B, k * k, H, W)).astype(np.float32)
    assert np.array_equal(RC.attn_reshape_fwd(torch.from_numpy(x).to(DEV), k).cpu().numpy(), ref_lib.attn_reshape_fwd(x, k))
    if k == 4:
        in2 = np.concatenate([f, np.full((B, 1, H, W), 2.0, np.float32)], 1)
        t2 = torch.from_numpy(in2).to(DEV)
        np.testing.assert_allclose(RC.resample2d_fwd(ts, t2, 4, 1).cpu().numpy(), ref_lib.resample2d_fwd(s, in2, 4, 1), rtol=1e-5, atol=1e-6)


# ----------------------------------------------------------------------------- full-size cfg2 samples vs the reference's kernels
@pytest.mark.parametrize("kind", ["smooth", "iid"])
def test_cfg2_fullsize_tile_path_vs_reference_cuda(RC, F_, kind):
    """B=2, C=256, 256x256, k=5, bf16 channels_last -- exactly the <5,256> kernels of the bench step (strip forward,
    tile backward) -- vs the reference's unfused pipeline on its own CUDA kernels in fp32 on the bf16-rounded inputs"""
    B, C, H, W, k = 2, 256, 256, 256, 5
    src, flow, logits, gout = _inputs(B, C, H, W, k, kind, seed=21)
    sb, lb, gb = src.bfloat16(), logits.bfloat16(), gout.bfloat16()
    ref_out, ref_gs, ref_gf, ref_gl = RC.local_attn_fwd_bwd(sb.float(), flow, lb.float(), gb.float(), k, chunk=1)
    s_cl, g_cl = sb.contiguous(memory_format=CL), gb.contiguous(memory_format=CL)
    out = F_.local_attn_fwd(s_cl, flow, lb, k, algo="tile")
    gs, gf, gl = F_.local_attn_bwd(s_cl, flow, lb, g_cl, k, algo="tile")
    assert (out.float() - ref_out).abs().max().item() <= 1e-2
    assert (gs.float() - ref_gs).abs().max().item() <= 1e-2                      # flat, like north_star
    assert (gs.float() - ref_gs).abs().max().item() <= 1e-2 * max(1.0, ref_gs.abs().max().item())
    assert (gl.float() - ref_gl).abs().max().item() <= 1e-2
    # grad_flow sums C*k*k products of O(1) terms: bf16 inputs are exact here, the difference is summation order / Q in fp32
    assert (gf - ref_gf).abs().max().item() <= 1e-2 * max(1.0, ref_gf.abs().max().item())
    # error histogram of grad_source (the bf16 reduce-add path): how far from the bound the bulk sits
    err = (gs.float() - ref_gs).abs()
    assert err.mean().item() <= 1e-3


def test_cfg2_fullsize_planar_nchw_vs_reference_cuda(RC, F_):
    """the reference's own contiguous-NCHW contract at full size (forward NCHW tile kernel, backward through the tile kernels)"""
    B, C, H, W, k = 1, 256, 256, 256, 5
    src, flow, logits, gout = _inputs(B, C, H, W, k, "smooth", seed=22)
    sb, lb, gb = src.bfloat16(), logits.bfloat16(), gout.bfloat16()
    ref_out, ref_gs, ref_gf, ref_gl = RC.local_attn_fwd_bwd(sb.float(), flow, lb.float(), gb.float(), k, chunk=1)
    out = F_.local_attn_fwd(sb, flow, lb, k)
    gs, gf, gl = F_.local_attn_bwd(sb, flow, lb, gb, k)
    assert out.is_contiguous() and gs.is_contiguous()
    assert (out.float() - ref_out).abs().max().item() <= 1e-2
    assert (gs.float() - ref_gs).abs().max().item() <= 1e-2
    assert (gl.float() - ref_gl).abs().max().item() <= 1e-2
    assert (gf - ref_gf).abs().max().item() <= 1e-2 * max(1.0, ref_gf.abs().max().item())


def test_cfg2_fullsize_fp32_vs_reference_cuda(RC, F_):
    """fp32 (the reference's dtype), one full-size sample: 1e-4"""
    B, C, H, W, k = 1, 256, 256, 256, 5
    src, flow, logits, gout = _inputs(B, C, H, W, k, "smooth", seed=23)
    ref_out, ref_gs, ref_gf, ref_gl = RC.local_attn_fwd_bwd(src, flow, logits, gout, k, chunk=1)
    out = F_.local_attn_fwd(src, flow, logits, k)
    gs, gf, gl = F_.local_attn_bwd(src, flow, logits, gout, k)
    assert (out - ref_out).abs().max().item() <= 1e-4
    assert (gs - ref_gs).abs().max().item() <= 1e-4 * max(1.0, ref_gs.abs().max().item())
    assert (gl - ref_gl).abs().max().item() <= 1e-4 * max(1.0, ref_gl.abs().max().item())
    assert (gf - ref_gf).abs().max().item() <= 1e-4 * max(1.0, ref_gf.abs().max().item())


def test_cfg2_one_fullsize_sample_vs_host_reference(ref_lib, F_):
    """...and one full-size sample against the HOST build of the reference bodies (all cores), forward + backward,
    tile path: closes the chain without going through any GPU-side checker"""
    import os
    from oracle.ref_pipeline import local_attn_fwd_bwd
    ref_lib.set_threads(max(1, (os.cpu_count() or 2) // 2))
    B, C, H, W, k = 1, 256, 256, 256, 5
    src, flow, logits, gout = _inputs(B, C, H, W, k, "smooth", seed=24)
    sb, lb, gb = src.bfloat16(), logits.bfloat16(), gout.bfloat16()
    r_out, _, r_gs, r_gf, r_gl = local_attn_fwd_bwd(ref_lib, sb.float().cpu().numpy(), flow.cpu().numpy(), lb.float().cpu().numpy(),
                                                    gb.float().cpu().numpy(), k)
    ref_lib.set_threads(1)
    s_cl, g_cl = sb.contiguous(memory_format=CL), gb.contiguous(memory_format=CL)
    out = F_.local_attn_fwd(s_cl, flow, lb, k, algo="tile")
    gs, gf, gl = F_.local_attn_bwd(s_cl, flow, lb, g_cl, k, algo="tile")
    t = lambda a: torch.from_numpy(a).to(DEV)
    assert (out.float() - t(r_out)).abs().max().item() <= 1e-2
    assert (gs.float() - t(r_gs)).abs().max().item() <= 1e-2
    assert (gl.float() - t(r_gl)).abs().max().item() <= 1e-2
    assert (gf - t(r_gf)).abs().max().item() <= 1e-2 * max(1.0, float(np.abs(r_gf).max()))


# ----------------------------------------------------------------------------- unfused ops at (chunks of) their BASELINE sizes
def test_block_extractor_cfg2_chunk_vs_reference_cuda(RC, F_):
    B, C, H, W, k = 1, 256, 256, 256, 5
    src, flow, _, _ = _inputs(B, C, H, W, k, "smooth", seed=25)
    ours = F_.block_extract_fwd(src, flow, k)
    ref = RC.block_extract_fwd(src, flow, k)
    assert (ours - ref).abs().max().item() <= 1e-5      # nvcc contracts the reference's mul+add chains, ours does not
    del ours, ref
    go = torch.randn(B, C, k * H, k * W, device=DEV)
    gs, gf = F_.block_extract_bwd(src, flow, go, k)
    rgs, rgf = RC.block_extract_bwd(src, flow, go, k)
    assert (gs - rgs).abs().max().item() <= 1e-4 * max(1.0, rgs.abs().max().item())
    assert (gf - rgf).abs().max().item() <= 1e-4 * max(1.0, rgf.abs().max().item())


@pytest.mark.parametrize("ks,sigma", [(2, 5.0), (4, 2.0)])
def test_resample2d_cfg3_chunk_vs_reference_cuda(RC, F_, ks, sigma):
    """cfg3 shape (C=128, 512x512 fp32), two samples: forward and both gradients vs the reference's kernels"""
    B, C, H, W = 2, 128, 512, 512
    g = torch.Generator(device="cpu").manual_seed(31)
    x = torch.randn(B, C, H, W, generator=g).to(DEV)
    go = torch.randn(B, C, H, W, generator=g).to(DEV)
    in2 = torch.cat([_smooth_flow(B, H, W, seed=3), torch.full((B, 1, H, W), sigma, device=DEV)], 1).contiguous()
    out = F_.resample2d_fwd(x, in2, ks, 1)
    ref = RC.resample2d_fwd(x, in2, ks, 1)
    assert (out - ref).abs().max().item() <= 1e-4
    g1, g2 = F_.resample2d_bwd(x, in2, go, ks, 1)
    r1, r2 = RC.resample2d_bwd(x, in2, go, ks, 1)
    assert (g1 - r1).abs().max().item() <= 1e-4 * max(1.0, r1.abs().max().item())
    assert (g2 - r2).abs().max().item() <= 1e-4 * max(1.0, r2.abs().max().item())
