"""CPU: the deterministic backward mode (csrc/det_accum.cuh), without a device.

  * the *_det entry points reject a NULL, misaligned or too small workspace before launching anything, and their
    workspace queries match the documented layout;
  * a numpy emulation of the per-image 64-bit fixed-point scatter (exponent rule of det_accum.cu) is bit-identical under
    any order of the partials and within its error bound, also at the extreme of R4 (every window folded onto one
    corner with |G| at the largest finite bf16);
  * injected faults fail: an exponent two above the proved one wraps int64, one exponent per tensor breaks the
    per-image property, a dropped partial and bf16-rounded partials break the bound.
"""
import ctypes
import math

import numpy as np
import pytest

BF16_MAX = float(np.float32(3.3895313892515355e38))


@pytest.fixture(scope="module")
def so():
    import __graft_entry__ as ge
    ge.build_cuda()
    import gfla_b200
    return gfla_b200._lib.lib()


# ------------------------------------------------------------------------------------------------------ ABI
def _rnd(b):
    return (b + 255) // 256 * 256


def test_workspace_queries(so):
    B, C, Hs, Ws, H, W, k = 2, 64, 9, 7, 5, 6, 3
    assert so.gfla_local_attn_bwd_det_workspace_bytes(B, C, Hs, Ws, H, W, k) == _rnd(8 * B * C * Hs * Ws) + _rnd(4 * B) + _rnd(8 * B)
    assert so.gfla_block_extract_bwd_det_workspace_bytes(B, C, Hs, Ws, H, W, k) == _rnd(8 * B * C * Hs * Ws) + _rnd(4 * B) + _rnd(8 * B)
    n = B * Hs * Ws * C + 128 * k * k * C
    assert so.gfla_patch_conv_bwd_det_workspace_bytes(B, C, Hs, Ws, H, W, k, 128) == _rnd(8 * n) + _rnd(4 * (B + 1)) + _rnd(8 * (B + 2))
    assert so.gfla_local_attn_bwd_det_workspace_bytes(0, C, Hs, Ws, H, W, k) == -2
    assert so.gfla_block_extract_bwd_det_workspace_bytes(B, C, Hs, Ws, H, W, 10) == -2


def test_det_entry_points_validate_the_workspace(so):
    launches = so.gfla_debug_launch_count()
    buf = (ctypes.c_double * 4096)()
    p = ctypes.addressof(buf)          # 16-byte aligned host memory: nothing may be launched on it
    assert p % 16 == 0
    B, C, Hs, Ws, H, W, k = 1, 2, 4, 4, 4, 4, 3
    need = so.gfla_local_attn_bwd_det_workspace_bytes(B, C, Hs, Ws, H, W, k)
    la = lambda ws, nb: so.gfla_local_attn_bwd_det(p, p, p, p, p, p, p, B, C, Hs, Ws, H, W, k, 0, 0, 0, 0, 0, ws, nb, None)
    assert la(None, need) == -1
    assert la(p + 8, need) == -4
    assert la(p, need - 1) == -2
    need = so.gfla_block_extract_bwd_det_workspace_bytes(B, C, Hs, Ws, H, W, k)
    be = lambda ws, nb: so.gfla_block_extract_bwd_det(p, p, p, p, p, B, C, Hs, Ws, H, W, k, 0, 0, 0, ws, nb, None)
    assert be(None, need) == -1
    assert be(p + 4, need) == -4
    assert be(p, 0) == -2
    C = 64
    need = so.gfla_patch_conv_bwd_det_workspace_bytes(B, C, Hs, Ws, H, W, k, 128)
    pc = lambda ws, nb: so.gfla_patch_conv_bwd_det(p, p, p, p, p, p, p, B, C, Hs, Ws, H, W, k, 128, 2, 0, 1, 0, ws, nb, None)
    assert pc(None, need) == -1
    assert pc(p, need - 16) == -2
    # the other argument checks come first, as in the default entry points
    assert so.gfla_local_attn_bwd_det(None, p, p, p, p, p, p, B, C, Hs, Ws, H, W, k, 0, 0, 0, 0, 0, p, 1 << 20, None) == -1
    assert so.gfla_local_attn_bwd_det(p, p, p, p, p, p, p, B, C, Hs, Ws, H, W, k, 7, 0, 0, 0, 0, p, 1 << 20, None) == -3
    assert so.gfla_debug_launch_count() == launches          # nothing was launched


# ------------------------------------------------------------------------------------------------------ emulation
def exponent(m):
    """det_accum.cu fx_exponent: 61 - e with m < 2^e (0 for m == 0)"""
    if m == 0:
        return 0
    return 61 - math.frexp(m)[1]


def fx_sum(idx, partials, n_out, e):
    """int64 fixed-point sum of fp32 partials at idx (numpy int64 adds wrap like red.global.add.u64)"""
    q = np.rint(partials.astype(np.float64) * 2.0 ** e).astype(np.int64)
    out = np.zeros(n_out, np.int64)
    with np.errstate(over="ignore"):
        np.add.at(out, idx, q)
    return out


def narrow(s, e):
    return (s.astype(np.float64) * 2.0 ** -e).astype(np.float32)


def scatter_partials(rng, H, W, Hs, Ws, k, g, flow):
    """the gather backward's partials g * p_ij * w_bilinear / k^2 of one channel of one image, in fp32, with their source
    positions: per pixel, softmax probabilities times bilinear weights times 1/k^2 sum to 1/k^2"""
    logits = rng.standard_normal((k * k, H, W)).astype(np.float32)
    p = np.exp(logits - logits.max(0))
    p = (p / p.sum(0)).astype(np.float32)
    idx, val = [], []
    ys, xs = np.mgrid[0:H, 0:W]
    for i in range(k):
        for j in range(k):
            dy = (flow[1] + np.float32(i - k // 2)) + ys.astype(np.float32)
            dx = (flow[0] + np.float32(j - k // 2)) + xs.astype(np.float32)
            fy, fx = np.floor(dy), np.floor(dx)
            wy1, wx1 = (dy - fy).astype(np.float32), (dx - fx).astype(np.float32)
            wy0, wx0 = np.float32(1) - wy1, np.float32(1) - wx1
            for wy, yy in ((wy0, fy), (wy1, fy + 1)):
                for wx, xx in ((wx0, fx), (wx1, fx + 1)):
                    pos = np.clip(yy, 0, Hs - 1).astype(np.int64) * Ws + np.clip(xx, 0, Ws - 1).astype(np.int64)
                    idx.append(pos.ravel())
                    val.append((g * p[i * k + j] * (wy * wx) / np.float32(k * k)).astype(np.float32).ravel())
    return np.concatenate(idx), np.concatenate(val)


def bound(idx, val, n_out, e):
    """per element: the fp64 sum's u_fp32 |r| for the one final rounding, n_partials 2^-(E+1) for the quantisation,
    2^-53 |r| for int64 -> double, plus 2^-24 per partial magnitude for the fp32 partials themselves"""
    ref = np.zeros(n_out)
    np.add.at(ref, idx, val.astype(np.float64))
    absum = np.zeros(n_out)
    np.add.at(absum, idx, np.abs(val.astype(np.float64)))
    cnt = np.bincount(idx, minlength=n_out)
    return ref, 2.0 ** -24 * np.abs(ref) + cnt * 2.0 ** -(e + 1) + 2.0 ** -53 * np.abs(ref) + 2.0 ** -23 * absum


def _flow(kind, rng, H, W):
    if kind == "smooth":
        return (rng.standard_normal((2, H, W)) * 3).astype(np.float32)
    if kind == "corner":
        return np.full((2, H, W), -1e4, np.float32)
    return (rng.standard_normal((2, H, W)) * 2 + 1e-7).astype(np.float32)       # irregular taps


@pytest.mark.parametrize("kind", ["smooth", "corner", "irregular"])
@pytest.mark.parametrize("k", [3, 5])
def test_emulated_fixed_point_is_order_free_and_within_bound(k, kind):
    rng = np.random.default_rng(k)
    H, W = 24, 40
    g = rng.standard_normal((H, W)).astype(np.float32)
    idx, val = scatter_partials(rng, H, W, H, W, k, g, _flow(kind, rng, H, W))
    e = exponent(H * W / k ** 2 * float(np.abs(g).max()))
    s = fx_sum(idx, val, H * W, e)
    perm = rng.permutation(len(idx))
    assert np.array_equal(s, fx_sum(idx[perm], val[perm], H * W, e))
    ref, b = bound(idx, val, H * W, e)
    assert (np.abs(narrow(s, e) - ref) <= b).all()
    # fault: a dropped partial
    d = fx_sum(idx[1:], val[1:], H * W, e)
    assert not (np.abs(narrow(d, e) - ref) <= b).all()
    # fault: partials rounded to bf16 first (the default tile path's scheme)
    v16 = (val.view(np.uint32) + 0x7fff + ((val.view(np.uint32) >> 16) & 1)) & 0xffff0000
    s16 = fx_sum(idx, v16.view(np.float32), H * W, e)
    assert not (np.abs(narrow(s16, e) - ref) <= b).all()


def test_extreme_corner_pileup_stays_in_range():
    """R4: every window of a 64x64 image folded onto the top-left corner, |G| the largest finite bf16"""
    rng = np.random.default_rng(0)
    H = W = 64
    k = 5
    g = np.full((H, W), BF16_MAX, np.float32)
    idx, val = scatter_partials(rng, H, W, H, W, k, g, _flow("corner", rng, H, W))
    e = exponent(H * W / k ** 2 * BF16_MAX)
    s = fx_sum(idx, val, H * W, e)
    assert abs(int(s[0])) < 2 ** 62
    ref, b = bound(idx, val, H * W, e)
    # the corner's true sum (~5.6e40) is past the fp32 range, so judge the sum before the final rounding
    wide = lambda x, ex: x.astype(np.float64) * 2.0 ** -ex
    assert (np.abs(wide(s, e) - ref) <= b).all()
    # fault: an exponent two larger than the bound allows wraps the int64 sum.  The bound allows 62 - e (|sum| < 2^62);
    # the exponent used keeps one more bit of margin for the fp32 rounding of the partials, so that is e + 3 here.
    w = fx_sum(idx, val, H * W, e + 3)
    assert int(w[0]) < 0
    assert not (np.abs(wide(w, e + 3) - ref) <= b).all()


def test_per_tensor_exponent_breaks_per_image_results():
    """a batch of two images whose gradients differ in scale by 2^20: with per-image exponents image 0's sum is the same
    alone and in the batch; with one exponent for the whole batch (taken from its largest image) it is not"""
    H = W = 16
    k = 3
    rng = np.random.default_rng(1)
    flows = [_flow("smooth", rng, H, W) for _ in range(2)]
    gs = [rng.standard_normal((H, W)).astype(np.float32), (rng.standard_normal((H, W)) * 2.0 ** 20).astype(np.float32)]
    parts = [scatter_partials(np.random.default_rng(2 + b), H, W, H, W, k, gs[b], flows[b]) for b in range(2)]
    M = [H * W / k ** 2 * float(np.abs(g).max()) for g in gs]

    def batch(E):
        """the batch's sums, image b at offset b H W, image b quantised with exponent E[b]"""
        idx = np.concatenate([parts[b][0] + b * H * W for b in range(2)])
        out = np.zeros(2 * H * W, np.int64)
        for b in range(2):
            q = np.rint(parts[b][1].astype(np.float64) * 2.0 ** E[b]).astype(np.int64)
            np.add.at(out, parts[b][0] + b * H * W, q)
        del idx
        return [narrow(out[b * H * W:(b + 1) * H * W], E[b]) for b in range(2)]

    alone = narrow(fx_sum(parts[0][0], parts[0][1], H * W, exponent(M[0])), exponent(M[0]))
    per_image = batch([exponent(M[0]), exponent(M[1])])
    assert np.array_equal(alone, per_image[0])
    e_tensor = exponent(max(M))
    per_tensor = batch([e_tensor, e_tensor])
    assert not np.array_equal(alone, per_tensor[0])
