"""GPU (-m gpu): the tile kernels skip the MMA tiles of 16-pixel group rows whose windows miss the current source row
segment, and the backward skips steps no pixel of the group touches.  These flows make that per-row activity differ
inside one 16x8 pixel group, so that partially skipped steps are common; tile results must still match the gather
kernel and the oracle at the tolerances of the other tile tests."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def host(t):
    a = t.detach().float().cpu().numpy() if t.dtype in (torch.bfloat16, torch.float16) else t.detach().cpu().numpy()
    return np.ascontiguousarray(a)


@pytest.fixture(scope="module")
def F_():
    import gfla_b200
    from gfla_b200 import _lib
    _lib.check(_lib.lib().gfla_device_check(), "device check")
    return gfla_b200.functional


def _mask_flow(kind, rng, B, H, W):
    ys, xs = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    fx = rng.uniform(-0.5, 0.5, (B, H, W))
    fy = rng.uniform(-0.5, 0.5, (B, H, W))
    if kind == "rows":        # every pixel row of a group looks at a different source row band
        fy += ((ys % 8) * 3.1 - 11.0)[None]
    elif kind == "halves":    # left and right halves of a group point 8 px apart
        fx += np.where(xs % 16 < 8, -4.0, 4.0)[None]
    elif kind == "outside":   # some windows lie wholly outside the image (left, top, right), folded onto the border
        # (few per group: every group adds its share of a border position with one rounding bf16 atomic add)
        fx += np.where(xs % 16 < 2, -(W + 9.0), np.where(xs % 16 > 13, W + 7.5, 0.0))[None]
        fy += np.where(ys % 8 == 0, -(H + 6.0), 0.0)[None]
    elif kind == "span3":     # one group's footprint spans three 16-position segments
        fx += ((xs % 16) - 8) * 2.3
        fy += ((ys % 8) - 4) * 0.7
    return np.stack([fx, fy], axis=1).astype(np.float32)


def _inputs(B, C, Hs, Ws, H, W, k, kind, seed):
    rng = np.random.default_rng(seed)
    s = torch.from_numpy(rng.standard_normal((B, C, Hs, Ws)).astype(np.float32)).to(DEV).bfloat16()
    s = s.contiguous(memory_format=torch.channels_last)
    f = torch.from_numpy(_mask_flow(kind, rng, B, H, W)).to(DEV)
    l = torch.from_numpy((2 * rng.standard_normal((B, k * k, H, W))).astype(np.float32)).to(DEV).bfloat16()
    g = torch.from_numpy(rng.standard_normal((B, C, H, W)).astype(np.float32)).to(DEV).bfloat16()
    return s, f, l, g.contiguous(memory_format=torch.channels_last)


KINDS = ["rows", "halves", "outside", "span3"]
SHAPES = [                          # B, C, Hs, Ws, H, W
    (2, 64, 21, 37, 21, 37),        # ragged H and W
    (1, 128, 24, 40, 24, 40),
    (1, 256, 19, 45, 19, 45),
    (1, 512, 16, 33, 16, 33),       # two passes of 256 channels: Q accumulates across passes
    (1, 64, 26, 40, 19, 27),        # source larger than the flow field
]


def _check_bwd(gs, gf, gl, ogs, ogf, ogl):
    np.testing.assert_allclose(host(gs), ogs, rtol=0, atol=1e-2 * max(1.0, float(np.abs(ogs).max())))
    np.testing.assert_allclose(host(gl), ogl, rtol=0, atol=1e-2)
    np.testing.assert_allclose(host(gf), ogf, rtol=2e-2, atol=2e-2 * max(1.0, float(np.abs(ogf).max())))


@pytest.mark.parametrize("k", [3, 5])
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("shape", SHAPES)
def test_tile_masks_fwd(F_, oracle_lib, shape, kind, k):
    B, C, Hs, Ws, H, W = shape
    s, f, l, _ = _inputs(B, C, Hs, Ws, H, W, k, kind, seed=sum(shape) + 7 * k + len(kind))
    ref = oracle_lib.local_attn_fwd(host(s), f.cpu().numpy(), host(l), k)
    gather = F_.local_attn_fwd(s, f, l, k, algo="gather")
    for layout in ("nhwc", "nchw") if Ws % 8 == 0 else ("nhwc",):     # the planar tile kernel needs Ws % 8 == 0
        src = s if layout == "nhwc" else s.contiguous()
        out = F_.local_attn_fwd(src, f, l, k, algo="tile")
        np.testing.assert_allclose(host(out), ref, rtol=0, atol=1e-2)
        err = (out.float() - gather.float()).abs().max().item()
        assert err <= 3e-3, (layout, err)


@pytest.mark.parametrize("k", [3, 5])
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("shape", SHAPES)
def test_tile_masks_bwd(F_, oracle_lib, shape, kind, k):
    B, C, Hs, Ws, H, W = shape
    s, f, l, g = _inputs(B, C, Hs, Ws, H, W, k, kind, seed=3 * sum(shape) + k + len(kind))
    ogs, ogf, ogl = oracle_lib.local_attn_bwd(host(s), f.cpu().numpy(), host(l), host(g), k)
    gs, gf, gl = F_.local_attn_bwd(s, f, l, g, k, algo="tile")
    _check_bwd(gs, gf, gl, ogs, ogf, ogl)
    _check_bwd(*F_.local_attn_bwd(s, f, l, g, k, algo="gather"), ogs, ogf, ogl)


@pytest.mark.parametrize("k", [3, 5])
@pytest.mark.parametrize("kind", ["halves", "span3"])
def test_tile_masks_bwd_accumulate(F_, oracle_lib, kind, k):
    """accumulate = 1: every gradient is added into what the caller's buffers hold"""
    from gfla_b200 import _lib
    from gfla_b200.functional import ALGO, _dt, _p, _stream
    B, C, Hs, Ws, H, W = 1, 256, 19, 45, 19, 45
    s, f, l, g = _inputs(B, C, Hs, Ws, H, W, k, kind, seed=101 + k)
    gs = torch.full(s.shape, 0.5, device=DEV, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
    gf = torch.full(f.shape, -0.25, device=DEV, dtype=torch.float32)
    gl = torch.full(l.shape, 0.125, device=DEV, dtype=torch.bfloat16)
    _lib.check(_lib.lib().gfla_local_attn_bwd(_p(s), _p(f), _p(l), _p(g), _p(gs), _p(gf), _p(gl), B, C, Hs, Ws, H, W, k,
                                              _dt(s), _dt(f), _lib.GFLA_NHWC, 1, ALGO["tile"], _stream(s)), "local_attn_bwd")
    ogs, ogf, ogl = oracle_lib.local_attn_bwd(host(s), f.cpu().numpy(), host(l), host(g), k)
    _check_bwd(gs, gf, gl, ogs + 0.5, ogf - 0.25, ogl + 0.125)
