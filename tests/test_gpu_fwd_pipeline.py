"""GPU (-m gpu): the channels-last tile forward walks 32-position steps and streams its source segments through a ring
that runs several steps ahead and crosses 64-channel pass boundaries.  The planar tile forward walks 16-position steps
and loads one step ahead, pass by pass.  Both run the same MMAs on the same operands in the same order, so `out`,
`probs` and the mask blend must agree bit for bit.

The cases cover 1, 2, 4 and 8 passes, ragged pixel groups, the flow families of the other tile tests, and footprints
shorter than the ring: every window folded onto one corner position (one step per pass) and a source two rows high
(at most two steps per pass)."""
import numpy as np
import pytest
import torch

from test_ref64 import make_flow

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


@pytest.fixture(scope="module")
def F_():
    import gfla_b200
    from gfla_b200 import _lib
    _lib.check(_lib.lib().gfla_device_check(), "device check")
    return gfla_b200.functional


def _flow(kind, rng, B, H, W, k):
    if kind == "corner_tl":     # every window wholly above and left of the image: folded onto position (0, 0)
        return np.stack([np.full((B, H, W), -(W + 40.0)), np.full((B, H, W), -(H + 40.0))], 1).astype(np.float32) \
            + rng.uniform(-0.5, 0.5, (B, 2, H, W)).astype(np.float32)
    if kind == "corner_br":     # every window wholly below and right of the image: folded onto (Hs - 1, Ws - 1)
        return np.stack([np.full((B, H, W), W + 40.0), np.full((B, H, W), H + 40.0)], 1).astype(np.float32) \
            + rng.uniform(-0.5, 0.5, (B, 2, H, W)).astype(np.float32)
    return make_flow(kind, rng, B, H, W, k)


def _inputs(B, C, Hs, Ws, H, W, k, kind, seed):
    rng = np.random.default_rng(seed)
    s = torch.from_numpy(rng.standard_normal((B, C, Hs, Ws)).astype(np.float32)).to(DEV).bfloat16()
    f = torch.from_numpy(np.ascontiguousarray(_flow(kind, rng, B, H, W, k), dtype=np.float32)).to(DEV)
    lg = torch.from_numpy((2 * rng.standard_normal((B, k * k, H, W))).astype(np.float32)).to(DEV).bfloat16()
    prev = torch.from_numpy(rng.standard_normal((B, C, H, W)).astype(np.float32)).to(DEV).bfloat16()
    mask = torch.from_numpy(rng.uniform(0, 1, (B, 1, H, W)).astype(np.float32)).to(DEV).bfloat16()
    return s, f, lg, prev, mask


def _same(a, b, what):
    a, b = a.contiguous(), b.contiguous()
    assert a.shape == b.shape, what
    diff = (a.view(torch.int16) != b.view(torch.int16)).sum().item()
    assert diff == 0, f"{what}: {diff} of {a.numel()} elements differ"


def _check(F_, B, C, Hs, Ws, H, W, k, kind, seed):
    s, f, lg, prev, mask = _inputs(B, C, Hs, Ws, H, W, k, kind, seed)
    s_cl, prev_cl = s.contiguous(memory_format=torch.channels_last), prev.contiguous(memory_format=torch.channels_last)
    out_cl, probs_cl = F_.local_attn_fwd(s_cl, f, lg, k, return_probs=True, algo="tile")
    out, probs = F_.local_attn_fwd(s, f, lg, k, return_probs=True, algo="tile")
    assert out_cl.is_contiguous(memory_format=torch.channels_last)
    _same(out_cl, out, "out")
    _same(probs_cl, probs, "probs")
    blend_cl = F_.local_attn_blend_fwd(s_cl, f, lg, prev_cl, mask, k, algo="tile")
    blend = F_.local_attn_blend_fwd(s, f, lg, prev, mask, k, algo="tile")
    _same(blend_cl, blend, "blend")


FLOWS = ["smooth", "iid", "border", "outside", "span3", "irregular", "corner_tl", "corner_br"]
SHAPES = [                          # B, C, Hs, Ws, H, W: ragged H and W, the planar kernel needs Ws % 8 == 0
    (2, 64, 21, 40, 19, 37),        # one pass
    (1, 128, 24, 48, 23, 45),       # two passes
    (1, 256, 19, 32, 21, 33),       # four passes
    (1, 512, 17, 40, 16, 27),       # eight passes
]


@pytest.mark.parametrize("k", [3, 5])
@pytest.mark.parametrize("kind", FLOWS)
@pytest.mark.parametrize("shape", SHAPES)
def test_fwd_pipeline_matches_planar(F_, shape, kind, k):
    _check(F_, *shape, k, kind, seed=sum(shape) + 11 * k + len(kind))


@pytest.mark.parametrize("k", [3, 5])
@pytest.mark.parametrize("kind", ["smooth", "iid", "border"])
@pytest.mark.parametrize("C", [64, 128, 256, 512])
def test_fwd_pipeline_two_row_source(F_, C, kind, k):
    """a 2 x 16 source: every footprint is one segment wide and at most two rows high"""
    _check(F_, 2, C, 2, 16, 13, 21, k, kind, seed=C + 5 * k + len(kind))
