"""GPU (-m gpu): the tile backward over footprints with long runs of steps that no pixel of the group touches.

Every 16x8 group is split four ways: its left and right halves look about 30 columns left and right, its top and bottom
halves about 20 rows up and down.  The group's footprint is then some 70 x 50 positions with active steps only at its
four corners, so most steps have no active pixel and several follow each other.  The pixel warpgroup scatters nothing
in them and may run up to two steps ahead of the grad_source warpgroup, which skips them.  The three gradients must still
match an fp64 evaluation of the same bf16 inputs, in one channel pass (C = 64) and in two (C = 512), in both the default
and the deterministic backward.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
CL = torch.channels_last


@pytest.fixture(scope="module")
def F():
    import gfla_b200
    from gfla_b200 import _lib, functional
    _lib.check(_lib.lib().gfla_device_check(), "device check")
    return functional


def split_flow_inputs(B, C, S, k, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    left = (torch.arange(S) % 16) < 8
    top = (torch.arange(S) % 8) < 4
    f = torch.empty(B, 2, S, S)
    f[:, 0] = torch.where(left, -30.3, 29.6)[None, None, :]
    f[:, 1] = torch.where(top, -20.4, 19.7)[None, :, None]
    f += torch.rand(B, 2, S, S, generator=g) * 0.5
    s = torch.randn(B, C, S, S, generator=g)
    lg = torch.randn(B, k * k, S, S, generator=g)
    go = torch.randn(B, C, S, S, generator=g)
    bf = torch.bfloat16
    return (s.to(DEV, bf).contiguous(memory_format=CL), f.to(DEV), lg.to(DEV, bf), go.to(DEV, bf).contiguous(memory_format=CL))


@pytest.mark.parametrize("deterministic", [False, True], ids=["default", "det"])
@pytest.mark.parametrize("C", [64, 512])
@pytest.mark.parametrize("k", [3, 5])
def test_tile_backward_with_empty_steps_matches_fp64(F, k, C, deterministic):
    args = split_flow_inputs(2, C, 96, k, seed=k * C)
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(deterministic)
    try:
        got = F.local_attn_bwd(*args, k, algo="tile")
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)
    ref = F.local_attn_bwd(*[t.double().contiguous() for t in args], k, algo="gather")
    for name, x, r in zip(("grad_source", "grad_flow", "grad_logits"), got, ref):
        err = (x.double() - r).abs().max().item()
        scale = r.abs().amax().item()
        assert scale > 0 and err <= 2 ** -7 * scale, (name, err, scale)
