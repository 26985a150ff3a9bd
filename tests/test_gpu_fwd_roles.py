"""GPU (-m gpu): the channels-last tile forward runs two warpgroups.  The pixel warpgroup writes each step's weight slab and
may run up to two steps ahead of the MMA warpgroup, also across channel passes; the MMA warpgroup loads the source
segments, multiplies, and writes `out`.  Its result must still be bit-identical to the planar tile forward, which runs
the same MMAs on the same operands in the same order with a single role.

The flow splits every 16x8 group four ways (as in test_gpu_tile_bwd_empty_steps.py): the left and right halves look about
30 columns left and right, the top and bottom halves about 20 rows up and down.  The footprint is then some 70 x 50
positions with active steps only at its four corners, so long runs of steps have no active pixel and the pixel role
runs ahead.  Some pixels get flows whose taps are not consecutive integers, so the literal path runs as well.  C covers
one 64-channel pass and one, two and four 128-channel passes; H and W are ragged."""
import numpy as np
import pytest
import torch

from test_gpu_parity import _irregular_flow_values

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
CL = torch.channels_last


@pytest.fixture(scope="module")
def F():
    import gfla_b200
    from gfla_b200 import _lib, functional
    _lib.check(_lib.lib().gfla_device_check(), "device check")
    return functional


def split_flow(B, H, W, k, rng):
    left = (np.arange(W) % 16) < 8
    top = (np.arange(H) % 8) < 4
    f = np.empty((B, 2, H, W), np.float32)
    f[:, 0] = np.where(left, -30.3, 29.6)[None, None, :]
    f[:, 1] = np.where(top, -20.4, 19.7)[None, :, None]
    f += rng.uniform(0, 0.5, (B, 2, H, W)).astype(np.float32)
    for i, (x, v) in enumerate(_irregular_flow_values(range(2, W - 2, 7), k, rng).items()):
        f[:, 0, (5 * i) % H, x] = v
    return f


def _same(a, b, what):
    a, b = a.contiguous(), b.contiguous()
    assert a.shape == b.shape, what
    diff = (a.view(torch.int16) != b.view(torch.int16)).sum().item()
    assert diff == 0, f"{what}: {diff} of {a.numel()} elements differ"


@pytest.mark.parametrize("k", [3, 5])
@pytest.mark.parametrize("C", [64, 128, 256, 512])
def test_fwd_roles_with_empty_steps_match_planar(F, C, k):
    B, Hs, Ws, H, W = 2, 67, 88, 61, 83      # ragged groups; the planar kernel needs Ws % 8 == 0
    rng = np.random.default_rng(C + k)
    f_np = split_flow(B, H, W, k, rng)
    irregular = sum(1 for x in range(W) for y in range(H)
                    if len({int(np.floor(np.float32(np.float32(f_np[0, 0, y, x] + np.float32(j - k // 2)) + np.float32(x))))
                            - j for j in range(k)}) > 1)
    assert irregular > 0
    s = torch.from_numpy(rng.standard_normal((B, C, Hs, Ws)).astype(np.float32)).to(DEV).bfloat16()
    f = torch.from_numpy(f_np).to(DEV)
    lg = torch.from_numpy((2 * rng.standard_normal((B, k * k, H, W))).astype(np.float32)).to(DEV).bfloat16()
    prev = torch.from_numpy(rng.standard_normal((B, C, H, W)).astype(np.float32)).to(DEV).bfloat16()
    mask = torch.from_numpy(rng.uniform(0, 1, (B, 1, H, W)).astype(np.float32)).to(DEV).bfloat16()
    s_cl, prev_cl = s.contiguous(memory_format=CL), prev.contiguous(memory_format=CL)

    out_cl, probs_cl = F.local_attn_fwd(s_cl, f, lg, k, return_probs=True, algo="tile")
    out, probs = F.local_attn_fwd(s, f, lg, k, return_probs=True, algo="tile")
    assert out_cl.is_contiguous(memory_format=CL)
    _same(out_cl, out, "out")
    _same(probs_cl, probs, "probs")
    _same(F.local_attn_blend_fwd(s_cl, f, lg, prev_cl, mask, k, algo="tile"),
          F.local_attn_blend_fwd(s, f, lg, prev, mask, k, algo="tile"), "blend")
    # and both agree with the gather kernel in fp64 on the same bf16 inputs, to bf16 rounding
    ref = F.local_attn_fwd(s.double(), f.double(), lg.double(), k, algo="gather")
    err = (out_cl.double() - ref).abs().max().item()
    assert err <= 2 ** -7 * ref.abs().amax().item(), err
