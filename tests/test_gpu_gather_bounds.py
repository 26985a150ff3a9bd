"""GPU (-m gpu): the CUDA-core kernels in fp32 and fp64 -- gather local attention (csrc/local_attn.cu) and block_extractor
(csrc/block_extract.cu) -- against the fp64 reference (ref64_gather), element by element, with bounds derived from what
each kernel rounds (DESIGN.md section 6), at every kernel size 1..9; local_attn_reshape and the NCHW <-> channels-last
relayout bit for bit.  The case lists cover one channel slice, several, and a ragged last slice of the forward, and both
grad_flow paths of the block_extractor backward, asserted through ref64_gather's mirror of channel_splits; the relayout
cases take both of its kernels, asserted through a mirror of its choice and confirmed by a profile in a fresh process."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import ref64
import ref64_gather as rg
from test_ref64_gather import LOGITS, make_flow, make_logits

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
DTYPES = {"fp32": np.float32, "fp64": np.float64}
WORST = {}
PATHS = set()


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def host(t):
    return np.ascontiguousarray(t.detach().double().cpu().numpy())


def within(row, y, ref, bound, **mags):
    r = ref64.assert_within(row, host(y) if torch.is_tensor(y) else y, ref, bound, **mags)
    WORST[row] = max(WORST.get(row, 0.0), r)


@pytest.fixture(scope="module", autouse=True)
def worst_ratios():
    yield
    print("\nlargest |err|/bound per output and path:")
    for row in sorted(WORST):
        print(f"  {row:52s} {WORST[row]:.3f}")
    print("launch paths run:", "; ".join(sorted(PATHS)))


@pytest.fixture(scope="module")
def F_():
    import gfla_b200
    from gfla_b200 import _lib
    _lib.check(_lib.lib().gfla_device_check(), "device check")
    return gfla_b200.functional


def sm_count():
    """what sm_count() (common.cuh:82-95) launches with"""
    v = int(os.environ.get("GFLA_SM_COUNT", "0") or 0)
    return v if v > 0 else torch.cuda.get_device_properties(0).multi_processor_count


def fwd_slicing(B, C, H, W):
    slices, cps = rg.launch_slices(B * H * W, C, 128, sm_count())
    return "one slice" if slices == 1 else ("ragged last slice" if C % cps else "full slices")


# --------------------------------------------------------------------------------------------- local attention
KINDS = ["smooth", "iid", "border", "zero", "int", "outside", "span3", "irregular"]
SHAPES = [                                  # B, C, Hs, Ws, H, W
    (2, 1, 13, 19, 13, 19),                 # C = 1: one channel slice; ragged H, W
    (1, 3, 17, 23, 11, 14),                 # source larger than the flow field; two slices, the last ragged
    (2, 48, 9, 11, 12, 15),                 # source smaller; full slices
    (1, 130, 11, 14, 11, 14),               # ragged last slice (43 x 3 + 1 channels)
]


def test_cases_cover_every_slicing():
    assert {fwd_slicing(B, C, H, W) for B, C, Hs, Ws, H, W in SHAPES} == {"one slice", "full slices",
                                                                          "ragged last slice"}


def la_inputs(dt, k, i, kind):
    A = DTYPES[dt]
    B, C, Hs, Ws, H, W = SHAPES[(i + k) % len(SHAPES)]
    rng = np.random.default_rng(1000 * k + 10 * i + len(dt))
    s = rng.standard_normal((B, C, Hs, Ws)).astype(A)
    f = make_flow(kind, rng, B, H, W, k, A).astype(A)
    lg = make_logits(LOGITS[(i + 2 * k) % 3], rng, B, k, H, W).astype(A)
    g = rng.standard_normal((B, C, H, W)).astype(A)
    return s, f, lg, g, rng


def layouts(t):
    return {"nchw": t, "nhwc": t.contiguous(memory_format=torch.channels_last)}


@pytest.mark.parametrize("k", range(1, 10))
@pytest.mark.parametrize("dt", sorted(DTYPES))
def test_local_attn_gather_within_bounds(F_, dt, k):
    for i, kind in enumerate(KINDS):
        s, f, lg, g, rng = la_inputs(dt, k, i, kind)
        B, C, Hs, Ws = s.shape
        H, W = f.shape[2:]
        la = rg.LocalAttn(f, lg, k, Hs, Ws, DTYPES[dt])
        if kind == "irregular" and k > 1:
            assert not la.taps.regular.all()
        r, mags = la.fwd(s)
        rb_in = rng.standard_normal((B, C, H, W)).astype(s.dtype), rng.uniform(0, 1, (B, 1, H, W)).astype(s.dtype)
        rb, Mb = ref64.blend_ref(r, mags["M"], *(x.astype(np.float64) for x in rb_in))
        bb = la.bound_blend(rb, mags, *(x.astype(np.float64) for x in rb_in))
        rr = la.bwd(s, g)
        sl = fwd_slicing(B, C, H, W)
        PATHS.add(f"forward C={C}: {sl}")
        tf, tl = cu(f), cu(lg)
        for lay, ts in layouts(cu(s)).items():
            out, probs = F_.local_attn_fwd(ts, tf, tl, k, return_probs=True, algo="gather")
            within(f"out {dt} {lay}", out, r, la.bound_out(mags), M=mags["M"], MR=mags["MR"])
            within(f"probs {dt}", probs, la.probs(), la.bound_probs(), L=la.L)
            prev = layouts(cu(rb_in[0]))[lay]
            blend = F_.local_attn_blend_fwd(ts, tf, tl, prev, cu(rb_in[1]), k, algo="gather")
            within(f"blend {dt} {lay}", blend, rb, bb, M=Mb)
            gs, gf, gl = F_.local_attn_bwd(ts, tf, tl, layouts(cu(g))[lay], k, algo="gather")
            within(f"grad_source {dt} {lay}", gs, rr["gs"], la.bound_gs(rr), Mgs=rr["Mgs"], m=la.m)
            within(f"grad_logits {dt} {lay}", gl, rr["gl"], la.bound_gl(rr, C), D=rr["D"], PD=rr["PD"])
            within(f"grad_flow {dt} {lay}", gf, rr["gf"], la.bound_gf(rr, C), Mgf=rr["Mgf"])


@pytest.mark.parametrize("k", range(1, 10))
@pytest.mark.parametrize("dt", sorted(DTYPES))
def test_local_attn_gather_accumulate(F_, dt, k):
    """accumulate = 1 through the C ABI (gfla_local_attn_bwd, gather kernel): the gradients are added into what the
    buffers hold"""
    from gfla_b200 import _lib
    from gfla_b200.functional import ALGO, _dt, _p, _stream
    i = k % len(KINDS)
    s, f, lg, g, rng = la_inputs(dt, k, i, KINDS[i])
    B, C, Hs, Ws = s.shape
    H, W = f.shape[2:]
    la = rg.LocalAttn(f, lg, k, Hs, Ws, DTYPES[dt])
    rr = la.bwd(s, g)
    init = [rng.standard_normal(a.shape).astype(s.dtype) for a in (s, f, lg)]
    for lay, code in (("nchw", _lib.GFLA_NCHW), ("nhwc", _lib.GFLA_NHWC)):
        ts, tg = layouts(cu(s))[lay], layouts(cu(g))[lay]
        gs, gf, gl = layouts(cu(init[0]))[lay].clone(memory_format=torch.preserve_format), cu(init[1]), cu(init[2])
        tf, tl = cu(f), cu(lg)
        _lib.check(_lib.lib().gfla_local_attn_bwd(_p(ts), _p(tf), _p(tl), _p(tg), _p(gs), _p(gf), _p(gl), B, C, Hs, Ws, H, W,
                                                  k, _dt(ts), _dt(tf), code, 1, ALGO["gather"], _stream(ts)),
                   "local_attn_bwd")
        i0, i1, i2 = (a.astype(np.float64) for a in init)
        within(f"grad_source {dt} accumulate", gs, rr["gs"] + i0, la.bound_gs(rr, i0))
        within(f"grad_logits {dt} accumulate", gl, rr["gl"] + i2, la.bound_gl(rr, C, i2))
        within(f"grad_flow {dt} accumulate", gf, rr["gf"] + i1, la.bound_gf(rr, C, i1))


# ------------------------------------------------------------------------------------------------ block_extractor
BE_SHAPES = [(2, 1, 13, 17, 11, 15), (2, 5, 9, 11, 12, 14)]    # C = 1: one slice (read-modify-write); C = 5: atomics
BE_KINDS = ["smooth", "iid", "border", "irregular"]


@pytest.mark.parametrize("k", range(1, 10))
@pytest.mark.parametrize("dt", sorted(DTYPES))
def test_block_extract_within_bounds(F_, oracle_lib, dt, k):
    A = DTYPES[dt]
    for i, kind in enumerate(BE_KINDS):
        B, C, Hs, Ws, H, W = BE_SHAPES[(i + k) % 2]
        rng = np.random.default_rng(100 * k + i + len(dt))
        s = rng.standard_normal((B, C, Hs, Ws)).astype(A)
        f = make_flow(kind, rng, B, H, W, k, A).astype(A)
        g = rng.standard_normal((B, C, k * H, k * W)).astype(A)
        ts, tf, tg = cu(s), cu(f), cu(g)
        assert np.array_equal(F_.block_extract_fwd(ts, tf, k).cpu().numpy(), oracle_lib.block_extract_fwd(s, f, k))
        be = rg.BlockExtract(s, f, k, g, A)
        slices = rg.launch_slices(B * H * W, C, 128, sm_count())[0]
        path = "read-modify-write" if slices == 1 else "atomic"
        assert (slices == 1) == (C == 1), (C, slices)
        PATHS.add(f"block_extract grad_flow C={C}: {path} ({slices} slices)")
        gs, gf = F_.block_extract_bwd(ts, tf, tg, k)
        within(f"block_extract grad_source {dt}", gs, be.r["gs"], be.bound_gs(), Mgs=be.r["Mgs"], m=be.m)
        within(f"block_extract grad_flow {dt} {path}", gf, be.r["gf"], be.bound_gf(), Mgf=be.r["Mgf"])
        # the legacy contract (block_extractor.py:35-40): the backward adds into the caller's buffers
        i0, i1 = rng.standard_normal(s.shape).astype(A), rng.standard_normal(f.shape).astype(A)
        gs, gf = F_.block_extract_bwd(ts, tf, tg, k, cu(i0), cu(i1))
        i0, i1 = i0.astype(np.float64), i1.astype(np.float64)
        within(f"block_extract grad_source {dt} accumulate", gs, be.r["gs"] + i0, be.bound_gs(i0))
        within(f"block_extract grad_flow {dt} {path} accumulate", gf, be.r["gf"] + i1, be.bound_gf(i1))


# ------------------------------------------------------------------------------------------- local_attn_reshape
ALL = {"fp32": torch.float32, "fp64": torch.float64, "bf16": torch.bfloat16, "fp16": torch.float16}


def round_to(x32, dt):
    """the A-typed sum rounded once into dt (as st(): RNE)"""
    if dt == "bf16":
        return ref64.round_bf16(x32)
    if dt == "fp16":
        return np.asarray(x32, np.float32).astype(np.float16).astype(np.float64)
    return np.asarray(x32, np.float64)


@pytest.mark.parametrize("k", range(1, 10))
@pytest.mark.parametrize("dt", sorted(ALL))
def test_attn_reshape_permutation(F_, dt, k):
    """forward and backward are numpy's permutation bit for bit; accumulate = 1 adds in A (fp64 for fp64, else fp32) and
    rounds once"""
    B, H, W = 2, 5, 7
    rng = np.random.default_rng(k + len(dt))
    x = torch.from_numpy(rng.standard_normal((B, k * k, H, W))).to(DEV).to(ALL[dt])
    xh = host(x)
    perm = xh.reshape(B, k, k, H, W).transpose(0, 3, 1, 4, 2).reshape(B, 1, k * H, k * W)
    assert np.array_equal(host(F_.attn_reshape_fwd(x, k)), perm)
    go = torch.from_numpy(rng.standard_normal((B, 1, k * H, k * W))).to(DEV).to(ALL[dt])
    back = host(go).reshape(B, H, k, W, k).transpose(0, 2, 4, 1, 3).reshape(B, k * k, H, W)
    assert np.array_equal(host(F_.attn_reshape_bwd(go, k)), back)
    init = torch.from_numpy(rng.standard_normal((B, k * k, H, W))).to(DEV).to(ALL[dt])
    A = np.float64 if dt == "fp64" else np.float32
    want = round_to(host(init).astype(A) + back.astype(A), dt)
    got = F_.attn_reshape_bwd(go, k, grad_in=init.clone())
    assert np.array_equal(host(got), want)


# ------------------------------------------------------------------------------------------------------ relayout
RELAYOUT = [                                # B, C, H, W, byte offset of the source view
    ((3, 72, 8, 17), 0),                    # C and H W multiples of 8 but not of 64: the vectorised 16-bit kernel
    ((3, 70, 13, 9), 0),                    # C % 8 != 0: scalar kernel
    ((3, 72, 13, 9), 0),                    # H W % 8 != 0: scalar kernel
    ((3, 72, 8, 17), 1),                    # a source one element past an aligned address: scalar kernel
]


def relayout_input(dt, case, to_nhwc):
    """-> (x, tensor.contiguous(memory_format=...) of x in the other layout)"""
    (B, C, H, W), off = RELAYOUT[case]
    torch.manual_seed(case)
    buf = torch.randn(B * C * H * W + off, device=DEV).to(ALL[dt])[off:]
    if to_nhwc:
        x = buf.view(B, C, H, W)
        return x, x.contiguous(memory_format=torch.channels_last)
    x = buf.view(B, H, W, C).permute(0, 3, 1, 2)
    assert x.is_contiguous(memory_format=torch.channels_last)
    return x, x.contiguous()


def vectorised(x):
    """relayout's choice of kernel (relayout.cu:72): 16-bit elements, rows and columns multiples of 8, 16-byte aligned
    pointers (the output is a fresh allocation)"""
    _, C, H, W = x.shape
    return x.element_size() == 2 and C % 8 == 0 and (H * W) % 8 == 0 and x.data_ptr() % 16 == 0


@pytest.mark.parametrize("to_nhwc", [True, False])
@pytest.mark.parametrize("case", range(len(RELAYOUT)))
@pytest.mark.parametrize("dt", sorted(ALL))
def test_relayout_bit_identical(F_, dt, case, to_nhwc):
    x, want = relayout_input(dt, case, to_nhwc)
    y = F_.relayout(x, to_nhwc)
    assert y.stride() == want.stride()
    bits = {2: torch.int16, 4: torch.int32, 8: torch.int64}[x.element_size()]
    assert torch.equal(y.view(bits), want.view(bits))
    PATHS.add(f"relayout {'vectorised' if vectorised(x) else 'scalar'}")


# Runs in a fresh process, so that no profiler session of an earlier test shares it: every relayout case above once
# (after an unprofiled warm-up call) inside ONE profiler session -- a process that opens many sessions eventually gets
# sessions that record no kernel.  Each call launches one transpose kernel and is synchronised before the next, so the
# kernels sorted by start time are the cases in order.  -> [dt, case, to_nhwc, vectorised(x), kernel name] per case.
_RUN = r"""
import json
import sys
import torch
import gfla_b200
from torch.profiler import ProfilerActivity, profile
sys.path.insert(0, "tests")
from test_gpu_gather_bounds import ALL, RELAYOUT, relayout_input, vectorised
cases = [(dt, case, to_nhwc) for dt in sorted(ALL) for case in range(len(RELAYOUT)) for to_nhwc in (True, False)]
xs = [relayout_input(*c)[0] for c in cases]
for x, c in zip(xs, cases):
    gfla_b200.functional.relayout(x, c[2])
torch.cuda.synchronize()
for _ in range(3):                                  # a session that missed a kernel is repeated
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for x, c in zip(xs, cases):
            gfla_b200.functional.relayout(x, c[2])
            torch.cuda.synchronize()
    kern = sorted((e for e in prof.events() if "k_transpose" in e.name), key=lambda e: e.time_range.start)
    if len(kern) == len(cases):
        break
names = [e.name for e in kern] if len(kern) == len(cases) else [None] * len(cases)
json.dump([list(c) + [vectorised(x), n] for c, x, n in zip(cases, xs, names)], open(sys.argv[1], "w"))
"""


def test_relayout_kernel_choice_profiled(tmp_path):
    """each case launched the kernel vectorised() says: k_transpose16_vec or the scalar k_transpose"""
    from conftest import ROOT
    dst = tmp_path / "relayout.json"
    subprocess.run([sys.executable, "-c", _RUN, str(dst)], cwd=ROOT, check=True)
    res = json.load(open(dst))
    assert len(res) == len(ALL) * len(RELAYOUT) * 2
    for dt, case, to_nhwc, vec, name in res:
        assert name is not None and ("k_transpose16_vec" in name) == vec, (dt, case, to_nhwc, vec, name)
    assert {vec for *_, vec, _ in res} == {True, False}
