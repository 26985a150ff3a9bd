"""GPU (-m gpu): resample2d and the fused resample2d -> cosine kernels (csrc/resample2d.cu) in fp32 and fp64 against the
fp64 reference (ref64_resample), element by element, with bounds derived from what each kernel rounds (DESIGN.md
section 6).  Covers both grad_input1 scatters (shuffle-merged and per tap), both channel slicings of the cosine kernels,
accumulate = 1 through the C ABI, the degenerate sigmas and the rejected kernel sizes."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import ref64
import ref64_resample as rr
from test_ref64_resample import FLOWS, SIGMAS, cosine_sources, make_in2

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
EPS = 1e-8
WORST = {}
DTYPES = {"fp32": np.float32, "fp64": np.float64}


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def host(t):
    return np.ascontiguousarray(t.detach().cpu().numpy()).astype(np.float64)


def within(row, y, ref, bound, **mags):
    r = ref64.assert_within(row, host(y) if torch.is_tensor(y) else y, ref, bound, **mags)
    WORST[row] = max(WORST.get(row, 0.0), r)


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
SHAPES = [                                  # B, C, Hi, Wi, H, W
    (2, 5, 13, 70, 13, 70),                 # ragged 32 x 4 tiles, odd C
    (2, 3, 29, 137, 21, 128),               # source larger than the flow grid
    (2, 5, 9, 40, 14, 67),                  # source smaller
    (3, 3, 1, 50, 6, 37),                   # one-row source
    (2, 3, 30, 1, 10, 33),                  # one-column source
]


def cases(dt, ks, dil):
    """the six flow families, each on one shape and sigma, in rotation so that every pair meets over the ks, dil grid.  The
    smooth flow always runs on the shape whose source has a margin, so that its warps keep their taps inside"""
    for i, kind in enumerate(FLOWS):
        B, C, Hi, Wi, H, W = SHAPES[1 if kind == "smooth" else (i + ks + dil) % len(SHAPES)]
        rng = np.random.default_rng(1000 * ks + 100 * dil + i)
        in2 = make_in2(kind, rng, B, H, W, Hi, Wi, SIGMAS[(i + dil) % len(SIGMAS)], dt)
        a = rng.standard_normal((B, C, Hi, Wi)).astype(dt)
        g = rng.standard_normal((B, C, H, W)).astype(dt)
        yield kind, a, in2, g


KS, DILS = [2, 3, 4, 5, 6, 8], [1, 2, 3]


def test_cases_run_both_grad_input1_paths():
    """host predicate of k_resample2d_bwd_in1's choice over the cases below that may take the shuffle path (NT <= 2,
    dil = 1): both paths on a substantial share of their warps"""
    fast = total = 0
    for ks in (2, 3, 4, 5):
        for kind, a, in2, g in cases(np.float32, ks, 1):
            f = rr.fast_warps(in2, ks, 1, *a.shape[2:])
            fast, total = fast + int(f.sum()), total + f.size
    assert 0.15 * total < fast < 0.85 * total, (fast, total)


@pytest.mark.parametrize("dil", DILS)
@pytest.mark.parametrize("ks", KS)
@pytest.mark.parametrize("dt", sorted(DTYPES))
def test_resample2d_within_bounds(F_, dt, ks, dil):
    for kind, a, in2, g in cases(DTYPES[dt], ks, dil):
        r = rr.resample2d(a, in2, ks, dil, g)
        u, eta = rr.unit(a.dtype)
        out = F_.resample2d_fwd(cu(a), cu(in2), ks, dil)
        within(f"fwd {dt}", out, r["out"], rr.bound_fwd(r["out"], r["mags_out"], u, eta), M=r["mags_out"]["M"])
        g1, g2 = F_.resample2d_bwd(cu(a), cu(in2), cu(g), ks, dil)
        path = "shuffle" if rr.fast_warps(in2, ks, dil, *a.shape[2:]).all() else "per tap/mixed"
        within(f"grad_in1 {dt} {path}", g1, r["gin1"], rr.bound_in1(r["gin1"], r["mags_in1"], u, eta),
               G1=r["mags_in1"]["G1"], m=r["mags_in1"]["m"])
        b2 = rr.bound_in2(r["gin2"], r["mags_in2"], u, eta)
        for p, name in enumerate(("dx", "dy", "dsigma")):
            within(f"grad_in2 {name} {dt}", host(g2)[:, p], r["gin2"][:, p], b2[:, p])


@pytest.mark.parametrize("ks", [4, 6])
@pytest.mark.parametrize("dt", sorted(DTYPES))
def test_resample2d_backward_accumulates(F_, dt, ks):
    """accumulate = 1 through the C ABI: both gradients are added into non-zero buffers"""
    from gfla_b200 import _lib
    from gfla_b200.functional import _dt, _p, _stream
    for kind in ("smooth", "iid"):
        B, C, Hi, Wi, H, W = SHAPES[1]
        rng = np.random.default_rng(ks + len(kind))
        in2 = make_in2(kind, rng, B, H, W, Hi, Wi, 2.0, DTYPES[dt])
        a = rng.standard_normal((B, C, Hi, Wi)).astype(in2.dtype)
        g = rng.standard_normal((B, C, H, W)).astype(in2.dtype)
        i1, i2 = rng.standard_normal(a.shape).astype(a.dtype), rng.standard_normal(in2.shape).astype(a.dtype)
        ta, t2, tg, g1, g2 = cu(a), cu(in2), cu(g), cu(i1), cu(i2)
        _lib.check(_lib.lib().gfla_resample2d_bwd(_p(ta), _p(t2), _p(tg), _p(g1), _p(g2), B, C, Hi, Wi, H, W, ks, 1,
                                                  _dt(ta), 1, _stream(ta)), "resample2d_bwd")
        r = rr.resample2d(a, in2, ks, 1, g)
        u, eta = rr.unit(a.dtype)
        i1, i2 = i1.astype(np.float64), i2.astype(np.float64)
        within(f"grad_in1 {dt} accumulate", g1, r["gin1"] + i1, rr.bound_in1(r["gin1"] + i1, r["mags_in1"], u, eta, i1))
        within(f"grad_in2 {dt} accumulate", g2, r["gin2"] + i2, rr.bound_in2(r["gin2"] + i2, r["mags_in2"], u, eta, i2))


# ------------------------------------------------------------------------------------------------ fused cosine
COS = [                                     # B, C, Hi, Wi, H, W, ks, dil: B H W >= 1024, so one SM never slices
    (2, 9, 14, 40, 12, 44, 4, 1),
    (2, 64, 70, 8, 70, 8, 2, 1),
    (2, 66, 36, 20, 40, 16, 4, 2),
    (2, 67, 15, 50, 13, 44, 5, 1),
    (2, 256, 9, 70, 8, 70, 3, 1),
    (2, 512, 33, 16, 33, 16, 4, 1),
    (2, 66, 13, 44, 13, 44, 6, 1),          # NT = 3: no sliced instance
]
NEEDS = [(False, False), (True, False), (False, True), (True, True)]


def cos_inputs(i, dt):
    B, C, Hi, Wi, H, W, ks, dil = COS[i]
    rng = np.random.default_rng(50 + i)
    in2 = make_in2(["smooth", "iid", "neg", "torn"][i % 4], rng, B, H, W, Hi, Wi, SIGMAS[i % 4], dt)
    a, t = cosine_sources(rng, B, C, Hi, Wi, H, W, dt)
    gc = rng.standard_normal((B, H, W)).astype(dt)
    return a, in2, t, gc, ks, dil


# Runs in a fresh process (sm_count() is read once per process): every cosine case through the library, all four
# need_input1 / need_target combinations, accumulate = 1 through the ABI, the one-hot identity, and the names of the
# kernels one profiled forward + backward of the first sliceable case launched.
_RUN = r"""
import sys
import numpy as np
import torch
import gfla_b200
from gfla_b200 import _lib
from gfla_b200.functional import _dt, _p, _stream
F = gfla_b200.functional
z = np.load(sys.argv[1])
out = {}
cu = lambda k: torch.from_numpy(z[k]).cuda()
host = lambda t: t.detach().cpu().numpy()
for key in sorted({k.split("/")[0] for k in z.files if "/" in k}):
    a, in2, t, gc = (cu(f"{key}/{n}") for n in ("a", "in2", "t", "gc"))
    ks, dil = (int(v) for v in z[f"{key}/ks_dil"])
    B, C, Hi, Wi = a.shape
    H, W = in2.shape[2:]
    cos, st = F.resample2d_cosine_fwd(a, in2, t, ks, dil, 1e-8)
    out[f"{key}/cos"], out[f"{key}/stats"] = host(cos), host(st)
    for n1, nt in [(False, False), (True, False), (False, True), (True, True)]:
        g1, g2, g3 = F.resample2d_cosine_bwd(a, in2, t, st, gc, ks, dil, 1e-8, need_input1=n1, need_target=nt)
        tag = f"{key}/{int(n1)}{int(nt)}"
        out[tag + "/gin2"] = host(g2)
        if n1: out[tag + "/gin1"] = host(g1)
        if nt: out[tag + "/gt"] = host(g3)
    i1, i2, it = cu(f"{key}/init1"), cu(f"{key}/init2"), cu(f"{key}/initt")
    gv = torch.empty_like(t)
    _lib.check(_lib.lib().gfla_resample2d_cosine_bwd(_p(a), _p(in2), _p(t), _p(st), _p(gc), _p(i1), _p(i2), _p(gv), _p(it), B, C,
               Hi, Wi, H, W, ks, dil, 1e-8, _dt(a), 1, _stream(a)), "resample2d_cosine_bwd")
    out[f"{key}/acc_gin1"], out[f"{key}/acc_gin2"], out[f"{key}/acc_gt"], out[f"{key}/gval"] = host(i1), host(i2), host(it), host(gv)
    c = C // 2                                            # one-hot target: stats[:, 0] is the warped channel c
    oh = torch.zeros_like(t)
    oh[:, c] = 1
    _, st1 = F.resample2d_cosine_fwd(a, in2, oh, ks, dil, 1e-8)
    w = F.resample2d_fwd(a, in2, ks, dil)
    out[f"{key}/onehot_equal"] = np.array(bool(torch.equal(st1[:, 0], w[:, c])))
first = z["profile_key"].item()
if first:
    from torch.profiler import ProfilerActivity, profile
    a, in2, t, gc = (cu(f"{first}/{n}") for n in ("a", "in2", "t", "gc"))
    ks, dil = (int(v) for v in z[f"{first}/ks_dil"])
    for _ in range(3):                                    # a session that recorded none of this library's kernels is repeated
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            cos, st = F.resample2d_cosine_fwd(a, in2, t, ks, dil, 1e-8)
            F.resample2d_cosine_bwd(a, in2, t, st, gc, ks, dil, 1e-8)
            torch.cuda.synchronize()
        names = [e.key for e in prof.key_averages()]
        if any("k_resample2d_cos" in n for n in names):
            break
    out["kernel_names"] = np.array(names)
np.savez(sys.argv[2], **out)
"""


@pytest.fixture(scope="module")
def cos_runs(tmp_path_factory):
    """{(dtype, sm_count): results} from a subprocess per SM count: 1 keeps every case on the TS = 1 kernels, 100000
    puts every case with C >= 64 and NT <= 2 on the TS = 4 kernels"""
    from conftest import ROOT
    d = tmp_path_factory.mktemp("cos")
    res = {}
    for dt in sorted(DTYPES):
        inp = {}
        for i in range(len(COS)):
            a, in2, t, gc, ks, dil = cos_inputs(i, DTYPES[dt])
            rng = np.random.default_rng(i)
            inp.update({f"c{i}/a": a, f"c{i}/in2": in2, f"c{i}/t": t, f"c{i}/gc": gc, f"c{i}/ks_dil": np.array([ks, dil]),
                        f"c{i}/init1": rng.standard_normal(a.shape).astype(a.dtype),
                        f"c{i}/init2": rng.standard_normal(in2.shape).astype(a.dtype),
                        f"c{i}/initt": rng.standard_normal(t.shape).astype(a.dtype)})
        for sm in (1, 100000):
            inp["profile_key"] = np.array("c1" if sm == 100000 and dt == "fp32" else "")
            src, dst = d / f"in_{dt}_{sm}.npz", d / f"out_{dt}_{sm}.npz"
            np.savez(src, **inp)
            env = dict(os.environ, GFLA_SM_COUNT=str(sm))
            subprocess.run([sys.executable, "-c", _RUN, str(src), str(dst)], cwd=ROOT, env=env, check=True)
            res[dt, sm] = dict(np.load(dst))
    return res


def test_cosine_sliced_kernel_ran(cos_runs):
    """the profiled run with a huge SM count launched the TS = 4 instances (cos_slices agrees)"""
    B, C, Hi, Wi, H, W, ks, dil = COS[1]
    assert rr.cos_slices(B, C, H, W, ks, 100000) == 4 and rr.cos_slices(B, C, H, W, ks, 1) == 1
    names = [str(n) for n in cos_runs["fp32", 100000]["kernel_names"]]
    assert any("k_resample2d_cos_fwd<float, 1, 4>" in n for n in names), names
    assert any("k_resample2d_cos_bwd<float, 1, 4>" in n for n in names), names


@pytest.mark.parametrize("i", range(len(COS)))
@pytest.mark.parametrize("dt", sorted(DTYPES))
def test_cosine_within_bounds(cos_runs, dt, i):
    a, in2, t, gc, ks, dil = cos_inputs(i, DTYPES[dt])
    B, C, Hi, Wi, H, W = COS[i][:6]
    c = rr.cosine(a, in2, t, ks, dil, EPS, gc)
    u, eta = rr.unit(a.dtype)
    # both clamp branches, and every non-zero norm well away from eps
    for n in (c["nv"], c["nt"]):
        assert (n == 0).any() and (n > EPS).any()
        assert (np.abs(n[n != 0] - EPS) > 1e-3 * EPS).all()
    rng = np.random.default_rng(i)
    i1, i2, itg = (rng.standard_normal(s).astype(a.dtype).astype(np.float64) for s in (a.shape, in2.shape, t.shape))
    ts = {sm: rr.cos_slices(B, C, H, W, ks, sm) for sm in (1, 100000)}
    assert ts[1] == 1 and ts[100000] == (4 if C >= 64 and ks // 2 <= 2 else 1)
    m1 = c["mags_in1"]
    for sm, TS in ts.items():
        res, k = cos_runs[dt, sm], f"c{i}"
        row = f"{dt} TS={TS}"
        within(f"cos {row}", res[f"{k}/cos"], c["cos"], rr.bound_cos(c, u, eta))
        within(f"stats {row}", res[f"{k}/stats"], c["stats"], rr.bound_stats(c, u, eta))
        b2 = rr.bound_in2(c["gin2"], c["mags_in2"], u, eta)
        bt = rr.bound_gt(c, u, eta)
        b1 = rr.bound_in1(c["gin1"], m1, u, eta)
        for n1, nt in NEEDS:
            tag = f"{k}/{int(n1)}{int(nt)}"
            within(f"cos grad_in2 {row}", res[tag + "/gin2"], c["gin2"], b2)
            if n1:
                within(f"cos grad_in1 {row}", res[tag + "/gin1"], c["gin1"], b1, G1=m1["G1"])
            if nt:
                within(f"cos grad_target {row}", res[tag + "/gt"], c["gt"], bt)
        within(f"cos grad_val {row}", res[f"{k}/gval"], c["gval"], rr.bound_gval(c, u, eta))
        within(f"cos grad_in1 {row} accumulate", res[f"{k}/acc_gin1"], c["gin1"] + i1,
               rr.bound_in1(c["gin1"] + i1, m1, u, eta, i1))
        within(f"cos grad_in2 {row} accumulate", res[f"{k}/acc_gin2"], c["gin2"] + i2,
               rr.bound_in2(c["gin2"] + i2, c["mags_in2"], u, eta, i2))
        within(f"cos grad_target {row} accumulate", res[f"{k}/acc_gt"], c["gt"] + itg, rr.bound_gt(c, u, eta, itg))
        # k_resample2d_cos_fwd's warped value is exactly k_resample2d_fwd's output element
        assert bool(res[f"{k}/onehot_equal"]), (dt, i, TS)


# ------------------------------------------------------------------------------------------- degenerate and rejected
@pytest.mark.parametrize("dt", sorted(DTYPES))
@pytest.mark.parametrize("case", ["sigma0-int", "sigma0-iid", "underflow"])
def test_degenerate_sigma_matches_oracle(F_, oracle_lib, dt, case):
    """sigma = 0 (SAFE_DIV's 1e-8 inside exp and in rs_in2_store) and a sigma so small that the weights leave the normal
    range (fp32: sum == 0 and sum*sum == 0; fp64: sum*sum subnormal): finite, and equal to the oracle of the same dtype"""
    B, C, Hi, Wi, H, W = SHAPES[0]
    rng = np.random.default_rng(len(case))
    kind, sigma = {"sigma0-int": ("int", 0.0), "sigma0-iid": ("iid", 0.0), "underflow": ("iid", 0.02)}[case]
    in2 = make_in2(kind, rng, B, H, W, Hi, Wi, sigma, DTYPES[dt])
    a = rng.standard_normal((B, C, Hi, Wi)).astype(in2.dtype)
    g = rng.standard_normal((B, C, H, W)).astype(in2.dtype)
    tol = 1e-5 if dt == "fp32" else 1e-11
    out = host(F_.resample2d_fwd(cu(a), cu(in2), 4, 1))
    g1, g2 = (host(x) for x in F_.resample2d_bwd(cu(a), cu(in2), cu(g), 4, 1))
    o, (o1, o2) = oracle_lib.resample2d_fwd(a, in2, 4, 1), oracle_lib.resample2d_bwd(a, in2, g, 4, 1)
    for y in (out, g1, g2):
        assert np.isfinite(y).all()
    np.testing.assert_allclose(out, o, rtol=tol, atol=tol * max(1.0, float(np.abs(o).max())))
    np.testing.assert_allclose(g1, o1, rtol=tol, atol=tol * max(1.0, float(np.abs(o1).max())))
    # grad_input2, every element: where weights leave A's normal range the two round differently (the oracle's A product
    # chains against the kernel's double products), and 1/sum, 1/sum^2 amplify that; bound_in2_vs_oracle names it
    r = rr.resample2d(a, in2, 4, 1, g)
    within(f"grad_in2 {dt} sigma {case} vs oracle", g2, o2.astype(np.float64), rr.bound_in2_vs_oracle(r, a, g, o2))
    if case == "underflow":
        t = r["taps"]
        if dt == "fp32":
            assert t.s2_zero.any() and t.s_zero.any()
        else:                                              # sum*sum subnormal: what the fix of rs_in2_store is about
            assert ((t.sum ** 2 < np.finfo(np.float64).tiny) & ~t.s2_zero).any()


@pytest.mark.parametrize("ks", [1, 10, 12])
def test_rejected_kernel_sizes_raise(F_, ks):
    from gfla_b200._lib import GflaError
    a = torch.randn(1, 3, 8, 40, device=DEV)
    in2 = torch.cat([torch.randn(1, 2, 8, 40, device=DEV), torch.full((1, 1, 8, 40), 2.0, device=DEV)], 1)
    t = torch.randn(1, 3, 8, 40, device=DEV)
    with pytest.raises(GflaError):
        F_.resample2d_fwd(a, in2, ks, 1)
    with pytest.raises(GflaError):
        F_.resample2d_bwd(a, in2, t, ks, 1)
    with pytest.raises(GflaError):
        F_.resample2d_cosine_fwd(a, in2, t, ks, 1)
