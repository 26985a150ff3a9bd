"""CPU checks of ref64_resample: the fp64 reference against the oracle's fp64 resample2d, the bounds against the oracle's
fp32 results and numpy emulations of the kernels' fp32 rounding (they pass), and against injected faults (they fail)."""
import numpy as np
import pytest

import ref64
import ref64_resample as rr

EPS = 1e-8
FLOWS = ["smooth", "iid", "int", "neg", "torn", "outside"]
SIGMAS = [5.0, 2.0, 1.5, "plane"]


def make_in2(kind, rng, B, H, W, Hi, Wi, sigma, dt):
    """in2 = (dx, dy, sigma) [B, 3, H, W].  smooth: a 4 x 4 nearest-upsampled fraction plus an integer shift per 32-column
    warp and 4-row block (as PerceptualCorrectness upsamples a coarse flow), so one integer shift per warp; iid; int
    (alpha = 0); neg: half the coordinates negative and non-integer (int() and floor differ); torn: smooth with the shift
    stepping inside each warp; outside: every tap beyond the image (all clamped)"""
    rep = lambda a, ry, rx: np.repeat(np.repeat(a, ry, -2), rx, -1)[..., :H, :W]
    if kind in ("smooth", "torn"):
        f = rep(rng.uniform(0.05, 0.95, (B, 2, (H + 3) // 4, (W + 3) // 4)), 4, 4)
        f = f + rep(rng.integers(1, 3, (B, 2, (H + 3) // 4, (W + 31) // 32)), 4, 32)
        if kind == "torn":
            cut = rng.integers(1, 31, (B, 1, H, (W + 31) // 32))
            f[:, :1] += (np.arange(W) % 32 >= rep(cut, 1, 32)).astype(np.float64)
    elif kind == "iid":
        f = rng.uniform(-4, 4, (B, 2, H, W))
    elif kind == "int":
        f = rng.integers(-3, 4, (B, 2, H, W)).astype(np.float64)
    elif kind == "neg":
        f = rng.uniform(-3, 3, (B, 2, H, W))
        neg = rng.random((B, 2, H, W)) < 0.5
        coord = np.stack(np.broadcast_arrays(np.arange(W)[None, :], np.arange(H)[:, None]))
        f = np.where(neg, -coord - rng.uniform(0.05, 2.5, (B, 2, H, W)), f)
    elif kind == "outside":
        lim = np.array([W + Wi, H + Hi]).reshape(1, 2, 1, 1) + 13       # the widest window reaches 4 taps x dil 3
        f = rng.choice([-1.0, 1.0], (B, 2, H, W)) * (lim + rng.uniform(0.1, 5, (B, 2, H, W)))
    else:
        raise ValueError(kind)
    s = rng.uniform(0.5, 6, (B, 1, H, W)) if sigma == "plane" else np.full((B, 1, H, W), sigma)
    return np.ascontiguousarray(np.concatenate([f, s], 1), dt)


def magnitude_close(y, ref, mag, rel):
    err = np.abs(np.asarray(y, np.float64) - ref)
    worst = float((err / (rel * (mag + np.abs(ref)) + 1e-300)).max())
    assert worst <= 1.0, worst


# ---------------------------------------------------------------------------------------- reference vs oracle fp64
@pytest.mark.parametrize("dil", [1, 2, 3])
@pytest.mark.parametrize("ks", [2, 3, 4, 5, 6, 8])
def test_reference_matches_oracle_fp64(oracle_lib, ks, dil):
    B, C, Hi, Wi, H, W = 2, 3, 11, 23, 9, 37
    for i, kind in enumerate(FLOWS):
        rng = np.random.default_rng(100 * ks + 10 * dil + i)
        in2 = make_in2(kind, rng, B, H, W, Hi, Wi, SIGMAS[(i + ks) % 4], np.float64)
        a = rng.standard_normal((B, C, Hi, Wi))
        g = rng.standard_normal((B, C, H, W))
        r = rr.resample2d(a, in2, ks, dil, g)
        o = oracle_lib.resample2d_fwd(a, in2, ks, dil)
        o1, o2 = oracle_lib.resample2d_bwd(a, in2, g, ks, dil)
        magnitude_close(o, r["out"], r["mags_out"]["M"], 1e-12)
        magnitude_close(o1, r["gin1"], r["mags_in1"]["G1"], 1e-12)
        magnitude_close(o2, r["gin2"], r["mags_in2"]["T"], 1e-12)


def test_cosine_reference_matches_oracle_chain(oracle_lib):
    from test_gpu_resample_cosine import _cos_chain
    for ks, dil, kind in [(4, 1, "smooth"), (2, 2, "iid"), (6, 1, "neg"), (3, 3, "outside")]:
        rng = np.random.default_rng(ks + dil)
        B, C, Hi, Wi, H, W = 2, 7, 13, 30, 11, 33
        in2 = make_in2(kind, rng, B, H, W, Hi, Wi, "plane", np.float64)
        a, t = cosine_sources(rng, B, C, Hi, Wi, H, W)
        gc = rng.standard_normal((B, H, W))
        c = rr.cosine(a, in2, t, ks, dil, EPS, gc)
        v = oracle_lib.resample2d_fwd(a, in2, ks, dil)
        cos, gv, gt = _cos_chain(v, t, gc)
        assert (c["nv"] == 0).any() and (c["nt"] == 0).any()
        np.testing.assert_allclose(c["cos"], cos, rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(c["gval"], gv, rtol=1e-11, atol=1e-11 * np.abs(gv).max())
        np.testing.assert_allclose(c["gt"], gt, rtol=1e-11, atol=1e-11 * np.abs(gt).max())
        o1, o2 = oracle_lib.resample2d_bwd(a, in2, gv, ks, dil)
        magnitude_close(o1, c["gin1"], c["mags_in1"]["G1"], 1e-11)
        magnitude_close(o2, c["gin2"], c["mags_in2"]["T"], 1e-11)


def cosine_sources(rng, B, C, Hi, Wi, H, W, dt=np.float64):
    """source with a zero block (warped vectors exactly zero where every tap lands inside it) and target with zero
    vectors: both eps clamps run"""
    a = rng.standard_normal((B, C, Hi, Wi))
    a[:, :, : Hi // 2, : Wi // 2] = 0
    t = rng.standard_normal((B, C, H, W))
    t[:, :, H // 3, :] = 0
    return a.astype(dt), t.astype(dt)


# ------------------------------------------------------------------------------------------ fp32 kernel emulation
f32, f64 = np.float32, np.float64


def emu_weights(t):
    """fp32 Gaussian factors and weights of rs_setup / rs_weight_sum: the quotient in fp32, exp in double, narrowed"""
    two = t.two_s2
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        def P(d):
            num = (-d) * d
            q = np.where(two == 0, num.astype(f64) / 1e-8, (num / np.where(two == 0, f32(1), two)).astype(f64))
            return np.exp(q).astype(f32)
    xL, xR, yT, yB = (P(d) for d in t.dist)
    Y, X = (yT, yT, yB, yB), (xL, xR, xL, xR)
    NT, shp = t.NT, (t.n, t.B, t.H * t.W)
    w = np.empty((NT, NT, 4, t.B, t.H, t.W), f32)
    for c in range(4):
        w[:, :, c] = Y[c][:, None] * X[c][None]
    w = w.reshape(shp)
    s = np.zeros(shp[1:], f32)
    for k in range(NT * NT):
        s = s + (((w[4 * k] + w[4 * k + 1]) + w[4 * k + 2]) + w[4 * k + 3])
    return w, s, (yT, yB, xL, xR)


def gather(t, src):
    """src [B, C, Hi, Wi] at every tap -> (n, B, C, H W); positions past the end read 0"""
    B, C = src.shape[:2]
    flat = np.concatenate([src.reshape(B, C, -1), np.zeros((B, C, t.Wi + 1), src.dtype)], 2)
    return np.stack([np.stack([flat[b][:, t.off[q, b]] for b in range(B)]) for q in range(t.n)])


def emu_fwd(t, src, fault=None):
    w, s, _ = emu_weights(t)
    taps = gather(t, src)
    val = np.zeros(taps.shape[1:], f32)
    for q in range(t.n):
        if fault == "drop_tap" and q == 0:
            continue
        val = val + w[q][:, None] * taps[q]
    out = val if fault == "no_sum" else val / s[:, None]
    return out.reshape(src.shape[:2] + (t.H, t.W))


def emu_in1(t, g, order, init=None, fault=None, fast=None):
    """the scatter with one fp32 add per partial, in the given order (seq / rev / shuffle)"""
    w, s, _ = emu_weights(t)
    B, C = g.shape[:2]
    wn = (w / s[None]).astype(f64)
    out = np.zeros((B, C, t.Hi * t.Wi), f32) if init is None else init.reshape(B, C, -1).astype(f32).copy()
    g = g.reshape(B, C, -1).astype(f64)
    lane = np.arange(t.W) % 32
    co = np.concatenate([[-fx, fx + 1, -fx, fx + 1] for _ in range(t.NT) for fx in range(t.NT)])
    for b in range(B):
        part = (wn[:, b][:, None] * g[b][None]).astype(f32)                     # (n, C, H W)
        idx = np.broadcast_to(t.off[:, b][:, None], part.shape)
        ch = np.broadcast_to(np.arange(C)[None, :, None], part.shape)
        keep = np.ones(part.shape, bool)
        if fault == "drop_oos":                                                  # the fast path's out-of-span taps
            oos = ((lane[None] + co[:, None] < 0) | (lane[None] + co[:, None] > 31))   # (n, W)
            onfast = np.repeat(fast[b], 32, axis=1)[:, :t.W].reshape(-1)             # (H W)
            keep &= ~(np.tile(oos, (1, t.H)) & onfast[None])[:, None]
        p, i, c = part[keep], idx[keep], ch[keep]
        perm = {"seq": np.arange(p.size), "rev": np.arange(p.size)[::-1],
                "shuffle": np.random.default_rng(b).permutation(p.size)}[order]
        np.add.at(out[b], (c[perm], i[perm]), p[perm])
    return out.reshape(B, C, t.Hi, t.Wi)


def emu_store(t, D, fault=None, init=None):
    """rs_in2_store (resample2d.cu:232-264): double arithmetic on the fp32 factors, distances and corner sums"""
    w, s, (yT, yB, xL, xR) = emu_weights(t)
    NT, B, HW = t.NT, t.B, t.H * t.W
    Y, X = (yT, yT, yB, yB), (xL, xR, xL, xR)
    w64 = np.empty((NT, NT, 4, B, t.H, t.W))
    for c in range(4):
        w64[:, :, c] = Y[c][:, None].astype(f64) * X[c][None].astype(f64)
    w64 = w64.reshape(t.n, B, HW)
    D = np.asarray(D, f64)
    if fault == "swap_tltr":
        D = D.reshape(NT * NT, 4, B, HW)[:, [1, 0, 2, 3]].reshape(t.n, B, HW)
    a = [x.copy() for x in t.a]
    if fault == "drop_dsigma":
        a[2] = a[2].reshape(NT * NT, 4, B, HW)
        a[2][:, 3] = 0
        a[2] = a[2].reshape(t.n, B, HW)
    wd = (w64 * D).sum(0)
    S = s.astype(f64)
    S = np.where(s == 0, 1e-8, S)                                   # quotients, as the kernel forms them
    S2 = np.where(s * s == 0, 1e-8, (s * s).astype(f64))
    planes = []
    for k in range(3):
        g1 = (a[k] * w64 * D).sum(0) / t.den[k]
        sg = (a[k] * w64).sum(0) / t.den[k]
        sign = 1.0 if fault == "sgrad_sign" else -1.0
        planes.append((g1 / S + sign * (sg * wd) / S2).astype(f32))
    if fault == "swap_xy":
        planes[0], planes[1] = planes[1], planes[0]
    out = np.stack(planes, 1).reshape(B, 3, t.H, t.W)
    return out if init is None else (init.astype(f32) + out)


def emu_in2(t, src, g, fault=None):
    taps = gather(t, src)
    B, C = g.shape[:2]
    g = g.reshape(B, C, -1)
    D = np.zeros((t.n, B, t.H * t.W), f32)
    for c in range(C):
        D = D + g[None, :, c] * taps[:, :, c]
    return emu_store(t, D, fault)


def emu_cos(t, src, tgt, gcos, TS, fault=None):
    """the fused forward and backward with TS channel slices combined in fp32 in slice order"""
    v = emu_fwd(t, src)
    B, C = v.shape[:2]
    cs = -(-C // TS)
    sl = [slice(k * cs, min(C, (k + 1) * cs)) for k in range(TS)]
    e = f32(EPS)

    def csum(x):
        parts = [np.zeros(x.shape[:1] + x.shape[2:], f32) for _ in sl]
        for k, ss in enumerate(sl):
            for c in range(ss.start, ss.stop):
                parts[k] = parts[k] + x[:, c]
        tot = np.zeros_like(parts[0])
        for k in range(TS):
            if not (fault == "drop_slice" and k == TS - 1):
                tot = tot + parts[k]
        return tot
    dot, vv, tt = csum(v * tgt), csum(v * v), csum(tgt * tgt)
    nv = np.sqrt(np.maximum(vv, e)) if fault == "clamp_vv" else np.sqrt(vv)
    nt = np.sqrt(tt)
    a, bb = np.maximum(nv, e), np.maximum(nt, e)
    cos = dot / (a * bb)
    stats = np.stack([dot, nv, nt], 1)
    g = gcos.astype(f32)
    with np.errstate(divide="ignore", invalid="ignore"):
        k1 = g / (a * bb)
        side = (nv <= e) if fault == "k2v_flip" else (nv > e)
        k2v = np.where(side, (g * dot) / (((a * a) * bb) * nv), f32(0)).astype(f32)
        k2t = np.where(nt > e, (g * dot) / (((a * bb) * bb) * nt), f32(0)).astype(f32)
    gv = k1[:, None] * tgt - k2v[:, None] * v
    gt = k1[:, None] * v if fault == "no_k2t" else k1[:, None] * v - k2t[:, None] * tgt
    taps = gather(t, src)
    Dp = [np.zeros((t.n, B, t.H * t.W), f32) for _ in sl]
    gvf = gv.reshape(B, C, -1)
    for k, ss in enumerate(sl):
        for c in range(ss.start, ss.stop):
            Dp[k] = Dp[k] + gvf[None, :, c] * taps[:, :, c]
    D = np.zeros_like(Dp[0])
    for k in range(TS):
        D = D + Dp[k]
    return cos, stats, gv, gt, emu_store(t, D)


# ----------------------------------------------------------------------------------------------- the standard inputs
STD = (2, 5, 20, 72, 12, 64)            # B, C, Hi, Wi, H, W: two full warps per row, source larger than the flow


def std_case(kind, ks=4, dil=1, seed=0):
    B, C, Hi, Wi, H, W = STD
    rng = np.random.default_rng(seed + len(kind))
    in2 = make_in2(kind, rng, B, H, W, Hi, Wi, "plane", f32)
    a = rng.standard_normal((B, C, Hi, Wi)).astype(f32)
    g = rng.standard_normal((B, C, H, W)).astype(f32)
    return a, in2, g


def check_fwd(r, y, name="fwd"):
    u, eta = rr.unit(f32)
    return ref64.check(name, y, r["out"], rr.bound_fwd(r["out"], r["mags_out"], u, eta))


def check_in1(r, y, init=0.0):
    u, eta = rr.unit(f32)
    return ref64.check("in1", y, r["gin1"] + init, rr.bound_in1(r["gin1"] + init, r["mags_in1"], u, eta, init))


def check_in2(r, y, init=0.0):
    u, eta = rr.unit(f32)
    return ref64.check("in2", y, r["gin2"] + init, rr.bound_in2(r["gin2"] + init, r["mags_in2"], u, eta, init))


@pytest.mark.parametrize("kind", FLOWS)
def test_oracle_fp32_within_bounds(oracle_lib, kind):
    for ks, dil in [(2, 1), (4, 1), (5, 2), (8, 3)]:
        a, in2, g = std_case(kind, ks, dil, seed=ks + dil)
        r = rr.resample2d(a, in2, ks, dil, g)
        assert check_fwd(r, oracle_lib.resample2d_fwd(a, in2, ks, dil))[1] is None
        o1, o2 = oracle_lib.resample2d_bwd(a, in2, g, ks, dil)
        assert check_in1(r, o1)[1] is None
        assert check_in2(r, o2)[1] is None


@pytest.mark.parametrize("order", ["seq", "rev", "shuffle"])
@pytest.mark.parametrize("kind", FLOWS)
def test_fp32_emulation_within_bounds(kind, order):
    for ks, dil in [(4, 1), (3, 2), (6, 1)]:
        a, in2, g = std_case(kind, ks, dil, seed=3 * ks + dil)
        r = rr.resample2d(a, in2, ks, dil, g)
        t, tt = r["taps"], rr.Resample2d(in2, ks, dil, *a.shape[2:], trunc=True)
        assert check_fwd(r, emu_fwd(t, a))[1] is None
        init = np.random.default_rng(1).standard_normal(a.shape).astype(f32)
        assert check_in1(r, emu_in1(tt, g, order))[1] is None
        assert check_in1(r, emu_in1(tt, g, order, init=init), init=init.astype(f64))[1] is None
        assert check_in2(r, emu_in2(t, a, g))[1] is None


def cos_case(seed=5, C=66, ks=4, dil=1, kind="iid"):
    B, H, W, Hi, Wi = 2, 12, 44, 14, 40
    rng = np.random.default_rng(seed)
    in2 = make_in2(kind, rng, B, H, W, Hi, Wi, "plane", f32)
    a, t = cosine_sources(rng, B, C, Hi, Wi, H, W, f32)
    gc = rng.standard_normal((B, H, W)).astype(f32)
    return a, in2, t, gc, ks, dil


def cos_checks(c, y):
    """-> list of (name, worst, message) of one emulated or kernel result y = (cos, stats, gval, gt, gin2)"""
    u, eta = rr.unit(f32)
    cos, stats, gv, gt, g2 = y
    return [ref64.check("cos", cos, c["cos"], rr.bound_cos(c, u, eta)),
            ref64.check("stats", stats, c["stats"], rr.bound_stats(c, u, eta)),
            ref64.check("gval", gv, c["gval"], rr.bound_gval(c, u, eta)),
            ref64.check("gt", gt, c["gt"], rr.bound_gt(c, u, eta)),
            ref64.check("gin2", g2, c["gin2"], rr.bound_in2(c["gin2"], c["mags_in2"], u, eta))]


@pytest.mark.parametrize("TS", [1, 4])
@pytest.mark.parametrize("C", [9, 66, 67])
def test_fp32_cosine_emulation_within_bounds(C, TS):
    a, in2, t, gc, ks, dil = cos_case(C=C)
    c = rr.cosine(a, in2, t, ks, dil, EPS, gc)
    assert (c["nv"] == 0).any() and (c["nt"] == 0).any()
    for _, msg in cos_checks(c, emu_cos(c["taps"], a, t, gc, TS)):
        assert msg is None, msg


# --------------------------------------------------------------------------------------------------- injected faults
def _fault_fwd(fault, kind):
    a, in2, g = std_case(kind)
    r = rr.resample2d(a, in2, 4, 1, g)
    t = r["taps"]
    if fault == "clamp_wi":                                    # the right-hand taps clamped to Wi instead of Wi - 1
        f = np.arange(t.NT).reshape(t.NT, 1, 1, 1)
        xlo = np.clip(t.flx - f, 0, t.Wi - 1)
        t2 = rr.Resample2d(in2, 4, 1, *a.shape[2:])
        t2.set_taps(np.clip(t.fly - f, 0, t.Hi - 1), np.clip(t.fly + f + 1, 0, t.Hi - 1), xlo, np.clip(t.flx + f + 1, 0, t.Wi))
        return check_fwd(r, emu_fwd(t2, a))
    return check_fwd(r, emu_fwd(t, a, fault))


FAULTS = {
    "dropped tap": lambda: _fault_fwd("drop_tap", "iid"),
    "clamp to Wi": lambda: _fault_fwd("clamp_wi", "outside"),
    "missing 1/sum": lambda: _fault_fwd("no_sum", "iid"),
}


def _fault_in1(fault):
    kind = "neg" if fault == "floor_frac" else "smooth"
    a, in2, g = std_case(kind)
    r = rr.resample2d(a, in2, 4, 1, g)
    tt = rr.Resample2d(in2, 4, 1, *a.shape[2:], trunc=fault != "floor_frac")
    fast = rr.fast_warps(in2, 4, 1, *a.shape[2:])
    if fault == "drop_oos":
        assert fast.mean() > 0.5
    return check_in1(r, emu_in1(tt, g, "seq", fault=fault, fast=fast))


FAULTS["floor for the grad_input1 fraction"] = lambda: _fault_in1("floor_frac")
FAULTS["dropped out-of-span partial"] = lambda: _fault_in1("drop_oos")


def _fault_in2(fault):
    a, in2, g = std_case("iid")
    r = rr.resample2d(a, in2, 4, 1, g)
    return check_in2(r, emu_in2(r["taps"], a, g, fault))


for _f, _n in [("swap_xy", "exchanged dx/dy planes"), ("sgrad_sign", "sign of sgrad wd"),
               ("drop_dsigma", "dropped dsigma term"), ("swap_tltr", "TL/TR swap in D")]:
    FAULTS[_n] = (lambda f: lambda: _fault_in2(f))(_f)


def _fault_cos(fault, name):
    a, in2, t, gc, ks, dil = cos_case()
    c = rr.cosine(a, in2, t, ks, dil, EPS, gc)
    res = cos_checks(c, emu_cos(c["taps"], a, t, gc, 4, fault))
    return res[("cos", "stats", "gval", "gt", "gin2").index(name)]


FAULTS["cosine slice missing"] = lambda: _fault_cos("drop_slice", "stats")
FAULTS["eps clamp on |v|^2"] = lambda: _fault_cos("clamp_vv", "stats")
FAULTS["k2v on the wrong side of eps"] = lambda: _fault_cos("k2v_flip", "gval")
FAULTS["grad_target without k2t"] = lambda: _fault_cos("no_k2t", "gt")


@pytest.mark.parametrize("fault", sorted(FAULTS))
def test_injected_fault_fails_its_bound(fault):
    worst, msg = FAULTS[fault]()
    assert msg is not None, f"{fault}: worst |err|/bound {worst:.3g} stays within the bound"


# ------------------------------------------------------------------------------------------------ host predicates
def test_fast_path_predicate():
    B, C, Hi, Wi, H, W = STD
    rng = np.random.default_rng(0)
    smooth = make_in2("smooth", rng, B, H, W, Hi, Wi, 2.0, f32)
    f = rr.fast_warps(smooth, 4, 1, Hi, Wi)
    assert f.shape == (B, H, 2) and f.all()                              # interior, one shift per warp
    assert not rr.fast_warps(smooth, 4, 2, Hi, Wi).any()                 # dilation
    assert not rr.fast_warps(smooth, 6, 1, Hi, Wi).any()                 # NT = 3
    assert not rr.fast_warps(smooth[..., :60], 4, 1, Hi, Wi)[..., 1].any()   # inactive lanes in the last warp
    torn = make_in2("torn", rng, B, H, W, Hi, Wi, 2.0, f32)
    assert not rr.fast_warps(torn, 4, 1, Hi, Wi).any()
    out = make_in2("outside", rng, B, H, W, Hi, Wi, 2.0, f32)
    assert not rr.fast_warps(out, 2, 1, Hi, Wi).any()


def test_cosine_slicing_predicate():
    # a batch of 8 at 256 x 176: VGG relu2_1 (128 x 88, 128 channels) and relu3_1 (64 x 44, 256) slice on a 114-SM and on
    # a 132-SM H100; 120,000 pixels slice only on the larger part; C < 64 and NT > 2 never do
    for sm in (114, 132):
        assert rr.cos_slices(8, 128, 128, 88, 4, sm) == 4
        assert rr.cos_slices(8, 256, 64, 44, 4, sm) == 4
        assert rr.cos_slices(8, 32, 64, 44, 4, sm) == 1
        assert rr.cos_slices(8, 256, 64, 44, 6, sm) == 1
    assert rr.cos_slices(1, 64, 300, 400, 4, 114) == 1
    assert rr.cos_slices(1, 64, 300, 400, 4, 132) == 4


def degenerate_case(dt, sigma=0.02, kind="iid"):
    """sigma small enough that weights leave the normal range (fp32: sum and sum*sum reach 0; fp64: sum*sum subnormal)"""
    B, C, Hi, Wi, H, W = 2, 5, 13, 70, 13, 70
    rng = np.random.default_rng(9)
    in2 = make_in2(kind, rng, B, H, W, Hi, Wi, sigma, dt)
    return rng.standard_normal((B, C, Hi, Wi)).astype(dt), in2, rng.standard_normal((B, C, H, W)).astype(dt)


@pytest.mark.parametrize("dt", [f32, f64])
def test_degenerate_grad_input2_bound(oracle_lib, dt):
    """bound_in2_vs_oracle: the fp32 emulation of the kernel (the fp64 reference for fp64) agrees with the oracle at a
    sigma whose weights leave A's normal range; exchanged planes or a flipped sign do not"""
    a, in2, g = degenerate_case(dt)
    r = rr.resample2d(a, in2, 4, 1, g)
    t = r["taps"]
    assert t.s2_zero.any() if dt == f32 else ((t.sum ** 2 < np.finfo(f64).tiny) & ~t.s2_zero).any()
    o2 = oracle_lib.resample2d_bwd(a, in2, g, 4, 1)[1]
    y = emu_in2(t, a, g) if dt == f32 else r["gin2"]
    bound = rr.bound_in2_vs_oracle(r, a, g, o2)
    assert ref64.check("in2 degenerate", y, o2, bound)[1] is None
    assert ref64.check("in2 planes exchanged", y[:, [1, 0, 2]], o2, bound)[1] is not None
    assert ref64.check("in2 sign flipped", -y, o2, bound)[1] is not None
