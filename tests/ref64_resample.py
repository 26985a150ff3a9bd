"""fp64 reference of resample2d (forward, grad_input1, grad_input2) and of the fused resample2d -> cosine op, with the
magnitudes that bound what the fp32 and fp64 kernels of csrc/resample2d.cu may return.

The reference takes the kernels' discrete decisions in their own arithmetic type A (fp32 for fp32 calls, fp64 for fp64
calls), exactly as rs_setup does (resample2d.cu:65-100): xf = x + dx in A, floor, the truncating int() fraction of
grad_input1, the distances xL_ .. yB_ in A, the clamped tap indices, and the SAFE_DIV branches 2 sigma^2 == 0 (inside
exp), sum == 0, sum*sum == 0 and sigma == 0 (rs_in2_store).  Everything else runs in fp64 on those A values: the Gaussian
factors, the weights and their sum, the forward, the grad_input1 scatter, the corner dot products and all three
grad_input2 planes, the cosine and its gradients with both eps clamps.  It is written from the operation's definition,
not from oracle/.

Next to every value it returns the magnitudes a rounding analysis needs, and the bound_* functions turn them into a
per-element bound |y - ref| <= bound for the unit roundoff u of A (unit(dtype)).  ref64.assert_within checks a kernel
output against one.  See DESIGN.md section 6.
"""
import numpy as np
import scipy.sparse as sps

from ref64 import gamma

U32, U64 = 2.0 ** -24, 2.0 ** -53
# absolute floor: a Gaussian factor or weight below A's smallest normal number is off by up to half a subnormal spacing
# (2^-150 in fp32, 2^-1075 in fp64), not by u of itself.  The sums here have at most 64 such terms, |source|, |grad| <= 2^6
# and sum >= e^-4 (sigma >= 0.5 puts the nearest tap within 1 of the pixel): together far below 2^-120 (2^-1000).
ETA32, ETA64 = 2.0 ** -120, 2.0 ** -1000
SAFE_EPS = 1e-8          # SAFE_DIV's double 1e-8 (resample2d.cu:32-34)


def unit(dtype):
    """-> (u, eta) of the kernels' arithmetic type"""
    return (U32, ETA32) if np.dtype(dtype) == np.float32 else (U64, ETA64)


def gam(n, u):
    """ref64.gamma(n) = 4 n 2^-24 for n A-products summed in A, scaled to A's unit roundoff"""
    return gamma(n) * (u / U32)


def fast_warps(in2, ks, dil, Hi, Wi):
    """Per warp, (B, H, ceil(W/32)) bools: does k_resample2d_bwd_in1 take the shuffle-merged scatter (resample2d.cu:175-186)?
    NT <= 2 and dil == 1, all 32 lanes active, every tap inside the source, and one integer shift flx - x and one fly for
    the whole warp.  flx, fly are floor(x + dx), floor(y + dy) in A."""
    in2 = np.asarray(in2)
    B, _, H, W = in2.shape
    NT, nw = ks // 2, (W + 31) // 32
    if NT > 2 or dil != 1:
        return np.zeros((B, H, nw), bool)
    A = in2.dtype.type
    xs = np.arange(W).astype(A)
    flx = np.floor(xs + in2[:, 0]).astype(np.int64)
    fly = np.floor(np.arange(H).astype(A)[:, None] + in2[:, 1]).astype(np.int64)
    ok = (flx - (NT - 1) >= 0) & (flx + NT <= Wi - 1) & (fly - (NT - 1) >= 0) & (fly + NT <= Hi - 1)
    pad = nw * 32 - W                                      # inactive lanes of the last warp vote no
    ok = np.pad(ok, ((0, 0), (0, 0), (0, pad)), constant_values=False).reshape(B, H, nw, 32)
    shift = np.pad(flx - np.arange(W), ((0, 0), (0, 0), (0, pad)), mode="edge").reshape(B, H, nw, 32)
    fy = np.pad(fly, ((0, 0), (0, 0), (0, pad)), mode="edge").reshape(B, H, nw, 32)
    return ok.all(-1) & (shift == shift[..., :1]).all(-1) & (fy == fy[..., :1]).all(-1)


def cos_slices(B, C, H, W, ks, sm_count):
    """channel slices TS of the fused cosine kernels on a GPU with sm_count SMs: rs_cos_slices (resample2d.cu:463-466),
    and only windows with NT <= 2 have a sliced instance (rs_launch_cos_fwd)"""
    return 4 if ks // 2 <= 2 and C >= 64 and B * H * W < sm_count * 1024 else 1


class Resample2d:
    """Taps and weights of every pixel of a flow in2 = [B, 3, H, W] (dx, dy, sigma) over a source of Hi x Wi.
    trunc=True: the Gaussian distances use xf - int(xf), as grad_input1 does (resample2d.cu:72-73, 159); the tap
    indices always use floor.  Taps q = (fy NT + fx) 4 + corner, corners TL, TR, BL, BR, arrays of shape (n, B, H W)."""

    def __init__(self, in2, ks, dil, Hi, Wi, trunc=False):
        in2 = np.asarray(in2)
        A = in2.dtype.type
        assert A in (np.float32, np.float64), in2.dtype
        assert 2 <= ks, ks
        self.A = A
        self.u, self.eta = unit(A)
        self.B, _, self.H, self.W = in2.shape
        self.Hi, self.Wi, self.ks, self.dil = Hi, Wi, ks, dil
        NT = self.NT = ks // 2
        self.n = n = 4 * NT * NT
        B, H, W = self.B, self.H, self.W
        dx, dy, sig = in2[:, 0], in2[:, 1], in2[:, 2]
        xf = np.arange(W).astype(A) + dx                                   # A
        yf = np.arange(H).astype(A)[:, None] + dy
        flx, fly = np.floor(xf), np.floor(yf)
        alpha = xf - (np.trunc(xf) if trunc else flx)                     # exact in A
        beta = yf - (np.trunc(yf) if trunc else fly)
        f = np.arange(NT).reshape(NT, 1, 1, 1)
        xL = (f * dil).astype(A) + alpha                                   # the distances, rounded in A
        xR = ((1 + f) * dil).astype(A) - alpha
        yT = (f * dil).astype(A) + beta
        yB = ((1 + f) * dil).astype(A) - beta
        two_s2 = A(2) * sig * sig                                          # A
        g0 = two_s2 == 0                                                   # SAFE_DIV's branch inside exp
        self.dist, self.two_s2 = (xL, xR, yT, yB), two_s2

        def gauss(d):
            """Gaussian factor exp(-d^2 / (2 sigma^2)) in fp64 and the size of its exponent"""
            num = -(np.asarray(d, np.float64) ** 2)                       # exact for fp32 d
            q = num / np.where(g0, SAFE_EPS, two_s2.astype(np.float64))
            return np.exp(q), -q

        (xLP, xLq), (xRP, xRq), (yTP, yTq), (yBP, yBq) = gauss(xL), gauss(xR), gauss(yT), gauss(yB)
        Y, X = (yTP, yTP, yBP, yBP), (xLP, xRP, xLP, xRP)
        YQ, XQ = (yTq, yTq, yBq, yBq), (xLq, xRq, xLq, xRq)
        w = np.empty((NT, NT, 4, B, H, W))
        Q = np.empty_like(w)
        for c in range(4):
            w[:, :, c] = Y[c][:, None] * X[c][None]
            Q[:, :, c] = YQ[c][:, None] + XQ[c][None]
        # coefficients of rs_in2_store (resample2d.cu:247-253): d/dx, d/dy and d/dsigma of each weight, up to 1/den
        xd, yd = np.asarray(xL, np.float64), np.asarray(yT, np.float64)
        xr, yb = np.asarray(xR, np.float64), np.asarray(yB, np.float64)
        ax = np.stack(np.broadcast_arrays(xd[None], -xr[None], xd[None], -xr[None]), 2)   # (1, NT, 4, ...)
        ay = np.stack(np.broadcast_arrays(yd[:, None], yd[:, None], -yb[:, None], -yb[:, None]), 2)
        rr = np.stack([yd[:, None] ** 2 + xd[None] ** 2, yd[:, None] ** 2 + xr[None] ** 2,
                       yb[:, None] ** 2 + xd[None] ** 2, yb[:, None] ** 2 + xr[None] ** 2], 2)
        shp = (n, B, H * W)
        self.a = [np.broadcast_to(c, w.shape).reshape(shp) for c in (ax, ay, rr)]
        self.w, self.Q = w.reshape(shp), Q.reshape(shp)
        self.sum = self.w.sum(0)                                           # (B, H W)
        sA = self.sum.astype(A)
        self.s_zero = sA == 0                                              # SAFE_DIV(., sum)
        self.s2_zero = (sA * sA) == 0                                      # SAFE_DIV(., sum*sum), rs_in2_store
        safe = np.where(self.s_zero, 1.0, self.sum)
        # quotients, as the kernels form them: x / sum (x / 1e-8 in the zero branch), and x y / sum^2 as
        # (x / den2)(y / den2) with den2 = sum, which stays finite where sum^2 is below fp64's range (x y / 1e-8 in the
        # zero branch of sum*sum: den2 = 1e-4)
        self.den1 = np.where(self.s_zero, SAFE_EPS, self.sum)
        self.den2 = np.where(self.s2_zero, 1e-4, safe)
        self.Qs = (self.w * self.Q).sum(0) / safe                          # exponent size averaged over the weights
        sg = np.asarray(sig, np.float64).reshape(B, H * W)
        z = sig.reshape(B, H * W) == 0                                     # rs_in2_store's sigma == 0 branch
        self.den = [np.where(z, SAFE_EPS, -sg * sg), np.where(z, SAFE_EPS, -sg * sg), np.where(z, SAFE_EPS, sg ** 3)]
        # clamped tap indices (resample2d.cu:89-99), floor in A
        fl_x, fl_y = flx.astype(np.int64), fly.astype(np.int64)
        fi = np.arange(NT).reshape(NT, 1, 1, 1)
        xlo, xhi = np.clip(fl_x - fi * dil, 0, Wi - 1), np.clip(fl_x + (fi + 1) * dil, 0, Wi - 1)
        ylo, yhi = np.clip(fl_y - fi * dil, 0, Hi - 1), np.clip(fl_y + (fi + 1) * dil, 0, Hi - 1)
        self.flx, self.fly = fl_x, fl_y
        self.set_taps(ylo, yhi, xlo, xhi)

    def set_taps(self, ylo, yhi, xlo, xhi):
        """tap positions from the per-axis clamped indices (tests edit these to inject faults)"""
        NT, B, HW = self.NT, self.B, self.H * self.W
        Yi, Xi = (ylo, ylo, yhi, yhi), (xlo, xhi, xlo, xhi)
        off = np.empty((NT, NT, 4) + ylo.shape[1:], np.int64)
        for c in range(4):
            off[:, :, c] = Yi[c][:, None] * self.Wi + Xi[c][None]
        self.off = off.reshape(self.n, B, HW)
        self._mats = {}

    def mat(self, data):
        """one sparse (H W) x (Hi Wi) matrix per image with entries data[q] at (pixel, tap q); duplicates are summed"""
        rows = np.broadcast_to(np.arange(self.H * self.W), (self.n, self.H * self.W))
        N = max(int(self.off.max()) + 1, self.Hi * self.Wi)
        return [sps.csr_matrix((data[:, b].ravel(), (rows.ravel(), self.off[:, b].ravel())), shape=(self.H * self.W, N))
                [:, :self.Hi * self.Wi] for b in range(self.B)]

    def _apply(self, mats, a, transpose=False):
        B, C = a.shape[:2]
        a = np.asarray(a, np.float64).reshape(B, C, -1)
        return np.stack([((m.T if transpose else m) @ a[b].T).T for b, m in enumerate(mats)])

    # ------------------------------------------------------------------------------------------------ forward
    def fwd(self, src):
        """-> out [B, C, H, W], mags: M = sum w|s| / sum, MQ = sum Q w |s| / sum (Q: size of the weight's exponents)"""
        src = np.asarray(src, np.float64)
        sh = (self.B, src.shape[1], self.H, self.W)
        wn = self.w / self.den1
        out = self._apply(self.mat(wn), src).reshape(sh)
        M = self._apply(self.mat(wn), np.abs(src)).reshape(sh)
        MQ = self._apply(self.mat(wn * self.Q), np.abs(src)).reshape(sh)
        hw = (self.B, 1, self.H, self.W)
        return out, {"M": M, "MQ": MQ, "Qs": self.Qs.reshape(hw), "n": self.n}

    # ------------------------------------------------------------------------------------------ grad_input1
    def bwd_in1(self, gout, gerr=None):
        """the scatter sum_{pixel, tap -> element} w / sum * g (build with trunc=True).  -> gin1 [B, C, Hi, Wi], mags:
        G1 = sum |partials|, G1Q = sum (Q + Qs) |partial|, m = partials per element, Gerr = the scatter of gerr (an
        error bound of gout, e.g. the fused backward's grad_val)"""
        g = np.asarray(gout, np.float64)
        sh = (self.B, g.shape[1], self.Hi, self.Wi)
        wn = self.w / self.den1
        r = self._apply(self.mat(wn), g, True).reshape(sh)
        G1 = self._apply(self.mat(wn), np.abs(g), True).reshape(sh)
        G1Q = self._apply(self.mat(wn * (self.Q + self.Qs[None])), np.abs(g), True).reshape(sh)
        m = np.stack([np.bincount(self.off[:, b].ravel(), minlength=self.Hi * self.Wi)[:self.Hi * self.Wi]
                      for b in range(self.B)]).reshape(self.B, 1, self.Hi, self.Wi).astype(np.float64)
        mags = {"G1": G1, "G1Q": G1Q, "m": m, "n": self.n}
        mags["Gerr"] = 0.0 if gerr is None else self._apply(self.mat(wn), gerr, True).reshape(sh)
        return r, mags

    # ------------------------------------------------------------------------------------------ grad_input2
    def corner(self, G, S):
        """corner dot products sum_c G[b, c, pixel] S[b, c, tap q] -> (n, B, H W)"""
        G = np.asarray(G, np.float64).reshape(self.B, G.shape[1], -1)
        S = np.asarray(S, np.float64).reshape(self.B, S.shape[1], -1)
        out = np.empty((self.n, self.B, self.H * self.W))
        for b in range(self.B):
            for q in range(self.n):
                out[q, b] = np.einsum("ch,ch->h", G[b], S[b][:, self.off[q, b]])
        return out

    def bwd_in2(self, D, Derr, Dabs):
        """d/d(dx, dy, sigma) from the corner dot products D (n, B, H W), as rs_in2_store (resample2d.cu:232-264) in fp64:
        g1 / sum - sgrad wd / sum^2 per plane.  Derr: a bound on the error of the kernel's D; Dabs: the sums of the
        absolute values of D's terms.  -> r [B, 3, H, W], mags with every term's absolute value: A1 = sum |a w D / den|
        / sum (g1 / sum), S = sum |a w / den| / sum (sgrad), Wd = sum w |D| / sum (wd), their Q-weighted forms and
        their Derr forms; T = the absolute sum of every per-channel term, sum |a w / den| Dabs / sum + S sum w Dabs / sum"""
        w, Q, d1, d2 = self.w, self.Q, self.den1, self.den2
        wd = (w * D).sum(0)
        aD = np.abs(D)
        WDabs = (w * Dabs).sum(0) / d2
        r, mags = [], {k: [] for k in ("A1", "A1q", "Aerr", "S", "Sq", "G1", "SG", "T")}
        for a, den in zip(self.a, self.den):
            g1 = (a * w * D).sum(0) / den
            sgrad = (a * w).sum(0) / den
            r.append(g1 / d1 - (sgrad / d2) * (wd / d2))
            aw = np.abs(a) * w / np.abs(den)
            mags["A1"].append((aw * aD).sum(0) / d1)
            mags["A1q"].append((aw * Q * aD).sum(0) / d1)
            mags["Aerr"].append((aw * Derr).sum(0) / d1)
            mags["S"].append(aw.sum(0) / d2)
            mags["Sq"].append((aw * Q).sum(0) / d2)
            mags["G1"].append(np.abs(g1) / d1)
            mags["SG"].append(np.abs(sgrad) / d2)
            mags["T"].append((aw * Dabs).sum(0) / d1 + mags["S"][-1] * WDabs)
        sh = (self.B, 3, self.H, self.W)
        out = {k: np.stack(v, 1).reshape(sh) for k, v in mags.items()}
        hw = (self.B, 1, self.H, self.W)
        out.update(Wd=((w * aD).sum(0) / d2).reshape(hw), Wdq=((w * Q * aD).sum(0) / d2).reshape(hw),
                   Werr=((w * Derr).sum(0) / d2).reshape(hw), WD=(np.abs(wd) / d2).reshape(hw), Qs=self.Qs.reshape(hw),
                   n=self.n)
        return np.stack(r, 1).reshape(sh), out


def resample2d(in1, in2, ks, dil, gout=None):
    """fp64 resample2d of in1 [B, C, Hi, Wi] by in2 in in2's arithmetic type.  -> dict: out and mags_out; with gout also
    gin1 / mags_in1 (the truncating weights) and gin2 / mags_in2, and the corner magnitudes Dabs"""
    Hi, Wi = in1.shape[2:]
    fw = Resample2d(in2, ks, dil, Hi, Wi)
    r = {"taps": fw}
    r["out"], r["mags_out"] = fw.fwd(in1)
    if gout is not None:
        bw = Resample2d(in2, ks, dil, Hi, Wi, trunc=True)
        r["gin1"], r["mags_in1"] = bw.bwd_in1(gout)
        D, r["Dabs"] = fw.corner(gout, in1), fw.corner(np.abs(gout), np.abs(in1))
        r["gin2"], r["mags_in2"] = fw.bwd_in2(D, gam(in1.shape[1], fw.u) * r["Dabs"], r["Dabs"])
    return r


def cosine(in1, in2, target, ks, dil, eps, gcos=None):
    """fp64 cos = sum_c v_c / max(|v|, eps) * t_c / max(|t|, eps) of the warped v = resample2d(in1, in2) and the target
    (ATen's cosine_similarity, each norm clamped), stats (v.t, |v|, |t|); with gcos the gradients grad_val = dcos/dv gcos,
    grad_target, grad_input2 (through the corner products of grad_val) and grad_input1 (the scatter of grad_val).  The
    bounds of the chain are computed here as well (they need the forward's per-element bound): keys e_*."""
    fw = Resample2d(in2, ks, dil, *in1.shape[2:])
    u, eta = fw.u, fw.eta
    C = in1.shape[1]
    v, mv = fw.fwd(in1)
    ev = bound_fwd(v, mv, u, eta)
    t = np.asarray(target, np.float64)
    at, av = np.abs(t), np.abs(v)
    dot, vv, tt = (v * t).sum(1), (v * v).sum(1), (t * t).sum(1)
    nv, nt = np.sqrt(vv), np.sqrt(tt)
    a, bb = np.maximum(nv, eps), np.maximum(nt, eps)
    r = {"taps": fw, "v": v, "cos": dot / (a * bb), "stats": np.stack([dot, nv, nt], 1), "nv": nv, "nt": nt}
    # what the kernel rounds (resample2d.cu:330-353): v_c (bound_fwd), C + TS fp32 products and adds per sum (TS <= 4
    # slices combined in shared memory, :345-348), sqrt (u), the clamped product and the quotient (2 u)
    g4 = gam(C + 4, u)
    e_dot = (at * ev).sum(1) + g4 * (av * at).sum(1)
    e_vv = 2.02 * (av * ev).sum(1) + g4 * vv
    e_tt = g4 * tt
    e_nv = np.minimum(e_vv / (2 * np.where(nv > 0, nv, 1.0)), np.sqrt(e_vv)) + u * nv
    e_nt = np.minimum(e_tt / (2 * np.where(nt > 0, nt, 1.0)), np.sqrt(e_tt)) + u * nt
    e_a, e_b = np.where(nv > eps, e_nv, 0.0), np.where(nt > eps, e_nt, 0.0)
    r["e_stats"] = 1.01 * np.stack([e_dot, e_nv, e_nt], 1) + eta
    r["e_cos"] = 1.01 * (e_dot / (a * bb) + np.abs(r["cos"]) * (e_a / a + e_b / bb + 2 * u)) + eta
    r["mags_cos"] = {"VT": (av * at).sum(1), "VV": vv, "TT": tt}
    if gcos is None:
        return r
    g = np.asarray(gcos, np.float64)
    k1 = g / (a * bb)
    k2v = np.where(nv > eps, g * dot / (a * a * bb * np.where(nv > 0, nv, 1.0)), 0.0)
    k2t = np.where(nt > eps, g * dot / (a * bb * bb * np.where(nt > 0, nt, 1.0)), 0.0)
    gv = k1[:, None] * t - k2v[:, None] * v
    gt = k1[:, None] * v - k2t[:, None] * t
    # the backward reads the forward's stats (resample2d.cu:389-394): their errors, then 2 (k1) or 5 (k2v, k2t) A roundings
    e_k1 = np.abs(k1) * (e_a / a + e_b / bb + 2 * u)
    sv, st_ = np.where(nv > 0, nv, 1.0), np.where(nt > 0, nt, 1.0)
    e_k2v = np.where(nv > eps, np.abs(k2v) * (2 * e_a / a + e_b / bb + e_nv / sv + 5 * u)
                     + np.abs(g) * e_dot / (a * a * bb * sv), 0.0)
    e_k2t = np.where(nt > eps, np.abs(k2t) * (e_a / a + 2 * e_b / bb + e_nt / st_ + 5 * u)
                     + np.abs(g) * e_dot / (a * bb * bb * st_), 0.0)
    K1, K2v, K2t = (x[:, None] for x in (k1, k2v, k2t))
    # g_c = k1 t_c - k2v v_c (:410): two products and a difference in A
    e_gv = 1.01 * (e_k1[:, None] * at + e_k2v[:, None] * av + np.abs(K2v) * ev
                   + 2 * u * (np.abs(K1) * at + np.abs(K2v) * av)) + eta
    e_gt = 1.01 * (e_k1[:, None] * av + np.abs(K1) * ev + e_k2t[:, None] * at
                   + 2 * u * (np.abs(K1) * av + np.abs(K2t) * at))
    r.update(gval=gv, gt=gt, e_gval=e_gv, e_gt=e_gt)
    # grad_input2: D_q = sum_c g_c tap_q in A (:412, + the slice combine :428-432)
    D = fw.corner(gv, in1)
    Derr = 1.01 * fw.corner(e_gv, np.abs(in1)) + g4 * fw.corner(np.abs(gv), np.abs(in1))
    r["gin2"], r["mags_in2"] = fw.bwd_in2(D, Derr, fw.corner(np.abs(gv), np.abs(in1)))
    bw = Resample2d(in2, ks, dil, *in1.shape[2:], trunc=True)
    r["gin1"], r["mags_in1"] = bw.bwd_in1(gv, gerr=e_gv)
    return r


# ----------------------------------------------------------------------------------------------------------- bounds
# Each returns the per-element bound on |y - ref|.  u, eta: unit(dtype).  init: what an accumulate=1 call's buffer held.
#
# One Gaussian factor P = exp(-d^2 / (2 sigma^2)) with exponent size q (rs_setup, resample2d.cu:83-86): -d*d, 2*sigma*sigma
# and their quotient are rounded in A (3 u of q, so 3.02 u q of P: the error grows with the argument), exp runs in double
# (<= 1 ulp = 2 u in fp64) and is narrowed to A (u): 3 u + 3.02 u q.  A weight yP * xP (:129-130, 245-246) adds one more
# rounding: 7 u + 3.02 u Q with Q the two exponents' sum.  The weight sum (rs_weight_sum, :104-111): those errors plus
# gam(n) for its n adds, so relative e_s = 7 u + gam(n) + 3.02 u Qs.

def _e_sum(m, u):
    return 7 * u + gam(m["n"], u) + 3.02 * u * m["Qs"]


def bound_fwd(r, m, u, eta):
    """forward (k_resample2d_fwd, :137-143): val = sum of n products in A (gam(n) of M), weight errors (7 u M + 3.02 u
    MQ), the sum's error against |r|, and the quotient val / sum rounded in A (u |r|)"""
    return 1.01 * ((7 * u + gam(m["n"], u)) * m["M"] + 3.02 * u * m["MQ"] + _e_sum(m, u) * np.abs(r)) + u * np.abs(r) + eta


def bound_in1(r, m, u, eta, init=0.0):
    """grad_input1 (k_resample2d_bwd_in1): each partial w / sum * g carries the weight's (7 u + 3.02 u Q) and the sum's
    error (e_s), the quotient w / sum rounded in A (:167-168, u) and the narrowing of w/sum * g to A (:211, :226, u):
    16 u + gam(n) + 3.02 u (Q + Qs) of |partial|, i.e. of G1, G1Q.  The m partials and the buffer's initial value are
    summed in A in any order -- atomics, and in the shuffle path an A sum over a tap row first (:207-216) -- : gam(m + 1)
    of their absolute sum.  Gerr: the scatter of an error already in g."""
    return (1.01 * ((16 * u + gam(m["n"], u)) * m["G1"] + 3.02 * u * m["G1Q"] + m["Gerr"])
            + gam(m["m"] + 1, u) * (m["G1"] + np.abs(init)) + eta)


def bound_in2(r, m, u, eta, init=0.0):
    """grad_input2 plane by plane (rs_in2_store, :232-264).  g1 / sum: the weights' errors (7 u A1 + 3.02 u A1q), the
    corner products' (Aerr: gam(C) Dabs for k_resample2d_bwd_in2's A sums over C channels, :284-288) and the sum's
    (e_s |g1 / sum|).  sgrad wd / sum^2: the weights' errors in sgrad (7 u S + 3.02 u Sq) times |wd|, in wd (7 u Wd +
    3.02 u Wdq + Werr) times |sgrad|, and sum*sum rounded in A (2 e_s + u).  The combine runs in double (gam(n + 4) at
    2^-53 of every term).  One rounding to A (:261) and, with accumulate, one add (:262): u (|r| + |init|)"""
    es = _e_sum(m, u)
    t1 = 7 * u * m["A1"] + 3.02 * u * m["A1q"] + m["Aerr"] + es * m["G1"]
    t2 = ((7 * u * m["S"] + 3.02 * u * m["Sq"]) * m["WD"] + m["SG"] * (7 * u * m["Wd"] + 3.02 * u * m["Wdq"] + m["Werr"])
          + (2 * es + u) * m["SG"] * m["WD"])
    comb = gam(m["n"] + 4, U64) * (m["A1"] + m["S"] * m["Wd"])
    return 1.01 * (t1 + t2 + comb) + u * (np.abs(r) + np.abs(init)) + eta


def bound_in2_vs_oracle(r, in1, gout, oracle_y):
    """|kernel - oracle| for grad_input2 at any sigma, including the degenerate ones whose weights leave A's normal
    range (r = resample2d(in1, in2, ks, dil, gout)).  Both sum 4 n C + n terms in A or double (2 gam(4 n C + n) of T, the
    terms' absolute sum) and round once to A (u |y| each).  Below A's normal range a rounding is off by up to the
    subnormal spacing eta_s (2^-149 in fp32, 2^-1074 in fp64) absolutely, not relatively: the oracle forms each term
    as an A product chain (w.xL_ * w.yT_P * w.xL_P * g * v, like the reference) where the kernel multiplies the factors
    in double (rs_in2_store, :245-246), and each such rounding carries on through at most G = max |g| max |in1| of later
    factors.  Per plane, for either side: 4 n C + n of them, divided by |den| sum_A in g1 / sum and by the A-rounded
    sum*sum in sgrad wd / sum^2 (:257-261); the sum of n weights itself (eta_s n / sum_A relative, twice in the second
    term); and sum*sum rounded in A (eta_s / sum*sum relative).  Where every weight is a normal number these vanish
    against the first terms."""
    t, m = r["taps"], r["mags_in2"]
    A, u, n = t.A, t.u, t.n
    ops = 4 * n * in1.shape[1] + n
    eta_s = 2.0 ** -149 if A == np.float32 else 2.0 ** -1074
    G = max(1.0, float(np.abs(gout).max()) * float(np.abs(in1).max()))
    sA = t.sum.astype(A)
    hw = (t.B, 1, t.H, t.W)
    d1 = np.where(sA == 0, SAFE_EPS, sA.astype(np.float64)).reshape(hw)
    d2 = np.where(t.s2_zero, SAFE_EPS, (sA * sA).astype(np.float64)).reshape(hw)
    den = np.stack([np.abs(d) for d in t.den], 1).reshape(t.B, 3, t.H, t.W)
    r1, r2 = m["G1"], m["SG"] * m["WD"]
    # divisions ordered so that no intermediate leaves fp64's range
    sub = (ops * G * eta_s / d1) / den + ops * G * eta_s / d2 + (r1 + 2 * r2) * (n * eta_s / d1) + r2 * (eta_s / d2)
    return 2 * (gam(ops, u) * m["T"] + sub) + u * (np.abs(oracle_y) + np.abs(r["gin2"])) + t.eta


def bound_cos(c, u, eta):
    """cos (k_resample2d_cos_fwd :350-351): computed in cosine() from the forward's bound, see there"""
    return c["e_cos"]


def bound_stats(c, u, eta):
    """stats = (v.t, |v|, |t|) (:353): computed in cosine()"""
    return c["e_stats"]


def bound_gval(c, u, eta):
    """grad_val = k1 t - k2v v (:410), materialised for the grad_input1 scatter: computed in cosine()"""
    return c["e_gval"]


def bound_gt(c, u, eta, init=0.0):
    """grad_target = k1 v - k2t t (:415-416), with accumulate one more A add: e_gt of cosine() + u (|r| + |init|)"""
    return c["e_gt"] + u * (np.abs(c["gt"] + init) + np.abs(init)) + eta
