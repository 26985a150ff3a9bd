"""Bounds for the CUDA-core kernels in fp32 and fp64: the gather local attention (csrc/local_attn.cu with the per-pixel
arithmetic of csrc/local_attn_pixel.cuh) and block_extractor (csrc/block_extract.cu).

The fp64 reference is ref64's, with the taps selected in the kernel's arithmetic type A (fp32 for fp32 and 16-bit
storage, fp64 for fp64: Acc<T>, common.cuh:18-19).  Given those taps, every difference between a kernel and the
reference is rounding after tap selection.  This module adds the magnitudes a rounding analysis needs beyond ref64's
M, Mgs, D, PD, Mgf, and one bound per output for u = 2^-24 or 2^-53.  Each bound is a sum of magnitudes times counts of
roundings, each count commented with the line that rounds; gam(n) = 4 n u as ref64.gamma.  The reference performs the
same kinds of operations in fp64, in another order, so each bound is the analysis at u plus the same analysis at 2^-53
(uu = u + 2^-53 below): in fp32 that second part is negligible, in fp64 it is half the bound.  See DESIGN.md section 6.
"""
import numpy as np
import scipy.sparse as sps

import ref64

U32, U64 = 2.0 ** -24, 2.0 ** -53
# absolute floor.  A probability whose exp lands below A's normal range (fp32: logits 87 below the pixel's largest) is off
# by up to 2^-147 (fp32) or 2^-1072 (fp64) absolutely, not relatively: two ulps of expf / exp in the subnormal range and
# the multiply by 1/s, s >= 1.  Through at most 81 taps and values below 2^12 (C = 130 dot products of N(0, 1) values)
# that stays below 2^-120 (2^-1000).
ETA32, ETA64 = 2.0 ** -120, 2.0 ** -1000


def unit(A):
    """-> (u, eta) of the arithmetic type A (np.float32 or np.float64)"""
    return (U32, ETA32) if np.dtype(A) == np.float32 else (U64, ETA64)


def gam(n):
    """ref64.gamma(n) / 2^-24 = 4 n: multiply by u for n A-roundings"""
    return 4.0 * np.asarray(n, np.float64)


# ------------------------------------------------------------------------------------------- launch shapes (host mirror)
def channel_splits(items, C, threads, sm_count):
    """channel_splits (common.cuh:99-105): the power-of-two slice count the launchers start from"""
    ctas = (items + threads - 1) // threads
    want = 4 * sm_count * (2048 // threads)
    s = 1
    while ctas * s < want and s * 2 <= C and s < 64:
        s *= 2
    return s


def launch_slices(items, C, threads, sm_count):
    """-> (grid.y, channels per slice) of la_launch_fwd (local_attn.cu:244-245; items = B H W, 128 threads),
    launch_be_fwd (block_extract.cu:162-164; items = B k^2 H W, 256) and launch_be_bwd (:175-177; items = B H W, 128).
    The last slice holds C - (grid.y - 1) cps channels: ragged when that is below cps."""
    cps = -(-C // channel_splits(items, C, threads, sm_count))
    return -(-C // cps), cps


# ------------------------------------------------------------------------------------------------------ flows
def irregular_flow_values(xs, k, rng, A=np.float32):
    """flows f (for pixel column x) whose taps floor((f + (j - k/2)) + x), evaluated in A, are NOT consecutive in j: the
    rounding of the two additions straddles an integer for some taps only (block_extractor_kernel.cu:62-69).  The A = fp32
    search is test_gpu_parity._irregular_flow_values; in fp64 the flows lie within 2^-47 of an integer."""
    out = {}
    tiny = 4e-6 if np.dtype(A) == np.float32 else 8e-15
    for x in xs:
        for n in (-3, 0, 2, 5):
            for _ in range(4000):
                f = A(A(n) + A(rng.uniform(-tiny, tiny)))
                fl = [int(np.floor(A(A(f + A(j - k // 2)) + A(x)))) for j in range(k)]
                if any(fl[j] != fl[0] + j for j in range(k)):
                    out[x] = float(f)
                    break
            if x in out:
                break
    return out


# --------------------------------------------------------------------------------------------- local attention
def literal_path(taps):
    """(B, H W) bools: pixels that k_local_attn_fwd / _bwd run on the literal 4-taps-per-(i, j) path.  Only the K = 2..5
    instances have the collapsed window (GFLA_K_DISPATCH, local_attn.cu:271-278), and there only for pixels whose taps
    are consecutive (taps_regular)"""
    if 2 <= taps.k <= 5:
        return ~taps.regular
    return np.ones_like(taps.regular)


def partials(taps):
    """grad_source partials landing on each source position, per image (B, Hs Ws): the (k+1)^2 window cells of a
    collapsed pixel (local_attn.cu:199, clamped cells land twice), the 4 k^2 corners of a literal one (:227-230)"""
    k, B, N = taps.k, taps.B, taps.H * taps.W
    lit = literal_path(taps)
    y0 = taps.ty[2][0].reshape(B, N)
    x0 = taps.tx[2][0].reshape(B, N)
    r = np.arange(k + 1)
    out = np.zeros((B, taps.Hs * taps.Ws))
    for b in range(B):
        reg = ~lit[b]
        rows = np.clip(y0[b, reg][:, None] + r, 0, taps.Hs - 1)
        cols = np.clip(x0[b, reg][:, None] + r, 0, taps.Ws - 1)
        cells = rows[:, :, None] * taps.Ws + cols[:, None, :]
        out[b] = np.bincount(cells.ravel(), minlength=taps.Hs * taps.Ws)
        out[b] += np.bincount(taps.pos[b][:, :, :, lit[b]].ravel(), minlength=taps.Hs * taps.Ws)
    return out


class LocalAttn:
    """ref64.LocalAttn with the taps of a kernel computing in A, and the rounding magnitudes and bounds of the gather
    kernels.  R_t (per tap, dimensionless) is the relative error of probability t in units of u:

    pixel_softmax (local_attn_pixel.cuh:19-35): l_t - m rounds in A (u |l_t - m|, which exp turns into a relative error
    of that size: L_t below), expf is within 2 ulp and exp within 1 (4 u), the k^2 adds of s (gam(k^2) relative to s,
    all terms positive) plus the errors of the e_u it sums (sum_u p_u (4 + L_u)), 1 / s (1) and p_t = e_t * inv (1):
    R_t = 10 + gam(k^2) + L_t + PL, PL = sum_u p_u L_u, times 1.01 for second-order terms."""

    def __init__(self, flow, logits, k, Hs, Ws, A):
        self.A = A
        self.u, self.eta = unit(A)
        self.uu = self.u + U64
        self.k = k
        self.la = ref64.LocalAttn(flow, logits, k, Hs, Ws, A)
        t = self.taps = self.la.taps
        lg = np.asarray(logits, np.float64)
        self.L = lg.max(1, keepdims=True) - lg                       # |l_t - max_u l_u|
        p = self.la.p
        self.PL = (p * self.L).sum(1, keepdims=True)
        self.R = 1.01 * (10 + gam(k * k) + self.L + self.PL)         # (B, k^2, H, W)
        B, N = t.B, t.H * t.W
        wr = self.R.reshape(B, k, k, 1, N) * self.la.wts            # p_t R_t / k^2 * corner weight
        rows = np.broadcast_to(np.arange(N), t.pos.shape[1:])
        self.WR = [sps.csr_matrix((wr[b].ravel(), (rows.ravel(), t.pos[b].ravel())), shape=(N, t.Hs * t.Ws))
                   for b in range(B)]
        self.m = partials(t).reshape(B, 1, t.Hs, t.Ws)

    def probs(self):
        return self.la.p

    def fwd(self, src):
        """-> out, mags: M = W |S|, MR = sum over taps of R_t p_t / k^2 bilinear_t(|S|)"""
        out, M = self.la.fwd(src)
        MR = self.la._apply(self.WR, np.abs(np.asarray(src, np.float64)), (self.taps.H, self.taps.W))
        return out, {"M": M, "MR": MR}

    def bwd(self, src, gout):
        """-> ref64.LocalAttn.bwd's dict plus MRgs = WR^T |G|, MgfR (Mgf with each tap's p R), PRD = sum_u R_u p_u D_u"""
        r = self.la.bwd(src, gout)
        t, k = self.taps, self.k
        B, N = t.B, t.H * t.W
        r["MRgs"] = self.la._apply([w.T.tocsr() for w in self.WR], np.abs(np.asarray(gout, np.float64)), (t.Hs, t.Ws))
        pR = (self.la.p * self.R).reshape(B, k, k, N) / (k * k)
        r["MgfR"] = self.la.flow_mag(r["qa"], pR)
        r["PRD"] = (self.R * self.la.p * r["D"]).sum(1, keepdims=True)
        return r

    # ------------------------------------------------------------------------------------------------- bounds
    def bound_probs(self):
        """R_t p_t: the softmax above; stored in A without a further rounding"""
        return self.uu * self.R * self.la.p + self.eta

    def e_out(self, mags):
        """forward without the store (local_attn.cu:64-99 collapsed, :102-115 literal).  Probabilities: MR.  Per term at
        most 4 k^2 + 8 roundings: collapsed, wx wy and p (wx wy) (:79-82, 2) plus <= 4 adds into a Wc cell, the product
        with the source value and (k+1)^2 adds (:95); literal, wx wy and the product with the value (tap_value, 2), 4
        adds, p v and k^2 adds (:109).  All weights are >= 0, so the terms' absolute sum is M.  1/k^2 rounds for k not
        in {1, 2, 4, 8} (:59) and acc * inv_kk rounds (:96): 2 M."""
        k = self.k
        return self.uu * (mags["MR"] + (gam(4 * k * k + 8) + 2) * mags["M"])

    def bound_out(self, mags):
        """fp32 / fp64 storage: st() of an A value into A is exact"""
        return self.e_out(mags) + self.eta

    def bound_blend(self, rb, mags, prev, mask):
        """fused blend acc = prev (1 - m) + acc m (local_attn.cu:97, :113): the attention's error times m; 1 - m, the two
        products and the add round (2 |prev| (1 - m) + m M + |rb|)"""
        return mask * self.e_out(mags) + 1.01 * self.uu * (2 * np.abs(prev) * (1 - mask) + mask * mags["M"]
                                                            + np.abs(rb)) + self.eta

    def bound_gs(self, r, init=0.0):
        """grad_source: each partial g * Wc[cell] (local_attn.cu:199) or (g p_ij) (wx wy) (:226-230) carries its
        probability's R and 9 roundings (p * inv_kk and inv_kk itself, wx wy, the weight product, <= 4 adds into the
        Wc cell, the product with g); the m partials and the buffer's initial value are summed by fp32 / fp64 atomics
        in any order: gam(m + 1) of their absolute sum"""
        return self.uu * (r["MRgs"] + 9.09 * r["Mgs"] + gam(self.m + 1) * (r["Mgs"] + np.abs(init))) + self.eta

    def bound_gl(self, r, C, init=0.0):
        """grad_logits = p_t (dp_t - dot), dot = sum_u p_u dp_u (store_pixel_grads, local_attn_pixel.cuh:80-86).
        dp_t (tap_backward, :69): its four dot products over C channels (local_attn.cu:198, :225: gam(C) of |g|.|s|),
        5 roundings in the formula and 2 for inv_kk: (gam(C) + 7) D_t, with D_t >= |dp_t|.  dot: the p_u errors
        (PRD), the dp_u errors ((gam(C) + 7) PD) and k^2 products and adds (gam(k^2) PD).  The difference and the product
        with p_t round (2 (D_t + PD)), and p_t carries R_t.  With accumulate one more add (:86): |r| + |init|."""
        k, p, D, PD = self.k, self.la.p, r["D"], r["PD"]
        e = p * ((self.R + gam(C) + 9) * (D + PD) + r["PRD"] + gam(k * k) * PD)
        return self.uu * (1.01 * e + np.abs(r["gl"] + init) + np.abs(init)) + self.eta

    def bound_gf(self, r, C, init=0.0):
        """grad_flow (tap_backward, local_attn_pixel.cuh:70-71): per tap the dot products' gam(C), four products, three
        adds, the product with p_ij (p * inv_kk: R and 2 more) and the sum over the k^2 taps (gam(k^2)): of Mgf, with the
        probabilities' share MgfR.  The store (:88-89) rounds only with accumulate: |r| + |init|."""
        k = self.k
        e = r["MgfR"] + (gam(C) + 10 + gam(k * k)) * r["Mgf"]
        return self.uu * (1.01 * e + np.abs(r["gf"] + init) + np.abs(init)) + self.eta


# ------------------------------------------------------------------------------------------------ block_extractor
class BlockExtract:
    """ref64.block_extract with the taps of a kernel computing in A, and the bounds of k_block_extract_bwd (the forward
    is compared bit for bit with the oracle: block_extract.cu is built without FMA contraction)"""

    def __init__(self, src, flow, k, gout, A):
        self.A, self.k = A, k
        self.u, self.eta = unit(A)
        self.uu = self.u + U64
        self.r = ref64.block_extract(src, flow, k, gout, A)
        t = self.r["taps"]
        self.C = np.asarray(src).shape[1]
        # every corner of every tap of every flow pixel is one partial of its source position (block_extract.cu:99-102)
        self.m = np.stack([np.bincount(t.pos[b].ravel(), minlength=t.Hs * t.Ws) for b in range(t.B)]
                          ).reshape(t.B, 1, t.Hs, t.Ws).astype(np.float64)

    def bound_out(self):
        """forward in 16-bit storage (for ref64.bound_gather16): four products (wx wy) v, 2 roundings each, and 3 adds
        (block_extract.cu:40, :48-52): 5 roundings of M"""
        return self.uu * 5.05 * self.r["M"]

    def bound_gs(self, init=0.0):
        """grad_source: each partial (g wx) wy rounds twice (block_extract.cu:99-102); the m partials and the buffer's
        initial value are summed by atomics in any order: gam(m + 1)"""
        r = self.r
        return self.uu * (2.02 * r["Mgs"] + gam(self.m + 1) * (r["Mgs"] + np.abs(init))) + self.eta

    def bound_gf(self, init=0.0):
        """grad_flow: per term four products, three adds and the product with g (block_extract.cu:103-104, 8 roundings of
        Mgf); the k^2 C terms of a flow element and the buffer's initial value are summed in A in slices, and the slices'
        partial sums by atomics (:112-113) or one read-modify-write (:109-110): any order, gam(k^2 C + 1)"""
        r, n = self.r, self.k * self.k * self.C
        return self.uu * (8.08 * r["Mgf"] + gam(n + 1) * (r["Mgf"] + np.abs(init))) + self.eta
