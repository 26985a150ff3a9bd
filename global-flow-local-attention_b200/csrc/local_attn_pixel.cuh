// Per-pixel arithmetic of the fused local-attention op, shared by the CUDA-core gather kernels (local_attn.cu) and the
// tensor-core tile kernels (tile_window.cuh): the softmax over the k*k logits, the tap test, the literal value of one tap
// and the backward formulas that turn one tap's grad_out . source dot products into d p, grad_flow and grad_logits.
// T = storage type, A = arithmetic type (float, or double for fp64).  Both paths evaluate these expressions with the
// same operands in the same order, so they round alike.
#pragma once
#include "common.cuh"

namespace gfla {

template <typename A> __device__ __forceinline__ A fexp(A v);
template <> __device__ __forceinline__ float fexp<float>(float v) { return expf(v); }
template <> __device__ __forceinline__ double fexp<double>(double v) { return exp(v); }

// softmax over the logits of one pixel (planes of stride hw) into p.  KK = k*k when known at compile time, else 0 and
// kk gives it.  fmax skips a NaN logit when taking the max, but the NaN still reaches the sum, so a NaN logit makes
// every probability of the pixel NaN.
template <typename T, typename A, int KK>
__device__ __forceinline__ void pixel_softmax(const T* __restrict__ lg, long long hw, int kk, A* p) {
    A m = -INFINITY;
#pragma unroll
    for (int t = 0; t < (KK ? KK : kk); ++t) {
        p[t] = ld(lg + t * hw);
        m = fmax(m, p[t]);
    }
    A s = static_cast<A>(0);
#pragma unroll
    for (int t = 0; t < (KK ? KK : kk); ++t) {
        p[t] = fexp<A>(p[t] - m);
        s += p[t];
    }
    const A inv = static_cast<A>(1) / s;
#pragma unroll
    for (int t = 0; t < (KK ? KK : kk); ++t) p[t] *= inv;
}

// the k taps per axis of pixel (x, y); true when each axis's taps are consecutive integers, which is when the 4*k*k
// bilinear taps collapse into a (k+1)x(k+1) window (always, except when rounding of (flow+offset)+coord straddles an
// integer)
template <typename A, int K>
__device__ __forceinline__ bool taps_regular(A flow_x, A flow_y, int x, int y, int Hs, int Ws, AxisTap<A> (&tx)[K],
                                             AxisTap<A> (&ty)[K]) {
    bool regular = true;
#pragma unroll
    for (int j = 0; j < K; ++j) {
        tx[j] = axis_tap<A>(flow_x, j - K / 2, x, Ws);
        ty[j] = axis_tap<A>(flow_y, j - K / 2, y, Hs);
        regular = regular && (tx[j].fl == tx[0].fl + j) && (ty[j].fl == ty[0].fl + j);
    }
    return regular;
}

// literal bilinear value of one tap from one channel plane s (sp = element stride of a source position)
template <typename T, typename A, typename I>
__device__ __forceinline__ A tap_value(const T* __restrict__ s, const AxisTap<A>& tx, const AxisTap<A>& ty, int Ws, I sp) {
    A v = static_cast<A>(0);
    v += tx.wlo * ty.wlo * ld(s + (ty.lo * Ws + tx.lo) * sp);
    v += tx.whi * ty.wlo * ld(s + (ty.lo * Ws + tx.hi) * sp);
    v += tx.wlo * ty.whi * ld(s + (ty.hi * Ws + tx.lo) * sp);
    v += tx.whi * ty.whi * ld(s + (ty.hi * Ws + tx.hi) * sp);
    return v;
}

// backward of one tap from q = sum_c grad_out[c] * source[c, corner] at its four corners: returns d loss / d p of the
// tap and adds the tap's share of d loss / d flow (pij = p of the tap times 1/k^2)
template <typename A>
__device__ __forceinline__ A tap_backward(const AxisTap<A>& tx, const AxisTap<A>& ty, A pij, A inv_kk, A qLT, A qRT, A qLB,
                                          A qRB, A& gfx, A& gfy) {
    const A dp = inv_kk * (ty.wlo * (tx.wlo * qLT + tx.whi * qRT) + ty.whi * (tx.wlo * qLB + tx.whi * qRB));
    gfy += pij * (-tx.wlo * qLT - tx.whi * qRT + tx.wlo * qLB + tx.whi * qRB);
    gfx += pij * (-ty.wlo * qLT - ty.whi * qLB + ty.wlo * qRT + ty.whi * qRB);
    return dp;
}

// softmax backward dl_t = p_t * (dp_t - sum_u p_u dp_u), stored to grad_logits (planes of stride hw from gl) and the
// flow gradient to grad_flow (x plane at gf, y plane at gf + hw); accumulate adds to what the buffers hold
template <typename T, typename TF, typename A, int KK>
__device__ __forceinline__ void store_pixel_grads(const A* p, const A* dp, int kk, A gfx, A gfy, T* __restrict__ gl,
                                                  TF* __restrict__ gf, long long hw, int accumulate) {
    A dot = static_cast<A>(0);
#pragma unroll
    for (int t = 0; t < (KK ? KK : kk); ++t) dot += p[t] * dp[t];
#pragma unroll
    for (int t = 0; t < (KK ? KK : kk); ++t) {
        const A v = p[t] * (dp[t] - dot);
        st(gl + t * hw, accumulate ? static_cast<A>(ld(gl + t * hw)) + v : v);
    }
    st(gf, accumulate ? static_cast<A>(ld(gf)) + gfx : gfx);
    st(gf + hw, accumulate ? static_cast<A>(ld(gf + hw)) + gfy : gfy);
}

}  // namespace gfla
