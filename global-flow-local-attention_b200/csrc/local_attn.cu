// Fused local attention (the tail of ExtractorAttn.forward,
// model/networks/base_function.py:804-810): CUDA-core "gather" kernels.
//
//   out[b,c,y,x] = 1/k^2 * sum_{i,j<k} softmax(logits[b,:,y,x])[i*k+j]
//                        * bilinear(source[b,c], y + flow_y + i - k/2, x + flow_x + j - k/2)
//
// with the bilinear tap arithmetic of block_extractor_kernel.cu:57-82 (replicate
// border by index clamp, weights from the unclamped fraction).  The
// [B,C,k*H,k*W] block tensor, the reshaped attention map and the product are
// never materialised.
//
// These kernels serve every dtype / k / shape (they are what fp32, fp64 and
// small or odd shapes run on: everything the tensor-core tile kernels in
// local_attn_tc.cu / local_attn_bwd_tc.cu do not serve).  One thread owns one output pixel:
//   * softmax over the k*k logits in registers (coalesced plane-strided loads);
//   * when the k taps along each axis are consecutive integers (always, except
//     when fp32 rounding of (flow+offset)+coord straddles an integer) the
//     4*k*k bilinear taps collapse into a (k+1)x(k+1) window whose weights are
//     computed once per pixel and reused for every channel;
//   * otherwise the pixel takes the literal 4-taps-per-(i,j) path.
#include "det_accum.cuh"
#include "local_attn_pixel.cuh"

namespace gfla {

constexpr int kMaxK = 9;

// ---------------------------------------------------------------------------
// forward
// ---------------------------------------------------------------------------
template <typename T, typename TF, int K>  // K = 0: run-time k (literal path only)
__global__ void __launch_bounds__(128)
k_local_attn_fwd(const T* __restrict__ src, const TF* __restrict__ flow, const T* __restrict__ logits,
                 T* __restrict__ out, T* __restrict__ probs, const T* __restrict__ prev, const T* __restrict__ mask, int B,
                 int C, int Hs, int Ws, int H, int W, int k_rt, int c_per_slice, int nhwc) {
    using A = typename Acc<T>::type;
    const int k = K ? K : k_rt, KK = k * k;
    const long long hw = (long long)H * W, total = (long long)B * hw;
    const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= total) return;
    const int x = (int)(pix % W), y = (int)((pix / W) % H), b = (int)(pix / hw);
    const long long pofs = (long long)y * W + x;

    A p[K ? K * K : kMaxK * kMaxK];
    pixel_softmax<T, A, K * K>(logits + (long long)b * KK * hw + pofs, hw, KK, p);
    if (probs != nullptr && blockIdx.y == 0) {
        T* pr = probs + (long long)b * KK * hw + pofs;
        for (int t = 0; t < KK; ++t) st(pr + t * hw, p[t]);
    }
    const A flow_x = static_cast<A>(ld(flow + (long long)b * 2 * hw + pofs));
    const A flow_y = static_cast<A>(ld(flow + (long long)b * 2 * hw + hw + pofs));
    const long long spl = (long long)Hs * Ws;
    const int c0 = blockIdx.y * c_per_slice, c1 = min(C, c0 + c_per_slice);
    // element strides (channel, position): NCHW planes or channels-last pixels
    const long long sc = nhwc ? 1 : spl, oc = nhwc ? 1 : hw;
    const int sp = nhwc ? C : 1;
    const T* s = src + (long long)b * C * spl + c0 * sc;
    T* o = out + (long long)b * C * hw + c0 * oc + pofs * (nhwc ? C : 1);
    const A inv_kk = static_cast<A>(1) / static_cast<A>(KK);
    // optional fused mask blend (generator.py:130): out = prev * (1 - mask) + attention * mask
    const T* pv = prev ? prev + (long long)b * C * hw + c0 * oc + pofs * (nhwc ? C : 1) : nullptr;
    const A mk = prev ? static_cast<A>(ld(mask + (long long)b * hw + pofs)) : static_cast<A>(1);

    bool regular = false;
    if constexpr (K > 0) {
        AxisTap<A> tx[K], ty[K];
        regular = taps_regular<A, K>(flow_x, flow_y, x, y, Hs, Ws, tx, ty);
        if (regular) {
            constexpr int K1 = K + 1;
            // collapsed window: row r <-> unclamped source row Y0 + r, clamped on use
            A Wc[K1 * K1];
#pragma unroll
            for (int q = 0; q < K1 * K1; ++q) Wc[q] = static_cast<A>(0);
#pragma unroll
            for (int i = 0; i < K; ++i)
#pragma unroll
                for (int j = 0; j < K; ++j) {
                    const A pij = p[i * K + j];
                    Wc[i * K1 + j] += pij * (tx[j].wlo * ty[i].wlo);
                    Wc[i * K1 + j + 1] += pij * (tx[j].whi * ty[i].wlo);
                    Wc[(i + 1) * K1 + j] += pij * (tx[j].wlo * ty[i].whi);
                    Wc[(i + 1) * K1 + j + 1] += pij * (tx[j].whi * ty[i].whi);
                }
            int cx[K1], cy[K1];
#pragma unroll
            for (int r = 0; r < K1; ++r) {
                cx[r] = clampi(tx[0].fl + r, Ws - 1) * sp;
                cy[r] = clampi(ty[0].fl + r, Hs - 1) * Ws * sp;
            }
            for (int c = c0; c < c1; ++c, s += sc, o += oc) {
                A acc = static_cast<A>(0);
#pragma unroll
                for (int r = 0; r < K1; ++r)
#pragma unroll
                    for (int q = 0; q < K1; ++q) acc += Wc[r * K1 + q] * ld(s + cy[r] + cx[q]);
                acc *= inv_kk;
                if (pv) { acc = static_cast<A>(ld(pv)) * (static_cast<A>(1) - mk) + acc * mk; pv += oc; }
                st(o, acc);
            }
        }
    }
    if (!regular) {
        for (int c = c0; c < c1; ++c, s += sc, o += oc) {
            A acc = static_cast<A>(0);
            for (int i = 0; i < k; ++i) {
                const AxisTap<A> ty = axis_tap<A>(flow_y, i - k / 2, y, Hs);
                for (int j = 0; j < k; ++j) {
                    const AxisTap<A> tx = axis_tap<A>(flow_x, j - k / 2, x, Ws);
                    acc += p[i * k + j] * tap_value(s, tx, ty, Ws, sp);
                }
            }
            acc *= inv_kk;
            if (pv) { acc = static_cast<A>(ld(pv)) * (static_cast<A>(1) - mk) + acc * mk; pv += oc; }
            st(o, acc);
        }
    }
}

// ---------------------------------------------------------------------------
// backward.  Per pixel:
//   Q[r][s]   = sum_c g[c] * source[c, window(r,s)]          (k+1)^2 dot products
//   d p_ij    = 1/k^2 * bilinear_ij(Q)                        -> softmax backward
//   d flow    = 1/k^2 * sum_ij p_ij * d bilinear_ij(Q)/d(x,y) (block_extractor_kernel.cu:163-164)
//   d source += g[c] * Wc[r][s] / k^2                         scatter-add
// so each source value is read once per (pixel, channel) and the flow / logits
// gradients need no atomics at all.
// DET: grad_source goes into the fixed-point sums gsum (det_accum.cuh) with the image's exponent fx_exp[b] instead.
// ---------------------------------------------------------------------------
template <typename T, typename TF, int K, bool DET = false>
__global__ void __launch_bounds__(128)
k_local_attn_bwd(const T* __restrict__ src, const TF* __restrict__ flow, const T* __restrict__ logits,
                 const T* __restrict__ gout, T* __restrict__ gsrc, TF* __restrict__ gflow, T* __restrict__ glogits,
                 int B, int C, int Hs, int Ws, int H, int W, int k_rt, int accumulate, int nhwc, fx_t* __restrict__ gsum,
                 const int* __restrict__ fx_exp) {
    using A = typename Acc<T>::type;
    const int k = K ? K : k_rt, KK = k * k;
    const long long hw = (long long)H * W, total = (long long)B * hw;
    const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= total) return;
    const int x = (int)(pix % W), y = (int)((pix / W) % H), b = (int)(pix / hw);
    const long long pofs = (long long)y * W + x;

    A p[K ? K * K : kMaxK * kMaxK];
    pixel_softmax<T, A, K * K>(logits + (long long)b * KK * hw + pofs, hw, KK, p);
    const A flow_x = static_cast<A>(ld(flow + (long long)b * 2 * hw + pofs));
    const A flow_y = static_cast<A>(ld(flow + (long long)b * 2 * hw + hw + pofs));
    const long long spl = (long long)Hs * Ws;
    const long long sc = nhwc ? 1 : spl, oc = nhwc ? 1 : hw;   // element strides per channel
    const int sp = nhwc ? C : 1;                               // element stride per source position
    const T* s = src + (long long)b * C * spl;
    using GS = std::conditional_t<DET, fx_t, T>;
    GS* gs;
    double2 fsc = make_double2(0.0, 0.0);
    if constexpr (DET) {
        gs = gsum + (long long)b * C * spl;
        fsc = fx_scale(fx_exp[b]);
    } else {
        gs = gsrc + (long long)b * C * spl;
    }
    const T* go = gout + (long long)b * C * hw + pofs * (nhwc ? C : 1);
    const A inv_kk = static_cast<A>(1) / static_cast<A>(KK);

    A dp[K ? K * K : kMaxK * kMaxK];  // d loss / d p_t
    A gfx = static_cast<A>(0), gfy = static_cast<A>(0);

    bool regular = false;
    if constexpr (K > 0) {
        AxisTap<A> tx[K], ty[K];
        regular = taps_regular<A, K>(flow_x, flow_y, x, y, Hs, Ws, tx, ty);
        if (regular) {
            constexpr int K1 = K + 1;
            A Wc[K1 * K1], Q[K1 * K1];
#pragma unroll
            for (int q = 0; q < K1 * K1; ++q) { Wc[q] = static_cast<A>(0); Q[q] = static_cast<A>(0); }
#pragma unroll
            for (int i = 0; i < K; ++i)
#pragma unroll
                for (int j = 0; j < K; ++j) {
                    const A pij = p[i * K + j] * inv_kk;
                    Wc[i * K1 + j] += pij * (tx[j].wlo * ty[i].wlo);
                    Wc[i * K1 + j + 1] += pij * (tx[j].whi * ty[i].wlo);
                    Wc[(i + 1) * K1 + j] += pij * (tx[j].wlo * ty[i].whi);
                    Wc[(i + 1) * K1 + j + 1] += pij * (tx[j].whi * ty[i].whi);
                }
            int cx[K1], cy[K1];
#pragma unroll
            for (int r = 0; r < K1; ++r) {
                cx[r] = clampi(tx[0].fl + r, Ws - 1) * sp;
                cy[r] = clampi(ty[0].fl + r, Hs - 1) * Ws * sp;
            }
            for (int c = 0; c < C; ++c, s += sc, gs += sc, go += oc) {
                const A g = ld(go);
#pragma unroll
                for (int r = 0; r < K1; ++r)
#pragma unroll
                    for (int q = 0; q < K1; ++q) {
                        const int o = cy[r] + cx[q];
                        Q[r * K1 + q] += g * ld(s + o);
                        scatter_add<DET>(gs + o, g * Wc[r * K1 + q], fsc);
                    }
            }
#pragma unroll
            for (int i = 0; i < K; ++i)
#pragma unroll
                for (int j = 0; j < K; ++j)
                    dp[i * K + j] = tap_backward<A>(tx[j], ty[i], p[i * K + j] * inv_kk, inv_kk, Q[i * K1 + j], Q[i * K1 + j + 1],
                                                    Q[(i + 1) * K1 + j], Q[(i + 1) * K1 + j + 1], gfx, gfy);
        }
    }
    if (!regular) {
        for (int i = 0; i < k; ++i) {
            const AxisTap<A> ty = axis_tap<A>(flow_y, i - k / 2, y, Hs);
            for (int j = 0; j < k; ++j) {
                const AxisTap<A> tx = axis_tap<A>(flow_x, j - k / 2, x, Ws);
                const int oLT = (ty.lo * Ws + tx.lo) * sp, oRT = (ty.lo * Ws + tx.hi) * sp, oLB = (ty.hi * Ws + tx.lo) * sp,
                          oRB = (ty.hi * Ws + tx.hi) * sp;
                const A pij = p[i * k + j] * inv_kk;
                A qLT = 0, qRT = 0, qLB = 0, qRB = 0;
                const T* sq = s;
                GS* gc = gs;
                const T* goc = go;
#pragma unroll 1   // rare path, k*k copies of this loop: unrolled, it would raise the register pressure of the whole kernel
                for (int c = 0; c < C; ++c, sq += sc, gc += sc, goc += oc) {
                    const A g = ld(goc);
                    qLT += g * ld(sq + oLT); qRT += g * ld(sq + oRT); qLB += g * ld(sq + oLB); qRB += g * ld(sq + oRB);
                    const A gp = g * pij;
                    scatter_add<DET>(gc + oLT, gp * (tx.wlo * ty.wlo), fsc);
                    scatter_add<DET>(gc + oRT, gp * (tx.whi * ty.wlo), fsc);
                    scatter_add<DET>(gc + oLB, gp * (tx.wlo * ty.whi), fsc);
                    scatter_add<DET>(gc + oRB, gp * (tx.whi * ty.whi), fsc);
                }
                dp[i * k + j] = tap_backward<A>(tx, ty, pij, inv_kk, qLT, qRT, qLB, qRB, gfx, gfy);
            }
        }
    }
    store_pixel_grads<T, TF, A, K * K>(p, dp, KK, gfx, gfy, glogits + (long long)b * KK * hw + pofs,
                                       gflow + (long long)b * 2 * hw + pofs, hw, accumulate);
}

template <typename T, typename TF, int K>
static int la_launch_fwd(const void* src, const void* flow, const void* logits, void* out, void* probs, const void* prev,
                         const void* mask, int B, int C, int Hs, int Ws, int H, int W, int k, int nhwc, cudaStream_t st_) {
    const long long total = (long long)B * H * W;
    const int threads = 128, slices0 = channel_splits(total, C, threads), cps = (C + slices0 - 1) / slices0;
    dim3 grid((unsigned)((total + threads - 1) / threads), (unsigned)((C + cps - 1) / cps));
    k_local_attn_fwd<T, TF, K><<<grid, threads, 0, st_>>>((const T*)src, (const TF*)flow, (const T*)logits, (T*)out,
                                                         (T*)probs, (const T*)prev, (const T*)mask, B, C, Hs, Ws, H, W, k, cps, nhwc);
    return launch_status();
}

template <typename T, typename TF, int K, bool DET = false>
static int la_launch_bwd(const void* src, const void* flow, const void* logits, const void* gout, void* gsrc,
                         void* gflow, void* glogits, int B, int C, int Hs, int Ws, int H, int W, int k, int accumulate,
                         int nhwc, cudaStream_t st_, fx_t* gsum = nullptr, const int* fx_exp = nullptr) {
    const long long total = (long long)B * H * W;
    const int threads = 128;
    k_local_attn_bwd<T, TF, K, DET><<<(unsigned)((total + threads - 1) / threads), threads, 0, st_>>>(
        (const T*)src, (const TF*)flow, (const T*)logits, (const T*)gout, (T*)gsrc, (TF*)gflow, (T*)glogits, B, C, Hs,
        Ws, H, W, k, accumulate, nhwc, gsum, fx_exp);
    return launch_status();
}

template <typename T, typename TF, int K>
static int la_launch_bwd_det(const void* src, const void* flow, const void* logits, const void* gout, void* gflow, void* glogits,
                             int B, int C, int Hs, int Ws, int H, int W, int k, int accumulate, int nhwc, fx_t* gsum,
                             const int* fx_exp, cudaStream_t st_) {
    return la_launch_bwd<T, TF, K, true>(src, flow, logits, gout, nullptr, gflow, glogits, B, C, Hs, Ws, H, W, k, accumulate, nhwc,
                                         st_, gsum, fx_exp);
}

#define GFLA_K_DISPATCH(fn, ...)                       \
    switch (k) {                                       \
        case 2: return fn<T, TF, 2>(__VA_ARGS__);      \
        case 3: return fn<T, TF, 3>(__VA_ARGS__);      \
        case 4: return fn<T, TF, 4>(__VA_ARGS__);      \
        case 5: return fn<T, TF, 5>(__VA_ARGS__);      \
        default: return fn<T, TF, 0>(__VA_ARGS__);     \
    }

int local_attn_fwd_gather(const void* src, const void* flow, const void* logits, void* out, void* probs, const void* prev,
                          const void* mask, int B, int C, int Hs, int Ws, int H, int W, int k, int dtype, int flow_dtype,
                          int layout, cudaStream_t st_) {
    const int nhwc = layout == GFLA_NHWC;
    return dispatch_dtypes(dtype, flow_dtype, dtype, [&](auto t, auto tf, auto) -> int {
        using T = typename decltype(t)::type;
        using TF = typename decltype(tf)::type;
        GFLA_K_DISPATCH(la_launch_fwd, src, flow, logits, out, probs, prev, mask, B, C, Hs, Ws, H, W, k, nhwc, st_)
    });
}

int local_attn_bwd_gather(const void* src, const void* flow, const void* logits, const void* gout, void* gsrc,
                          void* gflow, void* glogits, int B, int C, int Hs, int Ws, int H, int W, int k, int dtype,
                          int flow_dtype, int accumulate, int layout, cudaStream_t st_) {
    const int nhwc = layout == GFLA_NHWC;
    if (!accumulate) {
        const int e = zero_async(gsrc, (size_t)B * C * Hs * Ws * elem_size(dtype), st_);
        if (e != GFLA_OK) return e;
    }
    return dispatch_dtypes(dtype, flow_dtype, dtype, [&](auto t, auto tf, auto) -> int {
        using T = typename decltype(t)::type;
        using TF = typename decltype(tf)::type;
        GFLA_K_DISPATCH(la_launch_bwd, src, flow, logits, gout, gsrc, gflow, glogits, B, C, Hs, Ws, H, W, k, accumulate, nhwc, st_)
    });
}

// grad_source into the fixed-point sums gsum (zeroed, exponents in fx_exp: det_accum.cuh); grad_flow / grad_logits as above
int local_attn_bwd_gather_det(const void* src, const void* flow, const void* logits, const void* gout, void* gflow, void* glogits,
                              int B, int C, int Hs, int Ws, int H, int W, int k, int dtype, int flow_dtype, int accumulate,
                              int layout, fx_t* gsum, const int* fx_exp, cudaStream_t st_) {
    const int nhwc = layout == GFLA_NHWC;
    return dispatch_dtypes(dtype, flow_dtype, dtype, [&](auto t, auto tf, auto) -> int {
        using T = typename decltype(t)::type;
        using TF = typename decltype(tf)::type;
        GFLA_K_DISPATCH(la_launch_bwd_det, src, flow, logits, gout, gflow, glogits, B, C, Hs, Ws, H, W, k, accumulate, nhwc, gsum,
                        fx_exp, st_)
    });
}

}  // namespace gfla
