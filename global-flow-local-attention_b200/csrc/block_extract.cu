// block_extractor and local_attn_reshape for sm_90a (CUDA-core kernels).
//
// What they compute is fixed by the reference
// (block_extractor/block_extractor_kernel.cu:20-170,
//  local_attn_reshape/local_attn_reshape_kernel.cu:20-108); how they are laid
// out on the machine is not:
//   * forward: one thread per OUTPUT POSITION (b, yo, xo) -- the flow read, the
//     floor/clamp/weight arithmetic are done once and reused for every channel
//     of the slice (the reference redoes them per element); consecutive lanes
//     write consecutive xo (coalesced stores), channel slices in grid.y.
//   * backward: one thread per FLOW PIXEL (b, yf, xf); the k*k*C contributions
//     to grad_flow are summed in registers, so the reference's C*k*k-way
//     atomic collision per flow element (kernel.cu:167-168) disappears;
//     grad_source keeps a scatter-add (red.global) because the flow is arbitrary.
//   * 64-bit indexing throughout (the reference's `int n` overflows at cfg2).
// This translation unit is compiled with -fmad=false so that the fp32/fp64
// forward is bit-identical to the (uncontracted) CPU oracle.
#include "det_accum.cuh"

namespace gfla {

template <typename T, typename TF>
__global__ void __launch_bounds__(256)
k_block_extract_fwd(const T* __restrict__ src, const TF* __restrict__ flow, T* __restrict__ out,
                    int B, int C, int Hs, int Ws, int Hf, int Wf, int k, int c_per_slice) {
    using A = typename Acc<T>::type;
    const int Ho = k * Hf, Wo = k * Wf;
    const long long total = (long long)B * Ho * Wo;
    const long long pos = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (pos >= total) return;
    const int xo = (int)(pos % Wo);
    const int yo = (int)((pos / Wo) % Ho);
    const int b = (int)(pos / ((long long)Wo * Ho));
    const int yf = yo / k, xf = xo / k;
    const long long fpl = (long long)Hf * Wf;
    const TF* fp = flow + (long long)b * 2 * fpl + (long long)yf * Wf + xf;
    const A flow_x = static_cast<A>(ld(fp)), flow_y = static_cast<A>(ld(fp + fpl));
    const AxisTap<A> ty = axis_tap<A>(flow_y, yo % k - k / 2, yf, Hs);
    const AxisTap<A> tx = axis_tap<A>(flow_x, xo % k - k / 2, xf, Ws);
    const A wLT = tx.wlo * ty.wlo, wRT = tx.whi * ty.wlo, wLB = tx.wlo * ty.whi, wRB = tx.whi * ty.whi;
    const int oLT = ty.lo * Ws + tx.lo, oRT = ty.lo * Ws + tx.hi, oLB = ty.hi * Ws + tx.lo, oRB = ty.hi * Ws + tx.hi;
    const long long spl = (long long)Hs * Ws, opl = (long long)Ho * Wo;
    const int c0 = blockIdx.y * c_per_slice, c1 = min(C, c0 + c_per_slice);
    const T* s = src + ((long long)b * C + c0) * spl;
    T* o = out + ((long long)b * C + c0) * opl + (long long)yo * Wo + xo;
#pragma unroll 4
    for (int c = c0; c < c1; ++c, s += spl, o += opl) {
        A v = static_cast<A>(0);
        v += wLT * ld(s + oLT);
        v += wRT * ld(s + oRT);
        v += wLB * ld(s + oLB);
        v += wRB * ld(s + oRB);
        st(o, v);
    }
}

// TG = storage type of grad_source: T, or float for 16-bit T (native fp32 red.global instead of the
// compare-and-swap loop a 16-bit scalar atomicAdd turns into; the caller narrows the buffer afterwards).
// DET: grad_source goes into the fixed-point sums gsum with the image's exponent fx_exp[b] (det_accum.cuh).
template <typename T, typename TF, typename TG, bool DET = false>
__global__ void __launch_bounds__(128)
k_block_extract_bwd(const T* __restrict__ src, const TF* __restrict__ flow, const T* __restrict__ gout,
                    TG* __restrict__ gsrc, TF* __restrict__ gflow,
                    int B, int C, int Hs, int Ws, int Hf, int Wf, int k, int c_per_slice, int slices, fx_t* __restrict__ gsum,
                    const int* __restrict__ fx_exp) {
    using A = typename Acc<T>::type;
    const long long total = (long long)B * Hf * Wf;
    const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= total) return;
    const int xf = (int)(pix % Wf);
    const int yf = (int)((pix / Wf) % Hf);
    const int b = (int)(pix / ((long long)Wf * Hf));
    const int Ho = k * Hf, Wo = k * Wf;
    const long long fpl = (long long)Hf * Wf, spl = (long long)Hs * Ws, opl = (long long)Ho * Wo;
    const long long foff = (long long)b * 2 * fpl + (long long)yf * Wf + xf;
    const A flow_x = static_cast<A>(ld(flow + foff)), flow_y = static_cast<A>(ld(flow + foff + fpl));
    const int c0 = blockIdx.y * c_per_slice, c1 = min(C, c0 + c_per_slice);
    A gy = static_cast<A>(0), gx = static_cast<A>(0);
    using GS = std::conditional_t<DET, fx_t, TG>;
    GS* gs_img;
    double2 fsc = make_double2(0.0, 0.0);
    if constexpr (DET) {
        gs_img = gsum;
        fsc = fx_scale(fx_exp[b]);
    } else {
        gs_img = gsrc;
    }
    for (int i = 0; i < k; ++i) {
        const AxisTap<A> ty = axis_tap<A>(flow_y, i - k / 2, yf, Hs);
        for (int j = 0; j < k; ++j) {
            const AxisTap<A> tx = axis_tap<A>(flow_x, j - k / 2, xf, Ws);
            const int oLT = ty.lo * Ws + tx.lo, oRT = ty.lo * Ws + tx.hi, oLB = ty.hi * Ws + tx.lo, oRB = ty.hi * Ws + tx.hi;
            const T* s = src + ((long long)b * C + c0) * spl;
            GS* gs = gs_img + ((long long)b * C + c0) * spl;
            const T* go = gout + ((long long)b * C + c0) * opl + (long long)(yf * k + i) * Wo + (xf * k + j);
            for (int c = c0; c < c1; ++c, s += spl, gs += spl, go += opl) {
                const A g = ld(go);
                const A vLT = ld(s + oLT), vRT = ld(s + oRT), vLB = ld(s + oLB), vRB = ld(s + oRB);
                scatter_add<DET>(gs + oLT, g * tx.wlo * ty.wlo, fsc);
                scatter_add<DET>(gs + oRT, g * tx.whi * ty.wlo, fsc);
                scatter_add<DET>(gs + oLB, g * tx.wlo * ty.whi, fsc);
                scatter_add<DET>(gs + oRB, g * tx.whi * ty.whi, fsc);
                gy += g * (-tx.wlo * vLT - tx.whi * vRT + tx.wlo * vLB + tx.whi * vRB);
                gx += g * (-ty.wlo * vLT - ty.whi * vLB + ty.wlo * vRT + ty.whi * vRB);
            }
        }
    }
    if (slices == 1) {  // this thread owns the flow element: plain read-modify-write, deterministic
        st(gflow + foff, static_cast<A>(ld(gflow + foff)) + gx);
        st(gflow + foff + fpl, static_cast<A>(ld(gflow + foff + fpl)) + gy);
    } else {
        red_add(gflow + foff, gx);
        red_add(gflow + foff + fpl, gy);
    }
}

// depth-to-space: out[b,0,y,x] = in[b,(y%k)*k + x%k, y/k, x/k]
template <typename T>
__global__ void __launch_bounds__(256)
k_attn_reshape_fwd(const T* __restrict__ in, T* __restrict__ out, int B, int H, int W, int k) {
    const int Ho = k * H, Wo = k * W;
    const long long total = (long long)B * Ho * Wo;
    const long long pos = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (pos >= total) return;
    const int x = (int)(pos % Wo), y = (int)((pos / Wo) % Ho), b = (int)(pos / ((long long)Wo * Ho));
    const int cs = (y % k) * k + (x % k);
    out[pos] = in[(((long long)b * k * k + cs) * H + y / k) * W + x / k];
}

// the mapping is a bijection, so the reference's atomicAdd (kernel.cu:106) is a
// plain read-modify-write here; one thread per grad_in element -> coalesced stores.
template <typename T>
__global__ void __launch_bounds__(256)
k_attn_reshape_bwd(const T* __restrict__ gout, T* __restrict__ gin, int B, int H, int W, int k, int accumulate) {
    using A = typename Acc<T>::type;
    const long long total = (long long)B * k * k * H * W;
    const long long pos = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (pos >= total) return;
    const int x = (int)(pos % W), y = (int)((pos / W) % H);
    const int cs = (int)((pos / ((long long)W * H)) % (k * k)), b = (int)(pos / ((long long)W * H * k * k));
    const int Ho = k * H, Wo = k * W;
    const A g = ld(gout + ((long long)b * Ho + (y * k + cs / k)) * Wo + (x * k + cs % k));
    st(gin + pos, accumulate ? static_cast<A>(ld(gin + pos)) + g : g);
}

// element-wise dtype conversion (narrowing an fp32 gradient accumulator to 16-bit storage, etc.)
template <typename TS, typename TD>
__global__ void __launch_bounds__(256)
k_convert(const TS* __restrict__ src, TD* __restrict__ dst, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) st(dst + i, ld(src + i));
}

// ---------------------------------------------------------------------------
// host launchers (called from api.cu)
// ---------------------------------------------------------------------------
template <typename T, typename TF>
static int launch_be_fwd(const void* src, const void* flow, void* out, int B, int C, int Hs, int Ws, int Hf, int Wf,
                         int k, cudaStream_t st_) {
    const long long total = (long long)B * k * Hf * k * Wf;
    const int threads = 256;
    const int slices = channel_splits(total, C, threads);
    const int cps = (C + slices - 1) / slices;
    dim3 grid((unsigned)((total + threads - 1) / threads), (unsigned)((C + cps - 1) / cps));
    k_block_extract_fwd<T, TF><<<grid, threads, 0, st_>>>((const T*)src, (const TF*)flow, (T*)out, B, C, Hs, Ws, Hf, Wf, k, cps);
    return launch_status();
}

template <typename T, typename TF, typename TG, bool DET = false>
static int launch_be_bwd(const void* src, const void* flow, const void* gout, void* gsrc, void* gflow, int B, int C,
                         int Hs, int Ws, int Hf, int Wf, int k, cudaStream_t st_, fx_t* gsum = nullptr, const int* fx_exp = nullptr) {
    const long long total = (long long)B * Hf * Wf;
    const int threads = 128;
    // DET: one channel slice, so that every thread owns its grad_flow element whatever the SM count
    const int slices0 = DET ? 1 : channel_splits(total, C, threads);
    const int cps = (C + slices0 - 1) / slices0;
    const int slices = (C + cps - 1) / cps;
    dim3 grid((unsigned)((total + threads - 1) / threads), (unsigned)slices);
    k_block_extract_bwd<T, TF, TG, DET><<<grid, threads, 0, st_>>>((const T*)src, (const TF*)flow, (const T*)gout, (TG*)gsrc,
                                                              (TF*)gflow, B, C, Hs, Ws, Hf, Wf, k, cps, slices, gsum, fx_exp);
    return launch_status();
}

int block_extract_fwd(const void* src, const void* flow, void* out, int B, int C, int Hs, int Ws, int Hf, int Wf,
                      int k, int dtype, int flow_dtype, cudaStream_t st_) {
    return dispatch_dtypes(dtype, flow_dtype, dtype, [&](auto t, auto tf, auto) -> int {
        return launch_be_fwd<typename decltype(t)::type, typename decltype(tf)::type>(src, flow, out, B, C, Hs, Ws, Hf, Wf, k, st_);
    });
}

int block_extract_bwd(const void* src, const void* flow, const void* gout, void* gsrc, void* gflow, int B, int C,
                      int Hs, int Ws, int Hf, int Wf, int k, int dtype, int flow_dtype, int gs_dtype, int accumulate,
                      cudaStream_t st_) {
    if (!accumulate) {
        int e = zero_async(gsrc, (size_t)B * C * Hs * Ws * elem_size(gs_dtype), st_);
        if (e == GFLA_OK) e = zero_async(gflow, (size_t)B * 2 * Hf * Wf * elem_size(flow_dtype), st_);
        if (e != GFLA_OK) return e;
    }
    return dispatch_dtypes(dtype, flow_dtype, gs_dtype, [&](auto t, auto tf, auto tg) -> int {
        return launch_be_bwd<typename decltype(t)::type, typename decltype(tf)::type, typename decltype(tg)::type>(
            src, flow, gout, gsrc, gflow, B, C, Hs, Ws, Hf, Wf, k, st_);
    });
}

// grad_source into the fixed-point sums gsum (zeroed, exponents in fx_exp: det_accum.cuh); grad_flow follows `accumulate`
int block_extract_bwd_det(const void* src, const void* flow, const void* gout, void* gflow, int B, int C, int Hs, int Ws, int Hf,
                          int Wf, int k, int dtype, int flow_dtype, int accumulate, fx_t* gsum, const int* fx_exp, cudaStream_t st_) {
    if (!accumulate) {
        const int e = zero_async(gflow, (size_t)B * 2 * Hf * Wf * elem_size(flow_dtype), st_);
        if (e != GFLA_OK) return e;
    }
    return dispatch_dtypes(dtype, flow_dtype, dtype, [&](auto t, auto tf, auto) -> int {
        using T = typename decltype(t)::type;
        return launch_be_bwd<T, typename decltype(tf)::type, T, true>(src, flow, gout, nullptr, gflow, B, C, Hs, Ws, Hf, Wf, k, st_,
                                                                      gsum, fx_exp);
    });
}

int convert(const void* src, int src_dtype, void* dst, int dst_dtype, long long n, cudaStream_t st_) {
    const unsigned blocks = (unsigned)((n + 255) / 256);
#define GFLA_CVT(SD, ST, DD, DT) \
    if (src_dtype == SD && dst_dtype == DD) { k_convert<ST, DT><<<blocks, 256, 0, st_>>>((const ST*)src, (DT*)dst, n); return launch_status(); }
    GFLA_CVT(GFLA_F32, float, GFLA_BF16, __nv_bfloat16) GFLA_CVT(GFLA_F32, float, GFLA_F16, __half)
    GFLA_CVT(GFLA_BF16, __nv_bfloat16, GFLA_F32, float) GFLA_CVT(GFLA_F16, __half, GFLA_F32, float)
#undef GFLA_CVT
    return GFLA_E_DTYPE;
}

int attn_reshape_fwd(const void* in, void* out, int B, int H, int W, int k, int dtype, cudaStream_t st_) {
    const long long total = (long long)B * k * H * k * W;
    return GFLA_DISPATCH_T(dtype, [&]() -> int {
        k_attn_reshape_fwd<T><<<(unsigned)((total + 255) / 256), 256, 0, st_>>>((const T*)in, (T*)out, B, H, W, k);
        return launch_status();
    });
}

int attn_reshape_bwd(const void* gout, void* gin, int B, int H, int W, int k, int dtype, int accumulate,
                     cudaStream_t st_) {
    const long long total = (long long)B * k * H * k * W;
    return GFLA_DISPATCH_T(dtype, [&]() -> int {
        k_attn_reshape_bwd<T><<<(unsigned)((total + 255) / 256), 256, 0, st_>>>((const T*)gout, (T*)gin, B, H, W, k, accumulate);
        return launch_status();
    });
}

}  // namespace gfla
