// Shared device/host helpers for the GFLA warping library (sm_90a).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/gfla_warp.h"

namespace gfla {

// ---------------------------------------------------------------------------
// storage type -> arithmetic type.  The reference instantiates float and double
// (AT_DISPATCH_FLOATING_TYPES); 16-bit storage computes in fp32.
// ---------------------------------------------------------------------------
template <typename T> struct Acc { using type = float; };
template <> struct Acc<double> { using type = double; };

template <typename T> __device__ __forceinline__ typename Acc<T>::type ld(const T* p) { return static_cast<typename Acc<T>::type>(*p); }
template <> __device__ __forceinline__ float ld<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat162float(*p); }
template <> __device__ __forceinline__ float ld<__half>(const __half* p) { return __half2float(*p); }

template <typename T, typename A> __device__ __forceinline__ void st(T* p, A v) { *p = static_cast<T>(v); }
template <> __device__ __forceinline__ void st<__nv_bfloat16, float>(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ void st<__half, float>(__half* p, float v) { *p = __float2half_rn(v); }

// scatter-add of one element (grad_source / grad_in1).
template <typename T, typename A> __device__ __forceinline__ void red_add(T* p, A v) { atomicAdd(p, static_cast<T>(v)); }
template <> __device__ __forceinline__ void red_add<__nv_bfloat16, float>(__nv_bfloat16* p, float v) { atomicAdd(p, __float2bfloat16_rn(v)); }
template <> __device__ __forceinline__ void red_add<__half, float>(__half* p, float v) { atomicAdd(p, __float2half_rn(v)); }

__device__ __forceinline__ float flr(float v) { return floorf(v); }
__device__ __forceinline__ double flr(double v) { return floor(v); }

__device__ __forceinline__ int clampi(int v, int hi) { return max(min(v, hi), 0); }

// ---------------------------------------------------------------------------
// One block_extractor tap along one axis, evaluated exactly like the reference
// (block_extractor_kernel.cu:62-76):  d = (flow + offset) + coord in the
// arithmetic type, floor, int conversion, THEN clamp; weights from the
// unclamped fraction.
// ---------------------------------------------------------------------------
template <typename A>
struct AxisTap {
    int lo, hi;  // clamped indices (xL/xR or yT/yB)
    A wlo, whi;  // 1 - frac, frac
    int fl;      // unclamped floor (used by the tile kernels)
};

template <typename A>
__device__ __forceinline__ AxisTap<A> axis_tap(A flow, int offset, int coord, int dim) {
    AxisTap<A> t;
    A f = flow + static_cast<A>(offset);
    A d = f + static_cast<A>(coord);
    A fd = flr(d);
    t.fl = static_cast<int>(fd);
    t.lo = clampi(static_cast<int>(fd), dim - 1);
    t.hi = clampi(static_cast<int>(fd + static_cast<A>(1)), dim - 1);
    t.wlo = static_cast<A>(1) - (d - fd);
    t.whi = d - fd;
    return t;
}

// ---------------------------------------------------------------------------
// host-side helpers
// ---------------------------------------------------------------------------
inline int elem_size(int dtype) {
    switch (dtype) {
        case GFLA_F32: return 4;
        case GFLA_F64: return 8;
        case GFLA_BF16: case GFLA_F16: return 2;
        default: return 0;
    }
}
inline bool aligned(const void* p, int bytes) { return (reinterpret_cast<uintptr_t>(p) % bytes) == 0; }

inline int sm_count() {
    static int n = 0;  // immutable after first query; benign if raced
    if (n == 0) {
        int dev = 0, v = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
        n = v > 0 ? v : 148;
    }
    return n;
}

// How many channel slices (grid.y) to use so that `items` threads per slice
// still fill the machine with >= ~4 waves of 256-thread CTAs.
inline int channel_splits(long long items, int C, int threads) {
    long long ctas = (items + threads - 1) / threads;
    long long want = 4LL * sm_count() * (2048 / threads);
    int s = 1;
    while (ctas * s < want && s * 2 <= C && s < 64) s *= 2;
    return s;
}

// Process-wide count of kernels this library has launched (statistics only: bench.py reports it as
// `gpu_launches`; relaxed atomic, never read by the library itself).  Defined in api.cu.
void count_launch();

inline int launch_status() {
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) count_launch();
    return e == cudaSuccess ? GFLA_OK : static_cast<int>(e);
}

// zero-fill on the caller's stream; the status is the caller's to propagate (nothing may be launched after a failure)
inline int zero_async(void* p, size_t bytes, cudaStream_t st_) {
    cudaError_t e = cudaMemsetAsync(p, 0, bytes, st_);
    return e == cudaSuccess ? GFLA_OK : static_cast<int>(e);
}

#define GFLA_DISPATCH_T(dtype, ...)                                            \
    [&]() -> int {                                                             \
        switch (dtype) {                                                       \
            case GFLA_F32: { using T = float; return __VA_ARGS__(); }          \
            case GFLA_F64: { using T = double; return __VA_ARGS__(); }         \
            case GFLA_BF16: { using T = __nv_bfloat16; return __VA_ARGS__(); } \
            case GFLA_F16: { using T = __half; return __VA_ARGS__(); }         \
            default: return GFLA_E_DTYPE;                                      \
        }                                                                      \
    }()

template <typename T> struct Type { using type = T; };

// The (data, flow, grad_source) dtype combinations the library serves, listed nowhere else.  fp32 and fp64 data take
// flow and grad_source of their own type; 16-bit data may widen either to fp32.  Only the block_extractor backward
// offers an fp32 grad_source: every other op passes the data dtype as gs_dtype.  Calls f(Type<T>{}, Type<TF>{},
// Type<TG>{}) for a listed combination and returns GFLA_E_DTYPE for anything else.
template <typename F>
inline int dispatch_dtypes(int dtype, int flow_dtype, int gs_dtype, F&& f) {
#define GFLA_DTYPES(D, T, FD, TF, GD, TG) \
    if (dtype == D && flow_dtype == FD && gs_dtype == GD) return f(Type<T>{}, Type<TF>{}, Type<TG>{});
    GFLA_DTYPES(GFLA_F32, float, GFLA_F32, float, GFLA_F32, float)
    GFLA_DTYPES(GFLA_F64, double, GFLA_F64, double, GFLA_F64, double)
    GFLA_DTYPES(GFLA_BF16, __nv_bfloat16, GFLA_BF16, __nv_bfloat16, GFLA_BF16, __nv_bfloat16)
    GFLA_DTYPES(GFLA_BF16, __nv_bfloat16, GFLA_F32, float, GFLA_BF16, __nv_bfloat16)
    GFLA_DTYPES(GFLA_BF16, __nv_bfloat16, GFLA_BF16, __nv_bfloat16, GFLA_F32, float)
    GFLA_DTYPES(GFLA_BF16, __nv_bfloat16, GFLA_F32, float, GFLA_F32, float)
    GFLA_DTYPES(GFLA_F16, __half, GFLA_F16, __half, GFLA_F16, __half)
    GFLA_DTYPES(GFLA_F16, __half, GFLA_F32, float, GFLA_F16, __half)
    GFLA_DTYPES(GFLA_F16, __half, GFLA_F16, __half, GFLA_F32, float)
    GFLA_DTYPES(GFLA_F16, __half, GFLA_F32, float, GFLA_F32, float)
#undef GFLA_DTYPES
    return GFLA_E_DTYPE;
}

inline bool dtypes_ok(int dtype, int flow_dtype, int gs_dtype) {
    return dispatch_dtypes(dtype, flow_dtype, gs_dtype, [](auto, auto, auto) { return GFLA_OK; }) == GFLA_OK;
}

}  // namespace gfla
