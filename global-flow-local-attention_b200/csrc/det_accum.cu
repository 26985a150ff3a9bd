// Pre-pass (maxima, exponents) and narrowing of the deterministic fixed-point scatter (det_accum.cuh).
#include "det_accum.cuh"

namespace gfla {

__device__ __forceinline__ double ld_d(const float* p) { return static_cast<double>(*p); }
__device__ __forceinline__ double ld_d(const double* p) { return *p; }
__device__ __forceinline__ double ld_d(const __nv_bfloat16* p) { return static_cast<double>(__bfloat162float(*p)); }
__device__ __forceinline__ double ld_d(const __half* p) { return static_cast<double>(__half2float(*p)); }

__device__ __forceinline__ void st_d(float* p, double v) { *p = static_cast<float>(v); }
__device__ __forceinline__ void st_d(double* p, double v) { *p = v; }
__device__ __forceinline__ void st_d(__nv_bfloat16* p, double v) { *p = __double2bfloat16(v); }   // one rounding
__device__ __forceinline__ void st_d(__half* p, double v) { *p = __double2half(v); }

// grid (x: slices of one image, y: image).  The maximum of |x| as fp64 bits: for non-negative doubles the bit patterns
// order like the values, and NaN (0x7ff8...) > Inf (0x7ff0...) > every finite value, so one unsigned max also flags
// non-finite input.  A max does not depend on order.
template <typename T>
__global__ void __launch_bounds__(256) k_fx_amax(const T* __restrict__ x, long long per_img, fx_t* __restrict__ amax) {
    const T* xi = x + (long long)blockIdx.y * per_img;
    fx_t m = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < per_img; i += (long long)gridDim.x * blockDim.x)
        m = max(m, (fx_t)__double_as_longlong(fabs(ld_d(xi + i))));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = max(m, (fx_t)__shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0 && m != 0) atomicMax(amax + blockIdx.y, m);
}

// exponent of M = factor * a * b (each finite and >= 0): 61 - e with M < 2^e, clamped to [-FX_EMAX, FX_EMAX]
__device__ int fx_exponent(double a, double b, double factor) {
    if (!(a <= DBL_MAX) || !(b <= DBL_MAX)) return FX_NONFINITE;      // Inf or NaN
    if (a == 0.0 || b == 0.0 || factor == 0.0) return 0;              // every partial is zero
    int ea, eb, ef, em;
    const double ma = frexp(a, &ea), mb = frexp(b, &eb), mf = frexp(factor, &ef);
    frexp(ma * mb * mf, &em);          // product of three mantissas in [1/8, 1): rounding can only raise em (safe)
    const int e = 61 - (ea + eb + ef + em);
    return max(-FX_EMAX, min(FX_EMAX, e));
}

__global__ void k_fx_exponents(const fx_t* __restrict__ a, int n_a, const fx_t* __restrict__ b, double factor, int over_all,
                               int* __restrict__ exps) {
    const double vb = b ? __longlong_as_double((long long)b[0]) : 1.0;
    if (over_all) {
        if (threadIdx.x != 0 || blockIdx.x != 0) return;
        fx_t m = 0;
        for (int i = 0; i < n_a; ++i) m = max(m, a[i]);
        exps[0] = fx_exponent(__longlong_as_double((long long)m), vb, factor);
        return;
    }
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_a) exps[i] = fx_exponent(__longlong_as_double((long long)a[i]), vb, factor);
}

template <typename T>
__global__ void __launch_bounds__(256) k_fx_narrow(const fx_t* __restrict__ sums, const int* __restrict__ exps, long long per_img,
                                                   long long n, T* __restrict__ out, int accumulate) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int e = exps[i / per_img];
    double v;
    if (e == FX_NONFINITE) {
        v = __longlong_as_double(0x7ff8000000000000LL);
    } else {
        const int h = e / 2;        // 2^-E as two factors, like fx_scale
        v = static_cast<double>(static_cast<long long>(sums[i])) * ldexp(1.0, -h) * ldexp(1.0, h - e);
        if (accumulate) v += ld_d(out + i);
    }
    st_d(out + i, v);
}

int fx_amax(const void* x, int dtype, long long per_img, int n_img, fx_t* amax, cudaStream_t st_) {
    const long long want = (per_img + 255) / 256;
    const unsigned gx = (unsigned)max(1LL, min(want, (4LL * sm_count() + n_img - 1) / n_img * 4));
    return GFLA_DISPATCH_T(dtype, [&]() -> int {
        k_fx_amax<T><<<dim3(gx, (unsigned)n_img), 256, 0, st_>>>((const T*)x, per_img, amax);
        return launch_status();
    });
}

int fx_exponents(const fx_t* a, int n_a, const fx_t* b, double factor, bool over_all, int* exps, cudaStream_t st_) {
    const int n = over_all ? 1 : n_a;
    k_fx_exponents<<<(unsigned)((n + 127) / 128), 128, 0, st_>>>(a, n_a, b, factor, over_all ? 1 : 0, exps);
    return launch_status();
}

int fx_narrow(const fx_t* sums, const int* exps, long long per_img, long long n, void* out, int dtype, int accumulate,
              cudaStream_t st_) {
    return GFLA_DISPATCH_T(dtype, [&]() -> int {
        k_fx_narrow<T><<<(unsigned)((n + 255) / 256), 256, 0, st_>>>(sums, exps, per_img, n, (T*)out, accumulate);
        return launch_status();
    });
}

}  // namespace gfla
