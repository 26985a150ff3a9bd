// Deterministic scatter-add: per-image 64-bit fixed point (the backward passes under
// torch.use_deterministic_algorithms(True), the *_det entry points of the C ABI).
//
// Every scatter site converts its partial v to q = llrint(v * 2^E_b) and adds q with an integer reduction into an
// int64 buffer laid out like the output.  Integer addition is associative, so the sum does not depend on the order in
// which CTAs and threads reach memory.  One narrowing pass then computes (double)sum * 2^-E_b (+ the caller's value
// when accumulating, in double) and rounds once to the output dtype.
//
// E_b comes from a bound M_b >= sum_i |v_i| for every output element of image b (stated per op where the factor is
// formed, api.cu):  E_b = 61 - e with M_b < 2^e, so |sum| <= M_b 2^E_b < 2^61.  The bound is on exact arithmetic.  Each
// partial is an fp32 sum of n products, off by at most gamma_n = n 2^-24 / (1 - n 2^-24) relative to the sum of their
// magnitudes; the longest such sum is the patch convolution's weight-gradient slice, n = PCW_DET_GROUPS * 128 = 2^15
// (gamma_n < 2^-8), then the GEMMs over 128 pixels or outputs (gamma_n < 2^-16).  With the +-1/2 of each llrint (n
// partials add at most n/2 < 2^40) this stays inside the one bit of margin below 2^62, so no partial sum and no total can
// reach 2^62 and int64 cannot overflow.
//
// Only the inputs of the bound are checked for non-finite values.  A partial that is non-finite for another reason (NaN
// or Inf logits or flow, say) converts to INT64_MIN in __double2ll_rn, and the sum it lands in is then meaningless (two
// such partials cancel to 0); the default path would return NaN there.  Callers that need NaN propagation from those
// inputs check them before the backward.
//
//   * 2^E_b is never formed in fp32: E_b can exceed 127 when the gradients are tiny.  The scale is applied in fp64 as
//     two factors 2^(E/2) * 2^(E - E/2), with E clamped to [-2000, 2000], so neither factor over- or underflows;
//     clamping E down only makes the quantum coarser.
//   * max|G_b| == 0: every partial is 0 and the output is exactly the caller's value (0 without accumulate).
//   * a non-finite value in the bound's inputs: E_b = FX_NONFINITE and every output of that fixed-point sum for that
//     image (for that call, for sums over the batch) is NaN.
#pragma once
#include <cfloat>
#include <climits>
#include <type_traits>

#include "common.cuh"

namespace gfla {

using fx_t = unsigned long long;               // two's-complement int64 sums, added as u64 (the same bits)
constexpr int FX_NONFINITE = INT_MIN;
constexpr int FX_EMAX = 2000;

// scale factors of exponent E: v * s.x * s.y == v * 2^E exactly (no intermediate over/underflow that could matter)
__device__ __forceinline__ double2 fx_scale(int e) {
    if (e == FX_NONFINITE) return make_double2(0.0, 0.0);
    const int h = e / 2;
    return make_double2(ldexp(1.0, h), ldexp(1.0, e - h));
}

__device__ __forceinline__ void fx_red(fx_t* p, long long q) {
    asm volatile("red.global.add.u64 [%0], %1;" ::"l"(p), "l"(q) : "memory");
}

// add one partial into the fixed-point sum at p
__device__ __forceinline__ void fx_add(fx_t* p, double v, double2 s) {
    const long long q = __double2ll_rn(v * s.x * s.y);
    if (q != 0) fx_red(p, q);
}

// the scatter-add of a backward kernel: fp/bf16 atomics (default instances) or the fixed-point sum (DET)
template <bool DET, typename P, typename A>
__device__ __forceinline__ void scatter_add(P* p, A v, double2 s) {
    if constexpr (DET) fx_add(p, static_cast<double>(v), s);
    else red_add(p, v);
}

// Workspace of one deterministic call (all offsets 256-byte aligned, the base must be 16-byte aligned):
//   sums   fx_t[n_sum]     the fixed-point sums (zeroed by the call)
//   exps   int[n_exp]      per-image exponents (then any per-call exponents)
//   amax   fx_t[n_amax]    the bit patterns of the maxima |x| as fp64 (zeroed by the call)
struct FxLayout {
    size_t sums, exps, amax, total;
};
inline size_t fx_round(size_t b) { return (b + 255) & ~size_t(255); }
inline FxLayout fx_layout(long long n_sum, int n_exp, int n_amax) {
    FxLayout l;
    l.sums = 0;
    l.exps = fx_round((size_t)n_sum * sizeof(fx_t));
    l.amax = l.exps + fx_round((size_t)n_exp * sizeof(int));
    l.total = l.amax + fx_round((size_t)n_amax * sizeof(fx_t));
    return l;
}

// host side (det_accum.cu).  All launch on `st_` and return GFLA_OK or a cudaError_t.
// amax[b] = max |x| over the n_img images of `per_img` elements each (bit patterns of fp64; amax must be zeroed)
int fx_amax(const void* x, int dtype, long long per_img, int n_img, fx_t* amax, cudaStream_t st_);
// exps[i] for i < n: exponent of M = factor * a[i] * (b ? b[0] : 1).  With over_all, one exponent (n = 1) of
// factor * max_i<n_a a[i] * (b ? b[0] : 1).
int fx_exponents(const fx_t* a, int n_a, const fx_t* b, double factor, bool over_all, int* exps, cudaStream_t st_);
// out[i] = round_to_dtype((double)sum[i] * 2^-exps[i / per_img] (+ out[i] when accumulate)); NaN for FX_NONFINITE
int fx_narrow(const fx_t* sums, const int* exps, long long per_img, long long n, void* out, int dtype, int accumulate,
              cudaStream_t st_);

}  // namespace gfla
