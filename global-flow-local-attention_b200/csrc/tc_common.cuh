// sm_90a building blocks shared by the tensor-core tile kernels: cp.async staging, ldmatrix fragment loads and
// the warp-level bf16 MMA (m16n8k16, fp32 accumulate).  Raw PTX, no CUTLASS dependency.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "gfla_warp.h"

namespace gfla {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

// explicit shared-space accesses (32-bit shared addresses): keeps ptxas from falling back to generic LD/ST
__device__ __forceinline__ void sts128(uint32_t a, uint32_t x, uint32_t y, uint32_t z, uint32_t w) {
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(x), "r"(y), "r"(z), "r"(w) : "memory");
}
__device__ __forceinline__ void sts16(uint32_t a, uint32_t v) {
    asm volatile("{\n\t.reg .b16 h;\n\tcvt.u16.u32 h, %1;\n\tst.shared.b16 [%0], h;\n\t}" ::"r"(a), "r"(v) : "memory");
}
__device__ __forceinline__ void stsf(uint32_t a, float v) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(a), "f"(v) : "memory"); }
__device__ __forceinline__ float ldsf(uint32_t a) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a) : "memory");
    return v;
}

// ------------------------------------------------------------------ cp.async (global -> shared, 16 bytes)
// src_bytes = 0 zero-fills the destination without reading global memory
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, uint32_t src_bytes = 16) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
// wait until at most N of this thread's committed groups are still in flight
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// ------------------------------------------------------------------ ldmatrix / mma
// four 8x8 b16 matrices; lane l supplies the row address of matrix l/8
__device__ __forceinline__ void ldsm_x4(uint32_t a, uint32_t (&r)[4]) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a) : "memory");
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t a, uint32_t (&r)[4]) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a) : "memory");
}
// D (+)= A[16x16, row] * B[16x8, col], bf16 in, fp32 accumulate (warp-collective)
__device__ __forceinline__ void mma_bf16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// ------------------------------------------------------------------ named barriers and register reallocation
// bar.arrive signals without waiting; bar.sync waits until n threads (a multiple of 32) have arrived or synced on the
// barrier id.  Both order this thread's earlier shared-memory accesses before the accesses of the threads that sync.
__device__ __forceinline__ void bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void bar_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }
// per-thread register budget of the executing warp (sm_90a, warp-uniform; the kernel's launch bounds fix the starting
// budget).  A warp that raises its budget waits until other warps of the CTA have released enough.
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }

__device__ __forceinline__ uint32_t bf16_bits(float v) {
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    return static_cast<uint32_t>(*reinterpret_cast<const unsigned short*>(&h));
}

// Division of group indices by run-time image geometry: magic multiplier computed once, then umulhi + shift per use.
// Exact for 0 <= n < 2^31, d >= 1.
struct FastDiv {
    uint32_t d, mul, shr;
    __device__ __forceinline__ void init(uint32_t div) {
        d = div;
        if (div <= 1) { mul = 0; shr = 0; return; }
        const uint32_t p = 31 + (32 - __clz(div - 1));           // 31 + ceil(log2(div))
        mul = static_cast<uint32_t>(((1ull << p) + div - 1) / div);
        shr = p - 32;
    }
    __device__ __forceinline__ uint32_t div(uint32_t n) const { return d != 1 ? __umulhi(n, mul) >> shr : n; }
    __device__ __forceinline__ void divmod(uint32_t n, uint32_t& q, uint32_t& r) const { q = div(n); r = n - q * d; }
};

}  // namespace tc
}  // namespace gfla
