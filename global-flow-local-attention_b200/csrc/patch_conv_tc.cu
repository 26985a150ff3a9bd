// Patch convolution on the tensor cores (channels-last bf16 source, fp32 flow, C % 64 == 0, N = 128):
//     out = conv2d(BlockExtractor(k)(source, flow), weight, stride = k)
// (ExtractorAttn's source half, base_function.py:800,805,807) computed as an implicit GEMM whose A operand is gathered
// and blended on the fly: the [B,C,kH,kW] block tensor and its gradient are never written.
//
//   * forward  k_patch_conv_fwd_tc   per 16x8 pixel group: out[128 px][128 n] = sum over K = (tap, 64-channel chunk) of
//     A[128 px][64 ch] * W_t[64 ch][128 n].  A is blended from the four bilinear corners of the tap with the expression and
//     rounding of k_block_extract_fwd, so it is bit-identical to what BlockExtractor stores; W_t arrives by cp.async.
//   * backward k_patch_conv_bwd_tc   per pixel group: GA[128 px][64 ch] = G[128 px][128 n] * W_t^T (fp32, never rounded
//     to bf16), then per pixel grad_flow from GA and the corner values (the formulas of k_block_extract_bwd) summed in
//     registers and written once, and grad_source = w_corner * GA added to an fp32 buffer with 16-byte reductions.
//   * weight gradient k_patch_conv_wgrad_tc   per (tap, chunk) and slice of pixel groups: grad_W[128 n][64 ch] =
//     G^T * A, A rebuilt with the forward's gather_row; slices are summed in an fp32 buffer with 16-byte reductions.
// Each stage of a K loop is double-buffered: the next step's cp.async and gather are issued into the other buffer while
// this step's MMAs run, with one __syncthreads per step.  mma.sync m16n8k16, bf16 in, fp32 accumulate.
#include <climits>

#include "tile_window.cuh"

namespace gfla {
namespace tc {

constexpr int PC_THREADS = 256;
constexpr int PC_N = 128;                     // output channels (hidden_nc of ExtractorAttn)
constexpr int PC_CK = 64;                     // channels per K chunk
constexpr int PC_ASTR = PC_CK * 2 + 16;       // bf16 row of one chunk + pad: 144 B, conflict-free ldmatrix rows
constexpr int PC_GSTR = PC_N * 2 + 16;        // bf16 row of 128 outputs + pad: 272 B
constexpr int PC_FSTR = PC_CK * 4 + 16;       // fp32 row of one chunk + pad: 272 B
constexpr int PC_ABYTES = 128 * PC_ASTR;      // one [128][64] bf16 operand
constexpr int PC_GBYTES = 128 * PC_GSTR;      // one [128][128] bf16 operand

constexpr int PCF_SMEM = 4 * PC_ABYTES;                            // forward: A and W_t, two buffers each
constexpr int PCB_SMEM = PC_GBYTES + 2 * PC_ABYTES + 128 * PC_FSTR;  // backward: G, W_t x 2, GA (fp32)
constexpr int PCW_SMEM = 2 * PC_GBYTES + 2 * PC_ABYTES;            // weight gradient: G x 2, A x 2

__device__ __forceinline__ void lds128f(uint32_t a, float (&v)[4]) {
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v[0]), "=f"(v[1]), "=f"(v[2]), "=f"(v[3]) : "r"(a) : "memory");
}
__device__ __forceinline__ void sts64f(uint32_t a, float x, float y) {
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(x), "f"(y) : "memory");
}
// 16-byte reduction: 4 fp32 values added element-wise
__device__ __forceinline__ void red_add_f32x4(float* p, float x, float y, float z, float w) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(x), "f"(y), "f"(z), "f"(w) : "memory");
}
__device__ __forceinline__ float bf_lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf_hi(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }
__device__ __forceinline__ uint32_t word(const uint4& v, int e) { return e == 0 ? v.x : e == 1 ? v.y : e == 2 ? v.z : v.w; }

// Tap (i, j) of pixel (px, py): its four bilinear corners LT, RT, LB, RB as source positions y Ws + x with their weights,
// evaluated like k_block_extract_fwd (block_extract.cu:38-41: axis_tap, then one rounded product per corner weight),
// plus the per-axis weights the flow gradient needs.
struct PatchTap {
    int o[4];
    float w[4];
    float wxlo, wxhi, wylo, wyhi;
};

__device__ __forceinline__ PatchTap patch_tap(float fx, float fy, int px, int py, int i, int j, int k, int Hs, int Ws) {
    const AxisTap<float> ty = axis_tap<float>(fy, i - k / 2, py, Hs);
    const AxisTap<float> tx = axis_tap<float>(fx, j - k / 2, px, Ws);
    PatchTap q;
    q.o[0] = ty.lo * Ws + tx.lo;
    q.o[1] = ty.lo * Ws + tx.hi;
    q.o[2] = ty.hi * Ws + tx.lo;
    q.o[3] = ty.hi * Ws + tx.hi;
    q.w[0] = __fmul_rn(tx.wlo, ty.wlo);
    q.w[1] = __fmul_rn(tx.whi, ty.wlo);
    q.w[2] = __fmul_rn(tx.wlo, ty.whi);
    q.w[3] = __fmul_rn(tx.whi, ty.whi);
    q.wxlo = tx.wlo; q.wxhi = tx.whi; q.wylo = ty.wlo; q.wyhi = ty.whi;
    return q;
}

// Row m of the gathered operand A for one tap and the channels [c0, c0 + 64): thread half h (the two threads of a row
// are neighbouring lanes) takes the 8-channel groups 2 g + h, so that the pair reads and writes 32 contiguous bytes.
// v = 0; v += wLT LT; v += wRT RT; v += wLB LB; v += wRB RB with every product and sum rounded on its own: the
// expression and order of k_block_extract_fwd, whose translation unit is compiled with -fmad=false.  A row of a pixel
// outside the image is zero.
__device__ __forceinline__ void gather_row(uint32_t row, const __nv_bfloat16* __restrict__ s_img, const PatchTap& q, bool valid,
                                           int C, int c0, int h) {
#pragma unroll 2      // two groups' 8 loads in flight: fully unrolled, the forward's 64 accumulators leave too few registers
    for (int g = 0; g < 4; ++g) {
        const int j = 2 * g + h;
        if (!valid) {
            sts128(row + j * 16, 0u, 0u, 0u, 0u);
            continue;
        }
        uint4 v[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) v[c] = __ldg(reinterpret_cast<const uint4*>(s_img + (long long)q.o[c] * C + c0 + j * 8));
        uint32_t r[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            float lo = 0.f, hi = 0.f;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                lo = __fadd_rn(lo, __fmul_rn(q.w[c], bf_lo(word(v[c], e))));
                hi = __fadd_rn(hi, __fmul_rn(q.w[c], bf_hi(word(v[c], e))));
            }
            r[e] = bf16_bits(lo) | (bf16_bits(hi) << 16);
        }
        sts128(row + j * 16, r[0], r[1], r[2], r[3]);
    }
}

// pixel group g (row-major within each image): image b, top-left pixel (gx0, gy0)
__device__ __forceinline__ void group_at(int g, int gcols, int grows, int& b, int& gx0, int& gy0) {
    const int gc = g % gcols, r = g / gcols;
    gx0 = gc * GW;
    gy0 = (r % grows) * GH;
    b = r / grows;
}

// stage the [128][128] bf16 grad_out tile of a pixel group by cp.async (pixels outside the image: zeros)
__device__ __forceinline__ void stage_g(uint32_t g_s, const __nv_bfloat16* __restrict__ go_img, int gx0, int gy0, int H, int W, int tid) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int idx = i * PC_THREADS + tid, m = idx >> 4, j = idx & 15;
        const int qx = gx0 + (m & 15), qy = gy0 + (m >> 4);
        const bool in = qx < W && qy < H;
        cp_async16(g_s + m * PC_GSTR + j * 16, in ? go_img + ((long long)qy * W + qx) * PC_N + j * 8 : go_img, in ? 16u : 0u);
    }
}

// stage W_t[128 n][64 ch] of tap t, channels [c0, c0 + 64) from the packed weight [N][k*k][C] by cp.async
__device__ __forceinline__ void stage_w(uint32_t w_s, const __nv_bfloat16* __restrict__ wpk, int t, int kk, int C, int c0, int tid) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int idx = i * PC_THREADS + tid, n = idx >> 3, j = idx & 7;
        cp_async16(w_s + n * PC_ASTR + j * 16, wpk + ((long long)n * kk + t) * C + c0 + j * 8);
    }
}

// ---------------------------------------------------------------------------------------------------------- forward
// Warp w computes output rows 32 (w & 3) .. +32 and columns 64 (w >> 2) .. +64.
__global__ void __launch_bounds__(PC_THREADS, 2)
k_patch_conv_fwd_tc(const __nv_bfloat16* __restrict__ src, const float* __restrict__ flow, const __nv_bfloat16* __restrict__ wpk,
                    __nv_bfloat16* __restrict__ out, int C, int Hs, int Ws, int H, int W, int k, int gcols, int grows) {
    extern __shared__ __align__(16) unsigned char smem[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, gid = lane >> 2, tig = lane & 3;
    const int wm = warp & 3, wn = warp >> 2;
    int b, gx0, gy0;
    group_at(blockIdx.x, gcols, grows, b, gx0, gy0);
    const long long hw = (long long)H * W;
    // this thread's half of gather row m
    const int m = tid >> 1, h = tid & 1, px = gx0 + (m & 15), py = gy0 + (m >> 4);
    const bool valid = px < W && py < H;
    const float fx = valid ? flow[(long long)b * 2 * hw + (long long)py * W + px] : 0.f;
    const float fy = valid ? flow[(long long)b * 2 * hw + hw + (long long)py * W + px] : 0.f;
    const __nv_bfloat16* s_img = src + (long long)b * Hs * Ws * C;

    const uint32_t sb = smem_u32(smem), a_base = sb, w_base = sb + 2 * PC_ABYTES;
    const int nch = C / PC_CK, kk2 = k * k, steps = kk2 * nch;
    // step s = tap t * nch + chunk; its weight slice goes by cp.async, its A rows are gathered by the threads
    auto stage_weight = [&](int s, int buf) {
        const int t = s / nch;
        stage_w(w_base + buf * PC_ABYTES, wpk, t, kk2, C, (s - t * nch) * PC_CK, tid);
        cp_async_commit();
    };
    auto stage_a = [&](int s, int buf) {
        const int t = s / nch;
        const PatchTap q = patch_tap(fx, fy, px, py, t / k, t % k, k, Hs, Ws);
        gather_row(a_base + buf * PC_ABYTES + m * PC_ASTR, s_img, q, valid, C, (s - t * nch) * PC_CK, h);
    };

    float acc[2][8][4];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[i][j][q] = 0.f;
    const uint32_t a_frag = a_base + (wm * 32 + (lane & 15)) * PC_ASTR + (lane >> 4) * 16;
    const uint32_t b_frag = w_base + (wn * 64 + (lane & 7) + ((lane >> 4) << 3)) * PC_ASTR + ((lane >> 3) & 1) * 16;

    stage_weight(0, 0);
    stage_a(0, 0);
    cp_async_wait_all();
    __syncthreads();
    for (int s = 0; s < steps; ++s) {
        const int buf = s & 1;
        if (s + 1 < steps) stage_weight(s + 1, buf ^ 1);
#pragma unroll
        for (int kq = 0; kq < PC_CK / 16; ++kq) {
            uint32_t a0[4], a1[4];
            ldsm_x4(a_frag + buf * PC_ABYTES + kq * 32, a0);
            ldsm_x4(a_frag + buf * PC_ABYTES + 16 * PC_ASTR + kq * 32, a1);
#pragma unroll
            for (int np = 0; np < 4; ++np) {
                uint32_t bf[4];
                ldsm_x4(b_frag + buf * PC_ABYTES + np * 16 * PC_ASTR + kq * 32, bf);
                mma_bf16(acc[0][2 * np], a0, bf[0], bf[1]);
                mma_bf16(acc[0][2 * np + 1], a0, bf[2], bf[3]);
                mma_bf16(acc[1][2 * np], a1, bf[0], bf[1]);
                mma_bf16(acc[1][2 * np + 1], a1, bf[2], bf[3]);
            }
        }
        if (s + 1 < steps) stage_a(s + 1, buf ^ 1);
        cp_async_wait_all();
        __syncthreads();      // step s+1's operands complete; everybody is done reading step s's buffers
    }
    // epilogue: one bf16 rounding per output, channels-last rows of 128 outputs
    __nv_bfloat16* o_img = out + (long long)b * hw * PC_N;
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            const int r = wm * 32 + mt * 16 + gid + 8 * hh, qx = gx0 + (r & 15), qy = gy0 + (r >> 4);
            if (qx >= W || qy >= H) continue;
            __nv_bfloat16* o = o_img + ((long long)qy * W + qx) * PC_N + wn * 64 + 2 * tig;
#pragma unroll
            for (int nt = 0; nt < 8; ++nt)
                *reinterpret_cast<__nv_bfloat162*>(o + nt * 8) = __floats2bfloat162_rn(acc[mt][nt][2 * hh], acc[mt][nt][2 * hh + 1]);
        }
}

// --------------------------------------------------------------------------------------------- backward: data gradients
// Warp w computes GA rows 16 w .. +16 (all 64 channels of the chunk); its A fragments of G stay in registers for the whole
// K loop.  Then every thread takes half a pixel row of GA, as in the forward's gather.
__global__ void __launch_bounds__(PC_THREADS, 2)
k_patch_conv_bwd_tc(const __nv_bfloat16* __restrict__ src, const float* __restrict__ flow, const __nv_bfloat16* __restrict__ wpk,
                    const __nv_bfloat16* __restrict__ gout, float* __restrict__ gsrc, float* __restrict__ gflow, int C, int Hs,
                    int Ws, int H, int W, int k, int gcols, int grows, int accumulate) {
    extern __shared__ __align__(16) unsigned char smem[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, gid = lane >> 2, tig = lane & 3;
    int b, gx0, gy0;
    group_at(blockIdx.x, gcols, grows, b, gx0, gy0);
    const long long hw = (long long)H * W;
    const int m = tid >> 1, h = tid & 1, px = gx0 + (m & 15), py = gy0 + (m >> 4);
    const bool valid = px < W && py < H;
    const long long fofs = (long long)b * 2 * hw + (long long)py * W + px;
    const float fx = valid ? flow[fofs] : 0.f, fy = valid ? flow[fofs + hw] : 0.f;
    const __nv_bfloat16* s_img = src + (long long)b * Hs * Ws * C;
    float* gs_img = gsrc + (long long)b * Hs * Ws * C;

    const uint32_t sb = smem_u32(smem), g_base = sb, w_base = sb + PC_GBYTES, f_base = w_base + 2 * PC_ABYTES;
    const int nch = C / PC_CK, kk2 = k * k, steps = kk2 * nch;
    stage_g(g_base, gout + (long long)b * hw * PC_N, gx0, gy0, H, W, tid);
    stage_w(w_base, wpk, 0, kk2, C, 0, tid);
    cp_async_commit();
    cp_async_wait_all();
    __syncthreads();
    uint32_t ga[8][4];      // A fragments of this warp's 16 rows of G, k-steps over the 128 outputs
#pragma unroll
    for (int kq = 0; kq < 8; ++kq) ldsm_x4(g_base + (warp * 16 + (lane & 15)) * PC_GSTR + kq * 32 + (lane >> 4) * 16, ga[kq]);
    const uint32_t wt_frag = w_base + (lane & 15) * PC_ASTR + (lane >> 4) * 16;   // B = W_t^T: ldmatrix.trans of [n][ch]
    const uint32_t f_row = f_base + m * PC_FSTR;

    float gx = 0.f, gy = 0.f;
    for (int s = 0; s < steps; ++s) {
        const int buf = s & 1, t = s / nch, c0 = (s - t * nch) * PC_CK;
        if (s + 1 < steps) {
            const int tn = (s + 1) / nch;
            stage_w(w_base + (buf ^ 1) * PC_ABYTES, wpk, tn, kk2, C, (s + 1 - tn * nch) * PC_CK, tid);
            cp_async_commit();
        }
        float acc[8][4];
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[nt][q] = 0.f;
#pragma unroll
        for (int kq = 0; kq < 8; ++kq)
#pragma unroll
            for (int np = 0; np < 4; ++np) {
                uint32_t bw[4];
                ldsm_x4_t(wt_frag + buf * PC_ABYTES + kq * 16 * PC_ASTR + np * 32, bw);
                mma_bf16(acc[2 * np], ga[kq], bw[0], bw[1]);
                mma_bf16(acc[2 * np + 1], ga[kq], bw[2], bw[3]);
            }
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            const uint32_t row = f_base + (warp * 16 + gid + 8 * hh) * PC_FSTR + 2 * tig * 4;
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) sts64f(row + nt * 32, acc[nt][2 * hh], acc[nt][2 * hh + 1]);
        }
        __syncthreads();      // GA of the step complete
        if (valid) {
            const PatchTap q = patch_tap(fx, fy, px, py, t / k, t % k, k, Hs, Ws);
#pragma unroll
            for (int g = 0; g < 4; ++g) {
                const int j = 2 * g + h;
                float a[8];
                {
                    float a0[4], a1[4];
                    lds128f(f_row + j * 32, a0);
                    lds128f(f_row + j * 32 + 16, a1);
#pragma unroll
                    for (int e = 0; e < 4; ++e) { a[e] = a0[e]; a[4 + e] = a1[e]; }
                }
                uint4 v[4];
#pragma unroll
                for (int c = 0; c < 4; ++c) v[c] = __ldg(reinterpret_cast<const uint4*>(s_img + (long long)q.o[c] * C + c0 + j * 8));
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    const uint32_t sh = (e & 1) ? 0u : 16u;
                    const float vLT = __uint_as_float((word(v[0], e >> 1) << sh) & 0xffff0000u);
                    const float vRT = __uint_as_float((word(v[1], e >> 1) << sh) & 0xffff0000u);
                    const float vLB = __uint_as_float((word(v[2], e >> 1) << sh) & 0xffff0000u);
                    const float vRB = __uint_as_float((word(v[3], e >> 1) << sh) & 0xffff0000u);
                    gy += a[e] * (-q.wxlo * vLT - q.wxhi * vRT + q.wxlo * vLB + q.wxhi * vRB);   // block_extract.cu:92-93
                    gx += a[e] * (-q.wylo * vLT - q.wyhi * vLB + q.wylo * vRT + q.wyhi * vRB);
                }
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    float* d = gs_img + (long long)q.o[c] * C + c0 + j * 8;
                    const float w = q.w[c];
                    red_add_f32x4(d, w * a[0], w * a[1], w * a[2], w * a[3]);
                    red_add_f32x4(d + 4, w * a[4], w * a[5], w * a[6], w * a[7]);
                }
            }
        }
        cp_async_wait_all();
        __syncthreads();      // W_t of step s+1 complete; GA of step s read by everybody
    }
    // the two halves of the pixel's sum, in a fixed order: deterministic, written once
    gx += __shfl_xor_sync(0xffffffffu, gx, 1);
    gy += __shfl_xor_sync(0xffffffffu, gy, 1);
    if (valid && h == 0) {
        gflow[fofs] = accumulate ? gflow[fofs] + gx : gx;
        gflow[fofs + hw] = accumulate ? gflow[fofs + hw] + gy : gy;
    }
}

// ------------------------------------------------------------------------------------------- backward: weight gradient
// CTA (blockIdx.x = tap t * nch + chunk, blockIdx.y = slice of pixel groups): grad_W[128 n][64 ch] += G^T A over its groups.
// Warp w computes rows n 32 (w & 3) .. +32 and channels 32 (w >> 2) .. +32; both operands come through ldmatrix.trans.
__global__ void __launch_bounds__(PC_THREADS, 2)
k_patch_conv_wgrad_tc(const __nv_bfloat16* __restrict__ src, const float* __restrict__ flow, const __nv_bfloat16* __restrict__ gout,
                      float* __restrict__ gw, int C, int Hs, int Ws, int H, int W, int k, int gcols, int grows, int ngroups,
                      int per_slice) {
    extern __shared__ __align__(16) unsigned char smem[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, gid = lane >> 2, tig = lane & 3;
    const int wm = warp & 3, wn = warp >> 2;
    const int nch = C / PC_CK, t = blockIdx.x / nch, c0 = (blockIdx.x - t * nch) * PC_CK;
    const int g0 = blockIdx.y * per_slice, g1 = min(ngroups, g0 + per_slice);
    const long long hw = (long long)H * W;
    const int m = tid >> 1, h = tid & 1;
    const uint32_t sb = smem_u32(smem), g_base = sb, a_base = sb + 2 * PC_GBYTES;

    // pixel group g: its grad_out tile goes by cp.async, its A rows (the forward's gather) are built by the threads
    auto stage_gout = [&](int g, int buf) {
        int b, gx0, gy0;
        group_at(g, gcols, grows, b, gx0, gy0);
        stage_g(g_base + buf * PC_GBYTES, gout + (long long)b * hw * PC_N, gx0, gy0, H, W, tid);
        cp_async_commit();
    };
    auto stage_a = [&](int g, int buf) {
        int b, gx0, gy0;
        group_at(g, gcols, grows, b, gx0, gy0);
        const int px = gx0 + (m & 15), py = gy0 + (m >> 4);
        const bool valid = px < W && py < H;
        const long long fofs = (long long)b * 2 * hw + (long long)py * W + px;
        const float fx = valid ? flow[fofs] : 0.f, fy = valid ? flow[fofs + hw] : 0.f;
        const PatchTap q = patch_tap(fx, fy, px, py, t / k, t % k, k, Hs, Ws);
        gather_row(a_base + buf * PC_ABYTES + m * PC_ASTR, src + (long long)b * Hs * Ws * C, q, valid, C, c0, h);
    };

    float acc[2][4][4];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[i][j][q] = 0.f;
    // A = G^T [n][px] from G [px][n]; B = A^T-as-col [ch][px] from A [px][ch]
    const uint32_t gt_frag = g_base + ((lane & 7) + ((lane >> 4) << 3)) * PC_GSTR + (wm * 32 + ((lane >> 3) & 1) * 8) * 2;
    const uint32_t at_frag = a_base + (lane & 15) * PC_ASTR + (wn * 32 + (lane >> 4) * 8) * 2;

    if (g0 < g1) {
        stage_gout(g0, 0);
        stage_a(g0, 0);
    }
    cp_async_wait_all();
    __syncthreads();
    for (int g = g0; g < g1; ++g) {
        const int buf = (g - g0) & 1;
        if (g + 1 < g1) stage_gout(g + 1, buf ^ 1);
#pragma unroll
        for (int kq = 0; kq < 8; ++kq) {
            uint32_t a0[4], a1[4];
            ldsm_x4_t(gt_frag + buf * PC_GBYTES + kq * 16 * PC_GSTR, a0);
            ldsm_x4_t(gt_frag + buf * PC_GBYTES + kq * 16 * PC_GSTR + 32, a1);
#pragma unroll
            for (int np = 0; np < 2; ++np) {
                uint32_t bf[4];
                ldsm_x4_t(at_frag + buf * PC_ABYTES + kq * 16 * PC_ASTR + np * 32, bf);
                mma_bf16(acc[0][2 * np], a0, bf[0], bf[1]);
                mma_bf16(acc[0][2 * np + 1], a0, bf[2], bf[3]);
                mma_bf16(acc[1][2 * np], a1, bf[0], bf[1]);
                mma_bf16(acc[1][2 * np + 1], a1, bf[2], bf[3]);
            }
        }
        if (g + 1 < g1) stage_a(g + 1, buf ^ 1);
        cp_async_wait_all();
        __syncthreads();      // group g+1's operands complete; everybody is done reading group g's buffers
    }
    // the slice's sums through shared memory (fp32 [128 n][64 ch], over the G buffers), then 16-byte reductions
    const uint32_t f_base = g_base;
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            const uint32_t row = f_base + (wm * 32 + mt * 16 + gid + 8 * hh) * PC_FSTR + (wn * 32 + 2 * tig) * 4;
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) sts64f(row + nt * 32, acc[mt][nt][2 * hh], acc[mt][nt][2 * hh + 1]);
        }
    __syncthreads();
    const int kk2 = k * k;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int idx = i * PC_THREADS + tid, n = idx >> 4, j = idx & 15;
        float v[4];
        lds128f(f_base + n * PC_FSTR + j * 16, v);
        red_add_f32x4(gw + ((long long)n * kk2 + t) * C + c0 + j * 4, v[0], v[1], v[2], v[3]);
    }
}

}  // namespace tc

bool patch_conv_supported(int C, int N, int dtype, int flow_dtype, int layout) {
    return dtype == GFLA_BF16 && flow_dtype == GFLA_F32 && layout == GFLA_NHWC && C % tc::PC_CK == 0 && N == tc::PC_N;
}

static int set_smem(const void* kern, int bytes) {
    const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    return e == cudaSuccess ? GFLA_OK : static_cast<int>(e);
}

int patch_conv_fwd(const void* src, const void* flow, const void* weight, void* out, int B, int C, int Hs, int Ws, int H, int W,
                   int k, cudaStream_t st_) {
    using namespace tc;
    const int gcols = (W + GW - 1) / GW, grows = (H + GH - 1) / GH;
    const long long ngroups = (long long)B * gcols * grows;
    if (ngroups > INT_MAX) return GFLA_E_SHAPE;
    int r = set_smem((const void*)k_patch_conv_fwd_tc, PCF_SMEM);
    if (r != GFLA_OK) return r;
    k_patch_conv_fwd_tc<<<(unsigned)ngroups, PC_THREADS, PCF_SMEM, st_>>>((const __nv_bfloat16*)src, (const float*)flow,
                                                                        (const __nv_bfloat16*)weight, (__nv_bfloat16*)out, C, Hs, Ws,
                                                                        H, W, k, gcols, grows);
    return launch_status();
}

// accumulate = 0: the fp32 grad_source and grad_weight buffers are zero-filled here and grad_flow is overwritten; 1: all
// three gradients are added into the caller's buffers
int patch_conv_bwd(const void* src, const void* flow, const void* weight, const void* gout, void* gsrc, void* gflow, void* gweight,
                   int B, int C, int Hs, int Ws, int H, int W, int k, int accumulate, cudaStream_t st_) {
    using namespace tc;
    const int gcols = (W + GW - 1) / GW, grows = (H + GH - 1) / GH;
    const long long ngroups = (long long)B * gcols * grows;
    if (ngroups > INT_MAX) return GFLA_E_SHAPE;
    if (!accumulate) {
        int z = zero_async(gsrc, (size_t)B * Hs * Ws * C * sizeof(float), st_);
        if (z == GFLA_OK) z = zero_async(gweight, (size_t)PC_N * k * k * C * sizeof(float), st_);
        if (z != GFLA_OK) return z;
    }
    int r = set_smem((const void*)k_patch_conv_bwd_tc, PCB_SMEM);
    if (r == GFLA_OK) r = set_smem((const void*)k_patch_conv_wgrad_tc, PCW_SMEM);
    if (r != GFLA_OK) return r;
    k_patch_conv_bwd_tc<<<(unsigned)ngroups, PC_THREADS, PCB_SMEM, st_>>>((const __nv_bfloat16*)src, (const float*)flow,
                                                                        (const __nv_bfloat16*)weight, (const __nv_bfloat16*)gout,
                                                                        (float*)gsrc, (float*)gflow, C, Hs, Ws, H, W, k, gcols,
                                                                        grows, accumulate);
    r = launch_status();
    if (r != GFLA_OK) return r;
    // weight gradient: (tap, chunk) pairs x slices of pixel groups, about four CTAs per SM in all
    const int pairs = k * k * (C / PC_CK);
    const long long want = (4LL * sm_count() + pairs - 1) / pairs;
    const int per_slice = (int)((ngroups + want - 1) / want);
    const int slices = (int)((ngroups + per_slice - 1) / per_slice);
    k_patch_conv_wgrad_tc<<<dim3((unsigned)pairs, (unsigned)slices), PC_THREADS, PCW_SMEM, st_>>>(
        (const __nv_bfloat16*)src, (const float*)flow, (const __nv_bfloat16*)gout, (float*)gweight, C, Hs, Ws, H, W, k, gcols, grows,
        (int)ngroups, per_slice);
    return launch_status();
}

}  // namespace gfla
