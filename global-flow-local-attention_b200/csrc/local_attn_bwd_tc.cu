// Fused local-attention backward on the tensor cores (channels-last bf16 or fp16, fp32 flow, k in {3, 5}): ONE kernel for
// grad_source, grad_flow and grad_logits.  T, the data's 16-bit type, is also the type of the weight slab and of the
// grad_source partials; P stays fp32 in shared memory.
//
// Per 16x8 pixel group and 16-position row segment of the group's tap footprint (channels in passes of CN):
//   * P[128 px][16 pos] = G[128 px][CN] * S[16 pos][CN]^T    the grad_out . source dot products of every pixel with
//     every position of the segment; each pixel thread then picks its (k+1)^2 window entries out of P into Q (registers).
//     Q is exactly the CUDA-core kernel's Q (local_attn.cu), so grad_flow / grad_logits follow from it per pixel with
//     the same formulas (local_attn_pixel.cuh);
//   * GS[16 pos][CN] = Wfull^T[16 pos][128 px] * G[128 px][CN] grad_source of the segment, added with 16-byte T
//     reductions (the caller's buffer is zero-filled first unless the call accumulates).  Border positions, where the
//     windows folded onto the image edge pile up, are summed in an fp32 scratch instead and rounded once (k_fold_border).
// The grad_out tile G stays in shared memory for the whole pass; the source segment arrives by cp.async one step ahead.
// Two warpgroups share a CTA and run the two GEMMs of a step side by side (mma.sync m16n8k16):
//   * pixel warpgroup, warps 0-3: thread tid owns pixel tid; warp w owns pixel rows 32w..32w+31 of the P GEMM.  It
//     scatters the step's weight slab, runs P and the Q pick, and at the end computes grad_flow and grad_logits;
//   * grad_source warpgroup, warps 4-7: warp 4 + v owns channels [v CN/4, (v+1) CN/4) of the GS GEMM and its reductions.
// The weight slab and its row bits rotate through three buffers.  The pixel warpgroup signals "slab s written" (named
// barrier FULL), the grad_source warpgroup reads it, zeroes it and signals "slab s free" (FREE), which the pixel
// warpgroup waits for before it scatters step s + 3 into the same buffer: it may run up to two steps ahead.
// A 16-pixel group row none of whose windows meets the step (window_meets_step) is skipped as a P m-tile and as a GS
// k-step; the pixel warps publish these row bits next to the step's weight slab.  Steps that no pixel touches do no MMAs.
// Pixels whose taps are not consecutive integers take the reference's literal 4-tap arithmetic, one warp per pixel.
#include <mutex>

#include "det_accum.cuh"
#include "tile_window.cuh"

namespace gfla {
namespace tc {

constexpr int BT_THREADS = 256;                 // pixel warpgroup (warps 0-3) + grad_source warpgroup (warps 4-7)
// per-thread registers of the two roles after setmaxnreg: they sum to 256, the 128 per thread that 2 CTAs per SM leave
constexpr int BT_PIX_REGS = 168, BT_GS_REGS = 88;
// named barriers (0 is __syncthreads)
constexpr int BT_BAR_PASS = 1;                  // all threads: a pass's G is complete, or the previous pass is done with it
constexpr int BT_BAR_PIX = 2;                   // pixel warpgroup: the step's source segment is complete
constexpr int BT_BAR_GS = 3;                    // grad_source warpgroup: every warp has read the step's slab
constexpr int BT_BAR_FULL = 4;                  // + buffer: slab and row bits written (pixel arrives, grad_source syncs)
constexpr int BT_BAR_FREE = 7;                  // + buffer: slab read and zeroed (grad_source arrives, pixel syncs)
constexpr int BT_AWSTR = 128 * 2 + 16;          // transposed weight slab row (one position, 128 pixels) + pad
constexpr int BT_PSTR = SEG + 1;                // P row (floats): odd stride, conflict-free per-pixel reads

constexpr int BT_NAW = 3;                       // weight slabs (and row-bit words) in rotation

template <int CN>
struct BwdSmem {
    static constexpr int GSTR = CN * 2 + 16;
    static constexpr int G = 0;
    static constexpr int S = G + 128 * GSTR;
    static constexpr int AW = S + 2 * SEG * GSTR;
    static constexpr int P = AW + BT_NAW * SEG * BT_AWSTR;
    static constexpr int IRR = P + 128 * BT_PSTR * 4;
    static constexpr int ROWS = IRR + 129 * 4;      // per slab buffer: byte w = warp_row_bits of warp w for the step
    static constexpr int ALLOC = ROWS + BT_NAW * 4;
};

// 16-byte reduction: 8 T values added element-wise, each add rounded once (fp16: a sum beyond 65504 becomes Inf)
__device__ __forceinline__ void red_add_16x8(__nv_bfloat16* p, const uint32_t (&v)[4]) {
    asm volatile("red.global.add.noftz.v4.bf16x2 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v[0]), "r"(v[1]), "r"(v[2]), "r"(v[3])
                 : "memory");
}
__device__ __forceinline__ void red_add_16x8(__half* p, const uint32_t (&v)[4]) {
    asm volatile("red.global.add.noftz.v4.f16x2 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v[0]), "r"(v[1]), "r"(v[2]), "r"(v[3])
                 : "memory");
}

// 4x4 transpose of 32-bit words across the four lanes 4 g + t of a quad: on return lane t holds in v[n] what lane n held
// in v[t].  Two butterfly rounds (lane distance 2, then 1), each trading two words.
__device__ __forceinline__ void quad_transpose(uint32_t (&v)[4], int t) {
    const bool t1 = (t & 2) != 0, t0 = (t & 1) != 0;
    uint32_t y0 = __shfl_xor_sync(0xffffffffu, t1 ? v[0] : v[2], 2);
    uint32_t y1 = __shfl_xor_sync(0xffffffffu, t1 ? v[1] : v[3], 2);
    if (t1) { v[0] = y0; v[1] = y1; } else { v[2] = y0; v[3] = y1; }
    y0 = __shfl_xor_sync(0xffffffffu, t0 ? v[0] : v[1], 1);
    y1 = __shfl_xor_sync(0xffffffffu, t0 ? v[2] : v[3], 1);
    if (t0) { v[0] = y0; v[2] = y1; } else { v[1] = y0; v[3] = y1; }
}

// P GEMM of one warp for one step: the m-tiles whose pixel row is active (M0, M1) of its 32 pixels x 16 positions
template <typename T, int CN, bool M0, bool M1>
__device__ __forceinline__ void p_gemm(uint32_t ga, uint32_t sf, float (&pacc)[2][2][4]) {
    constexpr int GSTR = BwdSmem<CN>::GSTR;
#pragma unroll 4
    for (int kk = 0; kk < CN / 16; ++kk) {
        uint32_t a0[4], a1[4], bf[4];
        if (M0) ldsm_x4(ga + kk * 32, a0);
        if (M1) ldsm_x4(ga + 16 * GSTR + kk * 32, a1);
        ldsm_x4(sf + kk * 32, bf);
        if (M0) {
            mma16<T>(pacc[0][0], a0, bf[0], bf[1]);
            mma16<T>(pacc[0][1], a0, bf[2], bf[3]);
        }
        if (M1) {
            mma16<T>(pacc[1][0], a1, bf[0], bf[1]);
            mma16<T>(pacc[1][1], a1, bf[2], bf[3]);
        }
    }
}

// Slot of source position (y, x) on the image border (rows 0 and Hs-1, then columns 0 and Ws-1 of the rows between), in
// [0, 2 (Hs + Ws)); -1 inside the image.  Windows folded onto the edge make border positions collect a share of nearly
// every group of a border-clamped flow, and one 16-bit atomic add per group would round each time.  Their grad_source is
// summed in an fp32 buffer instead and rounded once by k_fold_border.
__device__ __forceinline__ int border_slot(int y, int x, int Hs, int Ws) {
    if (y == 0) return x;
    if (y == Hs - 1) return Ws + x;
    if (x == 0) return 2 * Ws + y;
    if (x == Ws - 1) return 2 * Ws + Hs + y;
    return -1;
}

// grad_out tile of the group for channels [c0, c0 + CN) into G, loaded by both warpgroups (pixels outside the image:
// zeros).  Not fully unrolled: the compiler would then keep all the pass-invariant 64-bit addresses live across the step
// loop, and at CN = 256 that spills.
template <typename T, int CN>
__device__ __forceinline__ void load_g_tile(uint32_t g_base, const T* __restrict__ go_b, int c0, int C, int gx0, int gy0,
                                            int H, int W, int tid) {
    constexpr int GSTR = BwdSmem<CN>::GSTR;
#pragma unroll 4
    for (int i = 0; i < CN / 16; ++i) {
        const int idx = i * BT_THREADS + tid, m = idx / (CN / 8), j = idx % (CN / 8);
        const int qx = gx0 + (m & 15), qy = gy0 + (m >> 4);
        const bool in = qx < W && qy < H;
        cp_async16(g_base + m * GSTR + j * 16, in ? go_b + ((long long)qy * W + qx) * C + c0 + j * 8 : go_b, in ? 16u : 0u);
    }
    cp_async_commit();
}

template <typename T, int K, bool DET>
__device__ __forceinline__ void irregular_pixel_bwd(const T* __restrict__ src, const float* __restrict__ flow, const T* __restrict__ logits,
                                                    const T* __restrict__ gout, T* __restrict__ gsrc, float* __restrict__ gflow,
                                                    T* __restrict__ glogits, int b, int C, int Hs, int Ws, int H, int W,
                                                    int qx, int qy, int accumulate, int lane, fx_t* __restrict__ gsum,
                                                    double2 fsc) {
    constexpr int KK = K * K;
    const long long hw = (long long)H * W, qofs = (long long)qy * W + qx;
    const float fx = flow[(long long)b * 2 * hw + qofs], fy = flow[(long long)b * 2 * hw + hw + qofs];
    float p[KK], dp[KK];
    pixel_softmax<T, float, KK>(logits + (long long)b * KK * hw + qofs, hw, KK, p);
    const float inv_kk = 1.0f / static_cast<float>(KK);
    const T* s = src + (long long)b * Hs * Ws * C;
    using GS = std::conditional_t<DET, fx_t, T>;
    GS* gs;
    if constexpr (DET) gs = gsum + (long long)b * Hs * Ws * C;
    else gs = gsrc + (long long)b * Hs * Ws * C;
    const T* go = gout + ((long long)b * hw + qofs) * C;
    float gfx = 0.f, gfy = 0.f;
#pragma unroll
    for (int i = 0; i < K; ++i) {
        const AxisTap<float> ty = axis_tap<float>(fy, i - K / 2, qy, Hs);
#pragma unroll
        for (int j = 0; j < K; ++j) {
            const AxisTap<float> tx = axis_tap<float>(fx, j - K / 2, qx, Ws);
            const long long oLT = ((long long)ty.lo * Ws + tx.lo) * C, oRT = ((long long)ty.lo * Ws + tx.hi) * C,
                            oLB = ((long long)ty.hi * Ws + tx.lo) * C, oRB = ((long long)ty.hi * Ws + tx.hi) * C;
            const float pij = p[i * K + j] * inv_kk;
            float q[4] = {0.f, 0.f, 0.f, 0.f};
            for (int c = lane; c < C; c += 32) {
                const float g = ld(go + c);
                q[0] += g * ld(s + oLT + c);
                q[1] += g * ld(s + oRT + c);
                q[2] += g * ld(s + oLB + c);
                q[3] += g * ld(s + oRB + c);
                const float gp = g * pij;
                scatter_add<DET>(gs + oLT + c, gp * (tx.wlo * ty.wlo), fsc);
                scatter_add<DET>(gs + oRT + c, gp * (tx.whi * ty.wlo), fsc);
                scatter_add<DET>(gs + oLB + c, gp * (tx.wlo * ty.whi), fsc);
                scatter_add<DET>(gs + oRB + c, gp * (tx.whi * ty.whi), fsc);
            }
#pragma unroll
            for (int t = 0; t < 4; ++t)
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) q[t] += __shfl_xor_sync(0xffffffffu, q[t], o);
            dp[i * K + j] = tap_backward<float>(tx, ty, pij, inv_kk, q[0], q[1], q[2], q[3], gfx, gfy);
        }
    }
    if (lane == 0)
        store_pixel_grads<T, float, float, KK>(p, dp, KK, gfx, gfy, glogits + (long long)b * KK * hw + qofs,
                                               gflow + (long long)b * 2 * hw + qofs, hw, accumulate);
}

// DET: grad_source goes into the fixed-point sums gsum with the image's exponent fx_exp[b] (det_accum.cuh); gsrc and
// gborder are unused.  T comes last (here and in the forward kernels), so an instance's name still begins with its
// shape parameters, k_local_attn_bwd_tc<K, CN, DET, T>.  Each quad regroups its fp32 values so that every u64 reduction instruction of a warp covers
// 8 positions x 32 contiguous bytes: whole sectors.
template <int K, int CN, bool DET, typename T>
__global__ void __launch_bounds__(BT_THREADS, 2)
k_local_attn_bwd_tc(const T* __restrict__ src, const float* __restrict__ flow, const T* __restrict__ logits, const T* __restrict__ gout,
                    T* __restrict__ gsrc, float* __restrict__ gflow, T* __restrict__ glogits, float* __restrict__ gborder, int C, int Hs, int Ws, int H, int W, int gcols,
                    int grows, int accumulate, fx_t* __restrict__ gsum, const int* __restrict__ fx_exp) {
    constexpr int K1 = K + 1, KK = K * K;
    using L = BwdSmem<CN>;
    constexpr int GSTR = L::GSTR, NTW = CN / 32;
    extern __shared__ __align__(16) unsigned char smem[];
    int* irr = reinterpret_cast<int*>(smem + L::IRR);
    int& nirr = irr[128];
    unsigned char* rows = smem + L::ROWS;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, gid = lane >> 2, tig = lane & 3;
    const float inv_kk = 1.0f / static_cast<float>(KK);
    const uint32_t sb = smem_u32(smem);
    const uint32_t g_base = sb + L::G, s_base = sb + L::S, aw_base = sb + L::AW, p_base = sb + L::P;

    // every weight slab starts zeroed; from then on the grad_source warpgroup zeroes each slab after reading it
    for (int i = tid; i < BT_NAW * SEG * 16; i += BT_THREADS) sts128(aw_base + (i >> 4) * BT_AWSTR + (i & 15) * 16, 0u, 0u, 0u, 0u);
    if (tid == 0) nirr = 0;
    __syncthreads();
    // Each role derives its group and pointers after its setmaxnreg: values live across the register reallocation
    // are spilled.
    if (warp < 4) {
        // ======== pixel warpgroup: thread tid owns pixel tid; P GEMM, Q pick, grad_flow and grad_logits
        setmaxnreg_inc<BT_PIX_REGS>();
        uint32_t b;
        int gx0, gy0, bx0, by0, bx1, by1;
        group_decode(gcols, grows, b, gx0, gy0);
        group_bbox<K>(flow, b, gx0, gy0, H, W, Hs, Ws, lane, bx0, by0, bx1, by1);
        const long long hw = (long long)H * W;
        const T* go_b = gout + (long long)b * hw * C;
        // ---- per pixel: softmax, taps, window (folded, for grad_source) and the unfolded window origin (for Q)
        const int px = gx0 + (tid & 15), py = gy0 + (tid >> 4);
        const bool valid = px < W && py < H;
        const long long pofs = (long long)py * W + px;
        uint32_t w[K1 * K1 / 2];
        float Q[K1 * K1];
#pragma unroll
        for (int i = 0; i < K1 * K1; ++i) Q[i] = 0.f;
        int X0 = 0, Y0 = 0, X0u = 0, Y0u = 0;
        bool regular = false;
        if (valid) {
            float p[KK];
            pixel_softmax<T, float, KK>(logits + (long long)b * KK * hw + pofs, hw, KK, p);
            AxisTap<float> tx[K], ty[K];
            regular = taps_regular<float, K>(flow[(long long)b * 2 * hw + pofs], flow[(long long)b * 2 * hw + hw + pofs], px, py, Hs, Ws, tx, ty);
            if (regular) {
                X0u = tx[0].fl;
                Y0u = ty[0].fl;
                build_window<T, K>(p, tx, ty, Hs, Ws, inv_kk, w, X0, Y0);
            } else {
                irr[atomicAdd(&nirr, 1)] = tid;
            }
        }
        const T* s_b = src + (long long)b * Hs * Ws * C;
        // ldmatrix lane addresses
        const uint32_t g_frag_a = g_base + (warp * 32 + (lane & 15)) * GSTR + (lane >> 4) * 16;        // A = G rows
        const uint32_t s_frag_b = s_base + ((lane & 7) + ((lane >> 4) << 3)) * GSTR + ((lane >> 3) & 1) * 16;   // B = S rows

        for (int c0 = 0; c0 < C; c0 += CN) {
            if (c0 != 0) bar_sync(BT_BAR_PASS, BT_THREADS);       // the previous pass is done with G and the segments
            load_g_tile<T, CN>(g_base, go_b, c0, C, gx0, gy0, H, W, tid);
            {
                const int i = tid >> 3;
                for (int j = tid & 7; j < CN / 8; j += 8)
                    cp_async16(s_base + i * GSTR + j * 16, s_b + ((long long)by0 * Ws + min(bx0 + i, Ws - 1)) * C + c0 + j * 8);
            }
            cp_async_commit();
            cp_async_wait<1>();
            bar_sync(BT_BAR_PASS, BT_THREADS);                    // G complete
            // steps walk the footprint row-major: y from by0, x = bx0, bx0 + SEG, ... while x <= bx1
            int s = 0;
            for (int a = 0, y = by0, x = bx0; y <= by1; ++s) {
                const int buf = s & 1;                      // source segment
                const int an = a == BT_NAW - 1 ? 0 : a + 1;   // a = s % 3: weight slab and row bits
                int xn = x + SEG, yn = y;
                if (xn > bx1) { xn = bx0; ++yn; }
                // this pixel's column of Wfull^T for the segment, into the slab that step s - 3 read and zeroed
                if (s >= BT_NAW) bar_sync(BT_BAR_FREE + a, BT_THREADS);
                const bool act = regular && window_meets_step<K>(X0u, Y0u, Hs, Ws, y, x);
                if (act) scatter_window_row<K>(aw_base + a * (SEG * BT_AWSTR) + tid * 2, BT_AWSTR, w, X0, Y0, y, x);
                const uint32_t pm = warp_row_bits(act);     // this warp's two group rows
                if (lane == 0) rows[a * 4 + warp] = static_cast<unsigned char>(pm);
                bar_arrive(BT_BAR_FULL + a, BT_THREADS);    // slab s and its row bits written
                cp_async_wait_all();
                bar_sync(BT_BAR_PIX, 128);    // segment s complete; every pixel warp is past the P GEMM of step s - 1
                if (yn <= by1) {
                    const int i = tid >> 3;
                    const uint32_t dst = s_base + (buf ^ 1) * (SEG * GSTR) + i * GSTR;
                    const T* sp = s_b + ((long long)yn * Ws + min(xn + i, Ws - 1)) * C + c0;
                    for (int j = tid & 7; j < CN / 8; j += 8) cp_async16(dst + j * 16, sp + j * 8);
                    cp_async_commit();
                }
                if (pm != 0u) {
                    // P = G * S^T: this warp's 32 pixels x 16 positions, m-tiles of inactive pixel rows skipped
                    float pacc[2][2][4];
#pragma unroll
                    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                        for (int nt = 0; nt < 2; ++nt)
#pragma unroll
                            for (int q = 0; q < 4; ++q) pacc[mt][nt][q] = 0.f;
                    const uint32_t sf = s_frag_b + buf * (SEG * GSTR);
                    if (pm == 3u) p_gemm<T, CN, true, true>(g_frag_a, sf, pacc);
                    else if (pm == 1u) p_gemm<T, CN, true, false>(g_frag_a, sf, pacc);
                    else p_gemm<T, CN, false, true>(g_frag_a, sf, pacc);
#pragma unroll
                    for (int mt = 0; mt < 2; ++mt) {
                        if (((pm >> mt) & 1u) == 0u) continue;      // nobody reads the P rows of inactive pixels
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const uint32_t row = p_base + (warp * 32 + mt * 16 + gid + 8 * h) * (BT_PSTR * 4);
#pragma unroll
                            for (int nt = 0; nt < 2; ++nt) {
                                stsf(row + (nt * 8 + 2 * tig) * 4, pacc[mt][nt][2 * h]);
                                stsf(row + (nt * 8 + 2 * tig + 1) * 4, pacc[mt][nt][2 * h + 1]);
                            }
                        }
                    }
                    __syncwarp();         // this warp's P rows of step s complete: they are the only rows its pixels read
                    if (act) {
                        const uint32_t prow = p_base + tid * (BT_PSTR * 4);
#pragma unroll
                        for (int r = 0; r < K1; ++r) {
                            if (clampi(Y0u + r, Hs - 1) != y) continue;
#pragma unroll
                            for (int t = 0; t < K1; ++t) {
                                const int e = clampi(X0u + t, Ws - 1) - x;
                                if (e >= 0 && e < SEG) Q[r * K1 + t] += ldsf(prow + e * 4);
                            }
                        }
                    }
                }
                x = xn;
                y = yn;
                a = an;
            }
            // the slabs of the last steps are read and zeroed before the next pass scatters into them
            for (int j = max(s - BT_NAW, 0); j < s; ++j) bar_sync(BT_BAR_FREE + j % BT_NAW, BT_THREADS);
        }

        // ---- regular pixels: grad_logits and grad_flow from Q (local_attn_pixel.cuh)
        if (regular) {
            float p[KK], dp[KK];
            pixel_softmax<T, float, KK>(logits + (long long)b * KK * hw + pofs, hw, KK, p);
            AxisTap<float> tx[K], ty[K];
            taps_regular<float, K>(flow[(long long)b * 2 * hw + pofs], flow[(long long)b * 2 * hw + hw + pofs], px, py, Hs, Ws, tx, ty);
            float gfx = 0.f, gfy = 0.f;
#pragma unroll
            for (int i = 0; i < K; ++i)
#pragma unroll
                for (int j = 0; j < K; ++j)
                    dp[i * K + j] = tap_backward<float>(tx[j], ty[i], p[i * K + j] * inv_kk, inv_kk, Q[i * K1 + j], Q[i * K1 + j + 1],
                                                        Q[(i + 1) * K1 + j], Q[(i + 1) * K1 + j + 1], gfx, gfy);
            store_pixel_grads<T, float, float, KK>(p, dp, KK, gfx, gfy, glogits + (long long)b * KK * hw + pofs,
                                                   gflow + (long long)b * 2 * hw + pofs, hw, accumulate);
        }
        // ---- pixels with non-consecutive taps: literal arithmetic, one pixel warp per pixel.  The grad_source warps
        // do not take part: within their register budget this path would spill, and such pixels are rare.
        const double2 fsc = DET ? fx_scale(fx_exp[b]) : make_double2(0.0, 0.0);
        for (int i = warp; i < nirr; i += 4) {
            const int m = irr[i];
            irregular_pixel_bwd<T, K, DET>(src, flow, logits, gout, gsrc, gflow, glogits, b, C, Hs, Ws, H, W, gx0 + (m & 15),
                                        gy0 + (m >> 4), accumulate, lane, gsum, fsc);
        }
    } else {
        // ======== grad_source warpgroup: warp 4 + v owns channels [v CN/4, (v+1) CN/4) of the GS GEMM and its reductions
        setmaxnreg_dec<BT_GS_REGS>();
        uint32_t b;
        int gx0, gy0, bx0, by0, bx1, by1;
        group_decode(gcols, grows, b, gx0, gy0);
        group_bbox<K>(flow, b, gx0, gy0, H, W, Hs, Ws, lane, bx0, by0, bx1, by1);
        const long long hw = (long long)H * W;
        const T* go_b = gout + (long long)b * hw * C;
        const int v = warp - 4, t = tid - 128;
        const uint32_t aw_frag = aw_base + (lane & 15) * BT_AWSTR + (lane >> 4) * 16;                  // A = Wfull^T
        const uint32_t g_frag_b = g_base + (lane & 15) * GSTR + (v * (CN / 4) + (lane >> 4) * 8) * 2;  // B = G (transposed)
        T* gs_b = gsrc + (long long)b * Hs * Ws * C;
        fx_t* gx_b = nullptr;
        double2 fsc = make_double2(0.0, 0.0);
        if constexpr (DET) {
            gx_b = gsum + (long long)b * Hs * Ws * C;
            fsc = fx_scale(fx_exp[b]);
        }

        for (int c0 = 0; c0 < C; c0 += CN) {
            if (c0 != 0) bar_sync(BT_BAR_PASS, BT_THREADS);       // the previous pass is done with G
            load_g_tile<T, CN>(g_base, go_b, c0, C, gx0, gy0, H, W, tid);
            cp_async_wait_all();
            bar_sync(BT_BAR_PASS, BT_THREADS);                    // G complete
            for (int a = 0, y = by0, x = bx0; y <= by1;) {
                const int an = a == BT_NAW - 1 ? 0 : a + 1;
                int xn = x + SEG, yn = y;
                if (xn > bx1) { xn = bx0; ++yn; }
                bar_sync(BT_BAR_FULL + a, BT_THREADS);            // slab a and its row bits hold this step
                // group rows with an active pixel: bit 8 u + h = group row 2 u + h (the same word in every thread)
                const uint32_t grows_on = *reinterpret_cast<const uint32_t*>(rows + a * 4);
                if (grows_on == 0u) {
                    bar_arrive(BT_BAR_FREE + a, BT_THREADS);      // no pixel scattered: the slab is still zero
                } else {
                    // GS = Wfull^T * G: 16 positions x this warp's CN/4 channels; the k-steps of inactive pixel rows add zeros
                    float gacc[NTW][4];
#pragma unroll
                    for (int nt = 0; nt < NTW; ++nt)
#pragma unroll
                        for (int q = 0; q < 4; ++q) gacc[nt][q] = 0.f;
#pragma unroll
                    for (int kk = 0; kk < 128 / 16; ++kk) {
                        if (((grows_on >> (8 * (kk >> 1) + (kk & 1))) & 1u) == 0u) continue;
                        uint32_t af[4];
                        ldsm_x4(aw_frag + a * (SEG * BT_AWSTR) + kk * 32, af);
#pragma unroll
                        for (int np = 0; np < NTW / 2; ++np) {
                            uint32_t bg[4];
                            ldsm_x4_t(g_frag_b + kk * 16 * GSTR + np * 32, bg);
                            mma16<T>(gacc[2 * np], af, bg[0], bg[1]);
                            mma16<T>(gacc[2 * np + 1], af, bg[2], bg[3]);
                        }
                    }
                    bar_sync(BT_BAR_GS, 128);                     // every grad_source warp has read slab a
                    {
                        const uint32_t z = aw_base + a * (SEG * BT_AWSTR) + (t >> 3) * BT_AWSTR + (t & 7) * 32;
                        sts128(z, 0u, 0u, 0u, 0u);
                        sts128(z + 16, 0u, 0u, 0u, 0u);
                    }
                    bar_arrive(BT_BAR_FREE + a, BT_THREADS);
                    if constexpr (DET) {
                        // grad_source of the segment as fixed-point sums, no rounding of the partials and no border scratch.
                        // Lane t of a quad holds channels 2t, 2t+1 of each 8-channel group nt.  Per pair of groups (2j, 2j+1):
                        // the exchange with lane t^1 gives lane t the 4 consecutive channels 4 (t >> 1) .. +3 of group
                        // 2j + (t & 1); the quad transpose then gives lane t channel 4 (n >> 1) + t of group 2j + (n & 1) in
                        // word n, so the four lanes of a quad add one whole 32-byte sector per instruction.
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const int xp = x + gid + 8 * h;
                            fx_t* d = gx_b + ((long long)y * Ws + xp) * C + c0 + v * (CN / 4);
                            const bool t0 = (tig & 1) != 0;
#pragma unroll
                            for (int j = 0; j < NTW / 2; ++j) {
                                const float a0 = gacc[2 * j][2 * h], a1 = gacc[2 * j][2 * h + 1];
                                const float b0 = gacc[2 * j + 1][2 * h], b1 = gacc[2 * j + 1][2 * h + 1];
                                const float r0 = __shfl_xor_sync(0xffffffffu, t0 ? a0 : b0, 1);
                                const float r1 = __shfl_xor_sync(0xffffffffu, t0 ? a1 : b1, 1);
                                uint32_t u[4];
                                u[0] = __float_as_uint(t0 ? r0 : a0);
                                u[1] = __float_as_uint(t0 ? r1 : a1);
                                u[2] = __float_as_uint(t0 ? b0 : r0);
                                u[3] = __float_as_uint(t0 ? b1 : r1);
                                quad_transpose(u, tig);
                                if (xp <= bx1) {
#pragma unroll
                                    for (int n = 0; n < 4; ++n)
                                        fx_add(d + (2 * j + (n & 1)) * 8 + 4 * (n >> 1) + tig, __uint_as_float(u[n]), fsc);
                                }
                            }
                        }
                    } else {
                        // grad_source of the segment.  Positions past the footprint add nothing and border positions add fp32
                        // pairs to the scratch.  The others are rounded to T pairs, regrouped within each quad so that a
                        // lane holds 8 consecutive channels of one position, and added 16 bytes at a time: per warp
                        // instruction, 8 positions x 64 contiguous bytes, two full 32-byte sectors each.
                        uint32_t gv[2 * NTW];       // [h NTW + nt]: channels nt 8 + 2 tig, +1 of position x + gid + 8 h, as T pair
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const int xp = x + gid + 8 * h;
                            const int slot = xp > bx1 ? -2 : border_slot(y, xp, Hs, Ws);
                            if (slot >= 0) {
                                float* d = gborder + ((long long)b * 2 * (Hs + Ws) + slot) * C + c0 + v * (CN / 4) + 2 * tig;
#pragma unroll
                                for (int nt = 0; nt < NTW; ++nt) {
                                    const float v0 = gacc[nt][2 * h], v1 = gacc[nt][2 * h + 1];
                                    if (v0 != 0.f || v1 != 0.f) atomicAdd(reinterpret_cast<float2*>(d + nt * 8), make_float2(v0, v1));
                                }
                            }
#pragma unroll
                            for (int nt = 0; nt < NTW; ++nt) {
                                const typename Pair16<T>::type hv = floats2_rn<T>(gacc[nt][2 * h], gacc[nt][2 * h + 1]);
                                gv[h * NTW + nt] = slot == -1 ? *reinterpret_cast<const uint32_t*>(&hv) : 0u;
                            }
                        }
#pragma unroll
                        for (int j = 0; j < NTW / 2; ++j) {
                            uint32_t u[4] = {gv[4 * j], gv[4 * j + 1], gv[4 * j + 2], gv[4 * j + 3]};
                            quad_transpose(u, tig);
                            if ((u[0] | u[1] | u[2] | u[3]) != 0u) {        // all 8 values zero (or no position): nothing to add
                                const int n = 4 * j + tig, h = n / NTW, nt = n % NTW;
                                red_add_16x8(gs_b + ((long long)y * Ws + x + gid + 8 * h) * C + c0 + v * (CN / 4) + nt * 8, u);
                            }
                        }
                    }
                }
                x = xn;
                y = yn;
                a = an;
            }
        }
    }
}

// grad_source of the border positions: what the buffer holds (the caller's values, plus the irregular pixels' adds) plus
// the fp32 sum of the groups' adds, rounded once.  One thread per (image, border slot, channel pair).
template <typename T>
__global__ void __launch_bounds__(256)
k_fold_border(T* __restrict__ gsrc, const float* __restrict__ gborder, int B, int C, int Hs, int Ws) {
    const int nb = 2 * (Hs + Ws), c2 = C / 2;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)B * nb * c2) return;
    const long long bs = i / c2;
    const int c = (int)(i % c2) * 2, s = (int)(bs % nb), b = (int)(bs / nb);
    int y, x;
    if (s < Ws) { y = 0; x = s; }
    else if (s < 2 * Ws) { y = Hs - 1; x = s - Ws; }
    else if (s < 2 * Ws + Hs) { y = s - 2 * Ws; x = 0; }
    else { y = s - 2 * Ws - Hs; x = Ws - 1; }
    if (border_slot(y, x, Hs, Ws) != s) return;       // a slot no position maps to (a corner, or Hs or Ws of 1)
    const float2 v = *reinterpret_cast<const float2*>(gborder + bs * C + c);
    typename Pair16<T>::type* d = reinterpret_cast<typename Pair16<T>::type*>(gsrc + (((long long)b * Hs + y) * Ws + x) * C + c);
    const float2 o = pair_to_float2(*d);
    *d = floats2_rn<T>(o.x + v.x, o.y + v.y);
}

template <int K, int CN, bool DET, typename T>
static int launch_bwd(const void* src, const void* flow, const void* logits, const void* gout, void* gsrc, void* gflow, void* glogits,
                      float* gborder, int B, int C, int Hs, int Ws, int H, int W, int accumulate, cudaStream_t st_,
                      fx_t* gsum = nullptr, const int* fx_exp = nullptr) {
    const int gcols = (W + GW - 1) / GW, grows = (H + GH - 1) / GH;
    const long long ngroups = (long long)B * gcols * grows;
    if (ngroups > INT_MAX) return GFLA_E_SHAPE;
    auto kern = k_local_attn_bwd_tc<K, CN, DET, T>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, BwdSmem<CN>::ALLOC);
    if (e != cudaSuccess) return static_cast<int>(e);
    kern<<<(unsigned)ngroups, BT_THREADS, BwdSmem<CN>::ALLOC, st_>>>(
        (const T*)src, (const float*)flow, (const T*)logits, (const T*)gout, (T*)gsrc, (float*)gflow, (T*)glogits, gborder, C, Hs, Ws, H, W, gcols, grows, accumulate, gsum, fx_exp);
    const int st = launch_status();
    if (st != GFLA_OK || DET) return st;
    const long long n = (long long)B * 2 * (Hs + Ws) * (C / 2);
    k_fold_border<T><<<(unsigned)((n + 255) / 256), 256, 0, st_>>>((T*)gsrc, gborder, B, C, Hs, Ws);
    return launch_status();
}

}  // namespace tc

// Stream-ordered scratch from a pool the library owns, one per device, that keeps its memory between calls: the device's
// default pool hands its memory back at every synchronisation, and mapping it again each step costs more than the work.
static cudaError_t scratch_alloc(void** p, size_t bytes, cudaStream_t st_) {
    static std::mutex mu;
    static cudaMemPool_t pools[64] = {};
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (dev >= 64) return cudaMallocAsync(p, bytes, st_);
    {
        std::lock_guard<std::mutex> lock(mu);
        if (pools[dev] == nullptr) {
            cudaMemPoolProps props = {};
            props.allocType = cudaMemAllocationTypePinned;
            props.location.type = cudaMemLocationTypeDevice;
            props.location.id = dev;
            e = cudaMemPoolCreate(&pools[dev], &props);
            if (e != cudaSuccess) { pools[dev] = nullptr; return e; }
            uint64_t keep = UINT64_MAX;
            e = cudaMemPoolSetAttribute(pools[dev], cudaMemPoolAttrReleaseThreshold, &keep);
            if (e != cudaSuccess) return e;
        }
    }
    return cudaMallocFromPoolAsync(p, bytes, pools[dev], st_);
}

static int pick_cn_bwd(int C) {
    if (C % 256 == 0) return 256;
    if (C == 128 || C == 64) return C;
    return 0;
}

// the instance of k_local_attn_bwd_tc for (dtype, k, cn); GFLA_E_NOTSUP for a (k, cn) without one
template <bool DET, typename T>
static int dispatch_bwd_t(int k, int cn, const void* src, const void* flow, const void* logits, const void* gout, void* gsrc, void* gflow,
                          void* glogits, float* gborder, int B, int C, int Hs, int Ws, int H, int W, int accumulate, cudaStream_t st_,
                          fx_t* gsum, const int* fx_exp) {
#define GFLA_BT_CASE(K_, CN_) \
    if (k == K_ && cn == CN_) return tc::launch_bwd<K_, CN_, DET, T>(src, flow, logits, gout, gsrc, gflow, glogits, gborder, B, C, Hs, Ws, \
                                                                     H, W, accumulate, st_, gsum, fx_exp);
    GFLA_BT_CASE(5, 256) GFLA_BT_CASE(5, 128) GFLA_BT_CASE(5, 64)
    GFLA_BT_CASE(3, 256) GFLA_BT_CASE(3, 128) GFLA_BT_CASE(3, 64)
#undef GFLA_BT_CASE
    return GFLA_E_NOTSUP;
}

template <bool DET, typename... A>
static int dispatch_bwd(int k, int cn, int dtype, A... a) {
    if (dtype == GFLA_F16) return dispatch_bwd_t<DET, __half>(k, cn, a...);
    return dispatch_bwd_t<DET, __nv_bfloat16>(k, cn, a...);
}

bool local_attn_bwd_tc_supported(int C, int k, int dtype, int flow_dtype, int layout, const void* src, const void* gout,
                                 const void* gsrc) {
    return (dtype == GFLA_BF16 || dtype == GFLA_F16) && flow_dtype == GFLA_F32 && layout == GFLA_NHWC && (k == 3 || k == 5) && pick_cn_bwd(C) != 0 &&
           aligned(src, 16) && aligned(gout, 16) && aligned(gsrc, 16);
}

// accumulate = 0: grad_source is zero-filled here and all three gradients are overwritten; 1: everything is added into the
// caller's buffers
int local_attn_bwd_tc(const void* src, const void* flow, const void* logits, const void* gout, void* gsrc, void* gflow, void* glogits,
                      int B, int C, int Hs, int Ws, int H, int W, int k, int dtype, int accumulate, cudaStream_t st_) {
    if (!accumulate) {
        const int z = zero_async(gsrc, (size_t)B * C * Hs * Ws * 2, st_);
        if (z != GFLA_OK) return z;
    }
    const int cn = pick_cn_bwd(C);
    if (cn == 0 || (k != 3 && k != 5)) return GFLA_E_NOTSUP;
    // fp32 sums of the border positions' grad_source (border_slot), stream-ordered scratch
    const size_t border_bytes = (size_t)B * 2 * (Hs + Ws) * C * sizeof(float);
    float* gborder = nullptr;
    cudaError_t e = scratch_alloc(reinterpret_cast<void**>(&gborder), border_bytes, st_);
    if (e != cudaSuccess) return static_cast<int>(e);
    int r = zero_async(gborder, border_bytes, st_);
    if (r == GFLA_OK)
        r = dispatch_bwd<false>(k, cn, dtype, src, flow, logits, gout, gsrc, gflow, glogits, gborder, B, C, Hs, Ws, H, W, accumulate, st_,
                                nullptr, nullptr);
    e = cudaFreeAsync(gborder, st_);
    return r != GFLA_OK ? r : static_cast<int>(e);
}

// grad_source into the fixed-point sums gsum (zeroed, channels-last, exponents in fx_exp: det_accum.cuh); no border scratch
// and no k_fold_border.  grad_flow / grad_logits follow `accumulate` as above.
int local_attn_bwd_tc_det(const void* src, const void* flow, const void* logits, const void* gout, void* gflow, void* glogits, int B,
                          int C, int Hs, int Ws, int H, int W, int k, int dtype, int accumulate, fx_t* gsum, const int* fx_exp,
                          cudaStream_t st_) {
    return dispatch_bwd<true>(k, pick_cn_bwd(C), dtype, src, flow, logits, gout, nullptr, gflow, glogits, nullptr, B, C, Hs, Ws, H, W,
                              accumulate, st_, gsum, fx_exp);
}

}  // namespace gfla
