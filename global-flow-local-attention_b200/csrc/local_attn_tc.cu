// Fused local-attention forward on the tensor cores (bf16 data, fp32 flow, k in {3, 5}, NCHW or channels-last).
//
// Per 16x8 pixel group the weighted gather is a dense GEMM
//     out[128 px][C] = Wfull[128 px][footprint] * S[footprint][C]
// with K running over the source positions of the group's tap footprint, one row segment per step (32 positions = two MMA
// K-steps for channels-last, 16 for planar; FwdGeom):
//   * one thread per pixel: softmax, taps (exactly like block_extractor_kernel.cu:62-76), the collapsed (k+1)^2 window
//     (tile_window.cuh) kept in registers;
//   * per step every thread writes its pixel's row of the weight slab A[128 px][NPOS] (bf16; at most k+1 non-zeros),
//     the source segment B[NPOS][64 ch] arrives by cp.async through a ring FT_STAGES - 1 steps ahead, across channel
//     passes (channels-last), or by plain loads one step ahead (planar);
//   * warp w multiplies pixel rows 32w..32w+31 with mma.sync m16n8k16 (fp32 accumulators in registers), skipping per
//     K-step the 16-pixel m-tiles none of whose windows meets it (window_meets_step: their slab rows are all zero);
//   * pixels whose taps are not consecutive integers keep the literal 4-tap arithmetic (irregular_pixel, warp-cooperative).
#include "tile_window.cuh"

namespace gfla {
namespace tc {

constexpr int FT_THREADS = 128;                 // one thread per pixel of the group
constexpr int FT_CN = 64;                       // channels per pass (N of the MMAs)
constexpr int FT_BSTR = FT_CN * 2 + 16;         // source-segment row: 128 B + 16 B pad
constexpr int FT_STAGES = 4;                    // channels-last source-segment ring: FT_STAGES - 1 segments ahead (DESIGN 3.2)

// Source positions per step: channels-last walks the footprint in segments of two MMA K-steps (2 x SEG), which halves the
// steps, barriers and per-step bookkeeping; planar keeps SEG (its next segment is staged in registers).
template <bool NHWC>
struct FwdGeom {
    static constexpr int NPOS = NHWC ? 2 * SEG : SEG;
    static constexpr int HALVES = NPOS / SEG;               // MMA K-steps per step
    static constexpr int ASTR = NPOS * 2 + 16;              // weight-slab row: NPOS bf16 + 16 B pad (conflict-free ldmatrix)
    static constexpr int BSEG = NPOS * FT_BSTR;             // one source segment in shared memory
    static constexpr int NBUF = NHWC ? FT_STAGES : 2;       // source-segment buffers
};

template <bool NHWC>
struct FwdSmem {
    alignas(16) unsigned char a[2][128 * FwdGeom<NHWC>::ASTR];
    alignas(16) unsigned char b[FwdGeom<NHWC>::NBUF][FwdGeom<NHWC>::BSEG];
    int irr[128];
    int nirr;
};

// planar: source row segment (16 positions from x, clamped at the right edge: those columns carry zero weight) x 64
// channels, loaded into registers one step ahead and stored to shared memory after the step's MMAs
struct SegRegs {
    __nv_bfloat16 v[8];
};
__device__ __forceinline__ void seg_load(const __nv_bfloat16* __restrict__ src, int b, int C, int c0, int Hs, int Ws, int y, int x,
                                         int tid, SegRegs& r) {
#pragma unroll
    for (int it = 0; it < 8; ++it) {
        const int idx = it * FT_THREADS + tid, c = idx >> 4, i = idx & 15;
        const int xs = min(x + i, Ws - 1);
        r.v[it] = src[(((long long)b * C + c0 + c) * Hs + y) * Ws + xs];
    }
}
__device__ __forceinline__ void seg_store(uint32_t dst, int tid, const SegRegs& r) {
#pragma unroll
    for (int it = 0; it < 8; ++it) {
        const int idx = it * FT_THREADS + tid, c = idx >> 4, i = idx & 15;
        sts16(dst + i * FT_BSTR + c * 2, static_cast<uint32_t>(*reinterpret_cast<const unsigned short*>(&r.v[it])));
    }
}

// channels-last: the producer of the segment ring.  Copies the segment at (c0, y, x) (NPOS positions, clamped at the right
// edge like the planar segment) with cp.async, then moves (c0, y, x) on in the consumer's order: row-major over the
// footprint, then on into the next 64-channel pass.  Past the last pass it copies nothing, but it commits a group on every
// call, so that the consumer's wait count holds to the end.
template <int NPOS>
__device__ __forceinline__ void seg_produce(const __nv_bfloat16* __restrict__ src, int b, int C, int Hs, int Ws, int bx0, int by0,
                                            int bx1, int by1, int& c0, int& y, int& x, uint32_t dst, int tid) {
    if (c0 < C) {
        const int j = tid & 7;                            // 8-channel chunk
        const __nv_bfloat16* row = src + ((long long)b * Hs + y) * Ws * C + c0 + j * 8;
#pragma unroll
        for (int i = tid >> 3; i < NPOS; i += FT_THREADS / 8)   // position
            cp_async16(dst + i * FT_BSTR + j * 16, row + (long long)min(x + i, Ws - 1) * C);
        x += NPOS;
        if (x > bx1) {
            x = bx0;
            if (++y > by1) { y = by0; c0 += FT_CN; }
        }
    }
    cp_async_commit();
}

// Channels-last: at most 168 registers, so that three CTAs share an SM and hide each other's per-step barrier (cfg2 on an
// H100 80GB HBM3 at 400 W: 1.67 ms against 2.21 ms at two CTAs).  The planar kernel holds its next source segment in
// registers (SegRegs) and stays at two.
template <int K, bool NHWC>
__global__ void __launch_bounds__(FT_THREADS, NHWC ? 3 : 1)
k_local_attn_fwd_tc(const __nv_bfloat16* __restrict__ src, const float* __restrict__ flow, const __nv_bfloat16* __restrict__ logits,
                    __nv_bfloat16* __restrict__ out, __nv_bfloat16* __restrict__ probs, const __nv_bfloat16* __restrict__ prev,
                    const __nv_bfloat16* __restrict__ mask, int C, int Hs, int Ws, int H, int W, int gcols, int grows) {
    constexpr int K1 = K + 1, KK = K * K;
    using G = FwdGeom<NHWC>;
    __shared__ FwdSmem<NHWC> sm;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, gid = lane >> 2, tig = lane & 3;
    uint32_t b;
    int gx0, gy0;
    group_decode(gcols, grows, b, gx0, gy0);
    const long long hw = (long long)H * W;

    if (tid == 0) sm.nirr = 0;
    int bx0, by0, bx1, by1;
    group_bbox<K>(flow, b, gx0, gy0, H, W, Hs, Ws, lane, bx0, by0, bx1, by1);
    const uint32_t a_base = smem_u32(sm.a[0]), b_base = smem_u32(sm.b[0]);
    // channels-last: the producer (nc0, ny, nx) runs FT_STAGES - 1 segments ahead of the steps; the first ones load while
    // the pixels compute their windows
    int nc0 = 0, ny = by0, nx = bx0;
    if constexpr (NHWC) {
#pragma unroll
        for (int s = 0; s < FT_STAGES - 1; ++s)
            seg_produce<G::NPOS>(src, b, C, Hs, Ws, bx0, by0, bx1, by1, nc0, ny, nx, b_base + s * G::BSEG, tid);
    }
    __syncthreads();
    // ---- per pixel: softmax, taps, window
    const int px = gx0 + (tid & 15), py = gy0 + (tid >> 4);
    const bool valid = px < W && py < H;
    uint32_t w[K1 * K1 / 2];
    int X0 = 0, Y0 = 0;
    bool regular = false;
    if (valid) {
        const long long pofs = (long long)py * W + px;
        float p[KK];
        pixel_softmax<__nv_bfloat16, float, KK>(logits + (long long)b * KK * hw + pofs, hw, KK, p);
        if (probs != nullptr) {
#pragma unroll
            for (int t = 0; t < KK; ++t) probs[(long long)b * KK * hw + t * hw + pofs] = __float2bfloat16_rn(p[t]);
        }
        AxisTap<float> tx[K], ty[K];
        regular = taps_regular<float, K>(flow[(long long)b * 2 * hw + pofs], flow[(long long)b * 2 * hw + hw + pofs], px, py, Hs, Ws, tx, ty);
        if (regular) build_window<K>(p, tx, ty, Hs, Ws, 1.0f / static_cast<float>(KK), w, X0, Y0);
        else sm.irr[atomicAdd(&sm.nirr, 1)] = tid;
    }

    const uint32_t a_row = a_base + tid * G::ASTR;
    // ldmatrix lane addresses: A (rows = pixels of this warp, K = positions), B (rows = positions, N = channels, transposed)
    const uint32_t a_frag = a_base + (warp * 32 + (lane & 15)) * G::ASTR + (lane >> 4) * 16;
    const uint32_t b_frag = b_base + (lane & 15) * FT_BSTR + (lane >> 4) * 16;

    // Steps: channels-last numbers them t = 0, 1, ... across all passes (one flat stream), planar restarts at every pass.
    // The weight slab alternates its two buffers with t; the channels-last step t reads ring slot t % FT_STAGES.
    int t = 0, slot = 0;
    for (int c0 = 0; c0 < C; c0 += FT_CN) {
        float acc[2][8][4];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int nt = 0; nt < 8; ++nt)
#pragma unroll
                for (int q = 0; q < 4; ++q) acc[mt][nt][q] = 0.f;
        SegRegs pend;
        if constexpr (!NHWC) {
            __syncthreads();      // the previous pass's MMAs are done with both buffers
            t = 0;
            seg_load(src, b, C, c0, Hs, Ws, by0, bx0, tid, pend);
            seg_store(b_base, tid, pend);
        }
        // steps walk the footprint row-major: y from by0, x = bx0, bx0 + NPOS, ... while x <= bx1
        for (int y = by0, x = bx0; y <= by1; ++t) {
            const int buf = t & 1;
            int xn = x + G::NPOS, yn = y;
            if (xn > bx1) { xn = bx0; ++yn; }
            // this pixel's row of the weight slab: zeros except window row y - Y0
            const uint32_t row = a_row + buf * (128 * G::ASTR);
#pragma unroll
            for (int q = 0; q < G::NPOS * 2; q += 16) sts128(row + q, 0u, 0u, 0u, 0u);
            // per MMA K-step (SEG positions): the m-tiles (16 pixels each) of this warp with an active pixel; the others'
            // slab rows are all zero there
            uint32_t wm[G::HALVES];
            bool act = false;
#pragma unroll
            for (int hk = 0; hk < G::HALVES; ++hk) {
                const bool a = regular && window_meets_step<K>(X0, Y0, Hs, Ws, y, x + hk * SEG);
                wm[hk] = warp_row_bits(a);
                act |= a;
            }
            if (act) scatter_window_row<K, G::NPOS>(row, 2, w, X0, Y0, y, x);
            uint32_t bseg;
            if constexpr (NHWC) {
                cp_async_wait<FT_STAGES - 2>();   // this thread's part of step t's segment has landed
                __syncthreads();      // slab and segment of step t complete; everybody is past step t-1's MMAs
                // so step t-1's slot is free: it takes the segment of step t + FT_STAGES - 1
                const int free_slot = slot == 0 ? FT_STAGES - 1 : slot - 1;
                seg_produce<G::NPOS>(src, b, C, Hs, Ws, bx0, by0, bx1, by1, nc0, ny, nx, b_base + free_slot * G::BSEG, tid);
                bseg = slot * G::BSEG;
                slot = slot == FT_STAGES - 1 ? 0 : slot + 1;
            } else {
                __syncthreads();      // slab and segment of step t complete; everybody is past step t-1's MMAs
                if (yn <= by1) seg_load(src, b, C, c0, Hs, Ws, yn, xn, tid, pend);
                bseg = buf * G::BSEG;
            }
            // K-steps in position order: every accumulator receives the same MMAs in the same order as with SEG-wide steps
#pragma unroll
            for (int hk = 0; hk < G::HALVES; ++hk) {
                if (wm[hk] == 0u) continue;
                const uint32_t a_k = a_frag + buf * (128 * G::ASTR) + hk * (SEG * 2);
                uint32_t af[2][4];
                if (wm[hk] & 1u) ldsm_x4(a_k, af[0]);
                if (wm[hk] & 2u) ldsm_x4(a_k + 16 * G::ASTR, af[1]);
#pragma unroll
                for (int np = 0; np < 4; ++np) {
                    uint32_t bf[4];
                    ldsm_x4_t(b_frag + bseg + hk * (SEG * FT_BSTR) + np * 32, bf);
#pragma unroll
                    for (int mt = 0; mt < 2; ++mt) {
                        if (((wm[hk] >> mt) & 1u) == 0u) continue;
                        mma_bf16(acc[mt][2 * np], af[mt], bf[0], bf[1]);
                        mma_bf16(acc[mt][2 * np + 1], af[mt], bf[2], bf[3]);
                    }
                }
            }
            if (!NHWC && yn <= by1) seg_store(b_base + (buf ^ 1) * G::BSEG, tid, pend);
            x = xn;
            y = yn;
        }
        // ---- epilogue: rows = pixels, columns = channels c0 + 8 nt + 2 tig (+1); channels-last keeps loading meanwhile
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = warp * 32 + mt * 16 + gid + 8 * h;
                const int qx = gx0 + (m & 15), qy = gy0 + (m >> 4);
                if (qx >= W || qy >= H) continue;
                const long long qofs = (long long)qy * W + qx;
                bool irr = false;
                for (int i = 0; i < sm.nirr; ++i) irr |= sm.irr[i] == m;
                if (irr) continue;
                const float qm = prev != nullptr ? __bfloat162float(mask[(long long)b * hw + qofs]) : 1.f;
#pragma unroll
                for (int nt = 0; nt < 8; ++nt) {
                    const int c = c0 + nt * 8 + 2 * tig;
                    float v0 = acc[mt][nt][2 * h], v1 = acc[mt][nt][2 * h + 1];
                    const long long o0 = NHWC ? ((long long)b * hw + qofs) * C + c : ((long long)b * C + c) * hw + qofs;
                    const long long o1 = NHWC ? o0 + 1 : o0 + hw;
                    if (prev != nullptr) {
                        v0 = __bfloat162float(prev[o0]) * (1.f - qm) + v0 * qm;
                        v1 = __bfloat162float(prev[o1]) * (1.f - qm) + v1 * qm;
                    }
                    if (NHWC) {
                        *reinterpret_cast<__nv_bfloat162*>(out + o0) = __floats2bfloat162_rn(v0, v1);
                    } else {
                        out[o0] = __float2bfloat16_rn(v0);
                        out[o1] = __float2bfloat16_rn(v1);
                    }
                }
            }
    }
    // ---- pixels with non-consecutive taps: the reference's literal arithmetic, one warp per pixel, all channels
    for (int i = warp; i < sm.nirr; i += FT_THREADS / 32) {
        const int m = sm.irr[i], qx = gx0 + (m & 15), qy = gy0 + (m >> 4);
        const long long qofs = (long long)qy * W + qx;
        irregular_pixel<K, NHWC>(src, logits, out, prev, mask, b, C, Hs, Ws, H, W, qx, qy, flow[(long long)b * 2 * hw + qofs],
                                 flow[(long long)b * 2 * hw + hw + qofs], lane);
    }
}

template <int K, bool NHWC>
static int launch_fwd(const void* src, const void* flow, const void* logits, void* out, void* probs, const void* prev, const void* mask,
                      int B, int C, int Hs, int Ws, int H, int W, cudaStream_t st_) {
    const int gcols = (W + GW - 1) / GW, grows = (H + GH - 1) / GH;
    const long long ngroups = (long long)B * gcols * grows;
    if (ngroups > INT_MAX) return GFLA_E_SHAPE;
    k_local_attn_fwd_tc<K, NHWC><<<(unsigned)ngroups, FT_THREADS, 0, st_>>>(
        (const __nv_bfloat16*)src, (const float*)flow, (const __nv_bfloat16*)logits, (__nv_bfloat16*)out, (__nv_bfloat16*)probs,
        (const __nv_bfloat16*)prev, (const __nv_bfloat16*)mask, C, Hs, Ws, H, W, gcols, grows);
    return launch_status();
}

}  // namespace tc

bool local_attn_fwd_tc_supported(int C, int Ws, int k, int dtype, int flow_dtype, int layout, const void* src, const void* out) {
    const bool c_ok = C % 256 == 0 || C == 128 || C == 64;
    if (!(dtype == GFLA_BF16 && flow_dtype == GFLA_F32 && (k == 3 || k == 5) && c_ok && aligned(src, 16))) return false;
    // channels-last: 16-byte cp.async of the source and 4-byte channel-pair stores need aligned pointers
    return layout == GFLA_NHWC ? aligned(out, 16) : (Ws % 8) == 0;
}

int local_attn_fwd_tc(const void* src, const void* flow, const void* logits, void* out, void* probs, const void* prev,
                      const void* mask, int B, int C, int Hs, int Ws, int H, int W, int k, int dtype, int flow_dtype,
                      int layout, cudaStream_t st_) {
    if (!local_attn_fwd_tc_supported(C, Ws, k, dtype, flow_dtype, layout, src, out)) return GFLA_E_NOTSUP;
    const bool nhwc = layout == GFLA_NHWC;
    if (k == 5) return nhwc ? tc::launch_fwd<5, true>(src, flow, logits, out, probs, prev, mask, B, C, Hs, Ws, H, W, st_)
                            : tc::launch_fwd<5, false>(src, flow, logits, out, probs, prev, mask, B, C, Hs, Ws, H, W, st_);
    return nhwc ? tc::launch_fwd<3, true>(src, flow, logits, out, probs, prev, mask, B, C, Hs, Ws, H, W, st_)
                : tc::launch_fwd<3, false>(src, flow, logits, out, probs, prev, mask, B, C, Hs, Ws, H, W, st_);
}

}  // namespace gfla
