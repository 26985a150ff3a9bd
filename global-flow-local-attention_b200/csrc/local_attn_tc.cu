// Fused local-attention forward on the tensor cores (bf16 or fp16 data, fp32 flow, k in {3, 5}, NCHW or channels-last).
// T, the data's 16-bit type, is also the type of the weight slab, so both MMA operands are T; the accumulators are fp32.
//
// Per 16x8 pixel group the weighted gather is a dense GEMM
//     out[128 px][C] = Wfull[128 px][footprint] * S[footprint][C]
// with K running over the source positions of the group's tap footprint, one row segment per step (32 positions = two MMA
// K-steps for channels-last, 16 for planar):
//   * one thread per pixel: softmax, taps (exactly like block_extractor_kernel.cu:62-76), the collapsed (k+1)^2 window
//     (tile_window.cuh) kept in registers;
//   * per step every pixel thread writes its pixel's row of the weight slab A[128 px][NPOS] (T; at most k+1 non-zeros);
//     the source segment B[NPOS][CN ch] is staged ahead;
//   * the warp that owns pixel rows 32w..32w+31 multiplies them with mma.sync m16n8k16 (fp32 accumulators in registers),
//     skipping per K-step the 16-pixel m-tiles none of whose windows meets it (window_meets_step: their slab rows are all
//     zero);
//   * pixels whose taps are not consecutive integers keep the literal 4-tap arithmetic (irregular_pixel, warp-cooperative).
// Planar (k_local_attn_fwd_tc): 128 threads do everything, 16-position steps, 64-channel passes, the next segment staged
// in registers one step ahead.  Channels-last (k_local_attn_fwd_tc_cl): a pixel warpgroup writes the slabs and an MMA
// warpgroup loads the segments and multiplies, 32-position steps, CN-channel passes (DESIGN 3.2).  Both give every
// accumulator the same MMAs in the same order, so out, probs and the blend are bit-identical between the layouts.
#include "tile_window.cuh"

namespace gfla {
namespace tc {

// ------------------------------------------------------------------ planar
constexpr int FT_THREADS = 128;                 // one thread per pixel of the group
constexpr int FT_CN = 64;                       // channels per pass (N of the MMAs)
constexpr int FT_BSTR = FT_CN * 2 + 16;         // source-segment row: 128 B + 16 B pad
constexpr int FT_ASTR = SEG * 2 + 16;           // weight-slab row: SEG 16-bit weights + 16 B pad (conflict-free ldmatrix)
constexpr int FT_BSEG = SEG * FT_BSTR;          // one source segment in shared memory

struct FwdSmem {
    alignas(16) unsigned char a[2][128 * FT_ASTR];
    alignas(16) unsigned char b[2][FT_BSEG];
    int irr[128];
    int nirr;
};

// source row segment (16 positions from x, clamped at the right edge: those columns carry zero weight) x 64 channels,
// loaded into registers one step ahead and stored to shared memory after the step's MMAs
template <typename T>
struct SegRegs {
    T v[8];
};
template <typename T>
__device__ __forceinline__ void seg_load(const T* __restrict__ src, int b, int C, int c0, int Hs, int Ws, int y, int x, int tid,
                                         SegRegs<T>& r) {
#pragma unroll
    for (int it = 0; it < 8; ++it) {
        const int idx = it * FT_THREADS + tid, c = idx >> 4, i = idx & 15;
        const int xs = min(x + i, Ws - 1);
        r.v[it] = src[(((long long)b * C + c0 + c) * Hs + y) * Ws + xs];
    }
}
template <typename T>
__device__ __forceinline__ void seg_store(uint32_t dst, int tid, const SegRegs<T>& r) {
#pragma unroll
    for (int it = 0; it < 8; ++it) {
        const int idx = it * FT_THREADS + tid, c = idx >> 4, i = idx & 15;
        sts16(dst + i * FT_BSTR + c * 2, static_cast<uint32_t>(*reinterpret_cast<const unsigned short*>(&r.v[it])));
    }
}

template <int K, typename T>
__global__ void __launch_bounds__(FT_THREADS, 1)
k_local_attn_fwd_tc(const T* __restrict__ src, const float* __restrict__ flow, const T* __restrict__ logits, T* __restrict__ out,
                    T* __restrict__ probs, const T* __restrict__ prev, const T* __restrict__ mask, int C, int Hs, int Ws, int H, int W,
                    int gcols, int grows) {
    constexpr int K1 = K + 1, KK = K * K;
    __shared__ FwdSmem sm;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, gid = lane >> 2, tig = lane & 3;
    uint32_t b;
    int gx0, gy0;
    group_decode(gcols, grows, b, gx0, gy0);
    const long long hw = (long long)H * W;

    if (tid == 0) sm.nirr = 0;
    int bx0, by0, bx1, by1;
    group_bbox<K>(flow, b, gx0, gy0, H, W, Hs, Ws, lane, bx0, by0, bx1, by1);
    const uint32_t a_base = smem_u32(sm.a[0]), b_base = smem_u32(sm.b[0]);
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
        pixel_softmax<T, float, KK>(logits + (long long)b * KK * hw + pofs, hw, KK, p);
        if (probs != nullptr) {
#pragma unroll
            for (int t = 0; t < KK; ++t) st(probs + (long long)b * KK * hw + t * hw + pofs, p[t]);
        }
        AxisTap<float> tx[K], ty[K];
        regular = taps_regular<float, K>(flow[(long long)b * 2 * hw + pofs], flow[(long long)b * 2 * hw + hw + pofs], px, py, Hs, Ws, tx, ty);
        if (regular) build_window<T, K>(p, tx, ty, Hs, Ws, 1.0f / static_cast<float>(KK), w, X0, Y0);
        else sm.irr[atomicAdd(&sm.nirr, 1)] = tid;
    }

    const uint32_t a_row = a_base + tid * FT_ASTR;
    // ldmatrix lane addresses: A (rows = pixels of this warp, K = positions), B (rows = positions, N = channels, transposed)
    const uint32_t a_frag = a_base + (warp * 32 + (lane & 15)) * FT_ASTR + (lane >> 4) * 16;
    const uint32_t b_frag = b_base + (lane & 15) * FT_BSTR + (lane >> 4) * 16;

    for (int c0 = 0; c0 < C; c0 += FT_CN) {
        float acc[2][8][4];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int nt = 0; nt < 8; ++nt)
#pragma unroll
                for (int q = 0; q < 4; ++q) acc[mt][nt][q] = 0.f;
        SegRegs<T> pend;
        __syncthreads();      // the previous pass's MMAs are done with both buffers
        seg_load(src, b, C, c0, Hs, Ws, by0, bx0, tid, pend);
        seg_store(b_base, tid, pend);
        // steps walk the footprint row-major: y from by0, x = bx0, bx0 + SEG, ... while x <= bx1; the weight slab and
        // the segment alternate their two buffers
        for (int t = 0, y = by0, x = bx0; y <= by1; ++t) {
            const int buf = t & 1;
            int xn = x + SEG, yn = y;
            if (xn > bx1) { xn = bx0; ++yn; }
            // this pixel's row of the weight slab: zeros except window row y - Y0
            const uint32_t row = a_row + buf * (128 * FT_ASTR);
#pragma unroll
            for (int q = 0; q < SEG * 2; q += 16) sts128(row + q, 0u, 0u, 0u, 0u);
            // the m-tiles (16 pixels each) of this warp with an active pixel; the others' slab rows are all zero
            const bool act = regular && window_meets_step<K>(X0, Y0, Hs, Ws, y, x);
            const uint32_t wm = warp_row_bits(act);
            if (act) scatter_window_row<K>(row, 2, w, X0, Y0, y, x);
            __syncthreads();      // slab and segment of step t complete; everybody is past step t-1's MMAs
            if (yn <= by1) seg_load(src, b, C, c0, Hs, Ws, yn, xn, tid, pend);
            const uint32_t bseg = buf * FT_BSEG;
            if (wm != 0u) {
                const uint32_t a_k = a_frag + buf * (128 * FT_ASTR);
                uint32_t af[2][4];
                if (wm & 1u) ldsm_x4(a_k, af[0]);
                if (wm & 2u) ldsm_x4(a_k + 16 * FT_ASTR, af[1]);
#pragma unroll
                for (int np = 0; np < 4; ++np) {
                    uint32_t bf[4];
                    ldsm_x4_t(b_frag + bseg + np * 32, bf);
#pragma unroll
                    for (int mt = 0; mt < 2; ++mt) {
                        if (((wm >> mt) & 1u) == 0u) continue;
                        mma16<T>(acc[mt][2 * np], af[mt], bf[0], bf[1]);
                        mma16<T>(acc[mt][2 * np + 1], af[mt], bf[2], bf[3]);
                    }
                }
            }
            if (yn <= by1) seg_store(b_base + (buf ^ 1) * FT_BSEG, tid, pend);
            x = xn;
            y = yn;
        }
        // ---- epilogue: rows = pixels, columns = channels c0 + 8 nt + 2 tig (+1)
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
                const float qm = prev != nullptr ? ld(mask + (long long)b * hw + qofs) : 1.f;
#pragma unroll
                for (int nt = 0; nt < 8; ++nt) {
                    const int c = c0 + nt * 8 + 2 * tig;
                    float v0 = acc[mt][nt][2 * h], v1 = acc[mt][nt][2 * h + 1];
                    const long long o0 = ((long long)b * C + c) * hw + qofs, o1 = o0 + hw;
                    if (prev != nullptr) {
                        v0 = ld(prev + o0) * (1.f - qm) + v0 * qm;
                        v1 = ld(prev + o1) * (1.f - qm) + v1 * qm;
                    }
                    st(out + o0, v0);
                    st(out + o1, v1);
                }
            }
    }
    // ---- pixels with non-consecutive taps: the reference's literal arithmetic, one warp per pixel, all channels
    for (int i = warp; i < sm.nirr; i += FT_THREADS / 32) {
        const int m = sm.irr[i], qx = gx0 + (m & 15), qy = gy0 + (m >> 4);
        const long long qofs = (long long)qy * W + qx;
        irregular_pixel<T, K, false>(src, logits, out, prev, mask, b, C, Hs, Ws, H, W, qx, qy, flow[(long long)b * 2 * hw + qofs],
                                  flow[(long long)b * 2 * hw + hw + qofs], lane);
    }
}

// ------------------------------------------------------------------ channels-last
constexpr int FC_THREADS = 256;                 // pixel warpgroup (warps 0-3) + MMA warpgroup (warps 4-7)
constexpr int FC_NPOS = 2 * SEG;                // source positions per step: two MMA K-steps
constexpr int FC_ASTR = FC_NPOS * 2 + 16;       // weight-slab row: 32 16-bit weights + 16 B pad (conflict-free ldmatrix)
constexpr int FC_NA = 3;                        // weight slabs (and row-bit words) in rotation
constexpr int FC_AHEAD = 3;                     // source segments in flight ahead of the step that writes its slab
constexpr int FC_NSEG = FC_AHEAD + FC_NA;       // ring slots: step s's slot is refilled once FREE of step s shows it read
// per-thread registers of the two roles after setmaxnreg: they sum to 256, the 128 per thread that 2 CTAs per SM leave
constexpr int FC_PIX_REGS = 72, FC_MMA_REGS = 184;
// named barriers (0 is __syncthreads)
constexpr int FC_BAR_FULL = 1;                  // + slab: slab, row bits and source segment complete (pixel arrives, MMA syncs)
constexpr int FC_BAR_FREE = 4;                  // + slab: slab and segment read, slab zeroed (MMA arrives, pixel syncs)

template <int CN>
struct FwdClSmem {
    static constexpr int BSTR = CN * 2 + 16;             // source-segment row: CN 16-bit values + 16 B pad
    static constexpr int BSEG = FC_NPOS * BSTR;          // one ring slot
    static constexpr int A = 0;
    static constexpr int B = A + FC_NA * 128 * FC_ASTR;
    static constexpr int IRR = B + FC_NSEG * BSEG;
    static constexpr int ROWS = IRR + 129 * 4;           // per slab: byte w = row bits of pixel warp w (bit 2 hk + mt)
    static constexpr int ALLOC = ROWS + FC_NA * 4;
};

// The producer of the segment ring (thread t of the pixel warpgroup).  Copies the segment at (c0, y, x) (FC_NPOS
// positions, clamped at the right edge like the planar segment) with cp.async and moves the cursor on in the steps'
// order: row-major over the footprint, then on into the next CN-channel pass.  Past the last pass it copies nothing, but
// it commits a group on every call, so that the wait count before each FULL holds to the end.
template <typename T, int CN>
__device__ __forceinline__ void seg_produce(const T* __restrict__ src, int b, int C, int Hs, int Ws, int bx0, int by0,
                                            int bx1, int by1, int& c0, int& y, int& x, uint32_t dst, int t) {
    constexpr int CH = CN / 8;                            // 16-byte chunks per position
    if (c0 < C) {
        const int j = t % CH;
        const T* row = src + ((long long)b * Hs + y) * Ws * C + c0 + j * 8;
#pragma unroll
        for (int i = t / CH; i < FC_NPOS; i += 128 / CH)   // position
            cp_async16(dst + i * FwdClSmem<CN>::BSTR + j * 16, row + (long long)min(x + i, Ws - 1) * C);
        x += FC_NPOS;
        if (x > bx1) {
            x = bx0;
            if (++y > by1) { y = by0; c0 += CN; }
        }
    }
    cp_async_commit();
}

// Two warpgroups per CTA, 2 CTAs per SM:
//   * pixel warpgroup, warps 0-3: thread tid owns pixel tid.  Softmax, probs, taps and window, the source-segment ring
//     (FC_AHEAD segments ahead), and per step the slab row and the warp's row bits into slab s % 3, signalled by FULL
//     once the step's segment has landed too;
//   * MMA warpgroup, warps 4-7: the MMAs (warp 4 + v owns pixel rows 32v..32v+31, so it alone reads, and then zeroes,
//     the slab rows pixel warp v wrote), signalled by FREE; the epilogue and the irregular pixels.
// The pixel warpgroup waits for FREE of step s - 3 before it writes slab s, so it runs up to two steps ahead, also across
// passes.  Steps are numbered across all passes; every slab is zero at the start of each step.
template <int K, int CN, typename T>
__global__ void __launch_bounds__(FC_THREADS, 2)
k_local_attn_fwd_tc_cl(const T* __restrict__ src, const float* __restrict__ flow, const T* __restrict__ logits, T* __restrict__ out,
                       T* __restrict__ probs, const T* __restrict__ prev, const T* __restrict__ mask, int C, int Hs, int Ws, int H,
                       int W, int gcols, int grows) {
    constexpr int K1 = K + 1, KK = K * K;
    using L = FwdClSmem<CN>;
    extern __shared__ __align__(16) unsigned char smem[];
    int* irr = reinterpret_cast<int*>(smem + L::IRR);
    int& nirr = irr[128];
    unsigned char* rows = smem + L::ROWS;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t sb = smem_u32(smem), a_base = sb + L::A, b_base = sb + L::B;

    for (int i = tid; i < FC_NA * 128 * FC_ASTR / 16; i += FC_THREADS) sts128(a_base + i * 16, 0u, 0u, 0u, 0u);
    if (tid == 0) nirr = 0;
    __syncthreads();
    if (warp < 4) {
        // ======== pixel warpgroup: thread tid owns pixel tid
        uint32_t b;
        int gx0, gy0, bx0, by0, bx1, by1;
        group_decode(gcols, grows, b, gx0, gy0);
        group_bbox<K>(flow, b, gx0, gy0, H, W, Hs, Ws, lane, bx0, by0, bx1, by1);
        // The ring's first segments load while the windows are computed.  The pixel warps own the ring: the MMA warps
        // then only wait for FULL, multiply and signal FREE.
        int nc0 = 0, ny = by0, nx = bx0;   // the ring's cursor: FC_AHEAD segments ahead of the steps
#pragma unroll
        for (int i = 0; i < FC_AHEAD; ++i)
            seg_produce<T, CN>(src, b, C, Hs, Ws, bx0, by0, bx1, by1, nc0, ny, nx, b_base + i * L::BSEG, tid);
        const long long hw = (long long)H * W;
        const int px = gx0 + (tid & 15), py = gy0 + (tid >> 4);
        uint32_t w[K1 * K1 / 2];
        int X0 = 0, Y0 = 0;
        bool regular = false;
        if (px < W && py < H) {
            const long long pofs = (long long)py * W + px;
            float p[KK];
            pixel_softmax<T, float, KK>(logits + (long long)b * KK * hw + pofs, hw, KK, p);
            if (probs != nullptr) {
#pragma unroll
                for (int t = 0; t < KK; ++t) st(probs + (long long)b * KK * hw + t * hw + pofs, p[t]);
            }
            AxisTap<float> tx[K], ty[K];
            regular = taps_regular<float, K>(flow[(long long)b * 2 * hw + pofs], flow[(long long)b * 2 * hw + hw + pofs], px, py, Hs, Ws, tx, ty);
            if (regular) build_window<T, K>(p, tx, ty, Hs, Ws, 1.0f / static_cast<float>(KK), w, X0, Y0);
            else irr[atomicAdd(&nirr, 1)] = tid;
        }
        // the window is built: the steady state needs only the window, its origin and the walk
        setmaxnreg_dec<FC_PIX_REGS>();
        const uint32_t a_row = a_base + tid * FC_ASTR;
        int s = 0, slot = FC_AHEAD;      // slot: where the segment of step s + FC_AHEAD goes
        for (int c0 = 0; c0 < C; c0 += CN) {
            for (int a = s % FC_NA, y = by0, x = bx0; y <= by1; ++s) {
                // slab a and the segment of step s - 3 are read, the slab is zeroed
                if (s >= FC_NA) bar_sync(FC_BAR_FREE + a, FC_THREADS);
                // so step s - 3's slot, (s + FC_AHEAD) % FC_NSEG, takes the segment of step s + FC_AHEAD
                seg_produce<T, CN>(src, b, C, Hs, Ws, bx0, by0, bx1, by1, nc0, ny, nx, b_base + slot * L::BSEG, tid);
                slot = slot == FC_NSEG - 1 ? 0 : slot + 1;
                // per MMA K-step (SEG positions): the m-tiles of this warp with an active pixel
                uint32_t bits = 0u;
                bool act = false;
#pragma unroll
                for (int hk = 0; hk < 2; ++hk) {
                    const bool on = regular && window_meets_step<K>(X0, Y0, Hs, Ws, y, x + hk * SEG);
                    bits |= warp_row_bits(on) << (2 * hk);
                    act |= on;
                }
                if (act) scatter_window_row<K, FC_NPOS>(a_row + a * (128 * FC_ASTR), 2, w, X0, Y0, y, x);
                if (lane == 0) rows[a * 4 + warp] = static_cast<unsigned char>(bits);
                // this thread's part of step s's segment has landed: one group per step since, FC_AHEAD still in flight
                cp_async_wait<FC_AHEAD>();
                bar_arrive(FC_BAR_FULL + a, FC_THREADS);                   // slab s, row bits and segment s complete
                x += FC_NPOS;
                if (x > bx1) { x = bx0; ++y; }
                a = a == FC_NA - 1 ? 0 : a + 1;
            }
        }
        // consume the FREE signals of the last steps, so that no barrier is left half-arrived
        for (int j = max(s - FC_NA, 0); j < s; ++j) bar_sync(FC_BAR_FREE + j % FC_NA, FC_THREADS);
    } else {
        // ======== MMA warpgroup: warp 4 + v owns pixel rows 32v..32v+31
        setmaxnreg_inc<FC_MMA_REGS>();
        const int v = warp - 4, gid = lane >> 2, tig = lane & 3;
        uint32_t b;
        int gx0, gy0, bx0, by0, bx1, by1;
        group_decode(gcols, grows, b, gx0, gy0);
        group_bbox<K>(flow, b, gx0, gy0, H, W, Hs, Ws, lane, bx0, by0, bx1, by1);
        const long long hw = (long long)H * W;
        // ldmatrix lane addresses: A (rows = pixels of this warp, K = positions), B (rows = positions, N = channels, transposed)
        const uint32_t a_frag = a_base + (v * 32 + (lane & 15)) * FC_ASTR + (lane >> 4) * 16;
        const uint32_t b_frag = b_base + (lane & 15) * L::BSTR + (lane >> 4) * 16;
        // the slab row this lane zeroes after the MMAs, and its m-tile
        const uint32_t z_row = a_base + (v * 32 + lane) * FC_ASTR;
        const int z_mt = lane >> 4;
        int slot = 0;
        for (int c0 = 0, a = 0; c0 < C; c0 += CN) {
            float acc[2][CN / 8][4];
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                for (int nt = 0; nt < CN / 8; ++nt)
#pragma unroll
                    for (int q = 0; q < 4; ++q) acc[mt][nt][q] = 0.f;
            for (int y = by0, x = bx0; y <= by1;) {
                const uint32_t bseg = slot * L::BSEG;
                slot = slot == FC_NSEG - 1 ? 0 : slot + 1;
                bar_sync(FC_BAR_FULL + a, FC_THREADS);           // slab a, its row bits and the step's segment hold this step
                const uint32_t bits = rows[a * 4 + v];
                if (bits != 0u) {
                    // K-steps in position order: every accumulator receives the same MMAs in the same order as with
                    // SEG-wide steps
#pragma unroll
                    for (int hk = 0; hk < 2; ++hk) {
                        const uint32_t wm = (bits >> (2 * hk)) & 3u;
                        if (wm == 0u) continue;
                        const uint32_t a_k = a_frag + a * (128 * FC_ASTR) + hk * (SEG * 2);
                        uint32_t af[2][4];
                        if (wm & 1u) ldsm_x4(a_k, af[0]);
                        if (wm & 2u) ldsm_x4(a_k + 16 * FC_ASTR, af[1]);
                        // B fragments one n-pair ahead of the MMAs, so that no MMA waits for its ldmatrix
                        const uint32_t b_k = b_frag + bseg + hk * (SEG * L::BSTR);
                        uint32_t bf[2][4];
                        ldsm_x4_t(b_k, bf[0]);
#pragma unroll
                        for (int np = 0; np < CN / 16; ++np) {
                            if (np + 1 < CN / 16) ldsm_x4_t(b_k + (np + 1) * 32, bf[(np + 1) & 1]);
#pragma unroll
                            for (int mt = 0; mt < 2; ++mt) {
                                if (((wm >> mt) & 1u) == 0u) continue;
                                mma16<T>(acc[mt][2 * np], af[mt], bf[np & 1][0], bf[np & 1][1]);
                                mma16<T>(acc[mt][2 * np + 1], af[mt], bf[np & 1][2], bf[np & 1][3]);
                            }
                        }
                    }
                    __syncwarp();                 // every lane's ldmatrix of the slab is done
                    // this warp alone read these rows; a row holds entries only if its m-tile is active in some K-step
                    if (((bits >> z_mt) & 5u) != 0u) {
                        const uint32_t z = z_row + a * (128 * FC_ASTR);
#pragma unroll
                        for (int q = 0; q < FC_NPOS * 2; q += 16) sts128(z + q, 0u, 0u, 0u, 0u);
                    }
                }
                bar_arrive(FC_BAR_FREE + a, FC_THREADS);
                x += FC_NPOS;
                if (x > bx1) { x = bx0; ++y; }
                a = a == FC_NA - 1 ? 0 : a + 1;
            }
            // ---- epilogue: rows = pixels, columns = channels c0 + 8 nt + 2 tig (+1); the ring keeps loading meanwhile.
            // The irregular-pixel list is complete: the pixel warps wrote it before they signalled the first step.
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int m = v * 32 + mt * 16 + gid + 8 * h;
                    const int qx = gx0 + (m & 15), qy = gy0 + (m >> 4);
                    if (qx >= W || qy >= H) continue;
                    const long long qofs = (long long)qy * W + qx;
                    bool ir = false;
                    for (int i = 0; i < nirr; ++i) ir |= irr[i] == m;
                    if (ir) continue;
                    const float qm = prev != nullptr ? ld(mask + (long long)b * hw + qofs) : 1.f;
#pragma unroll
                    for (int nt = 0; nt < CN / 8; ++nt) {
                        const int c = c0 + nt * 8 + 2 * tig;
                        float v0 = acc[mt][nt][2 * h], v1 = acc[mt][nt][2 * h + 1];
                        const long long o0 = ((long long)b * hw + qofs) * C + c;
                        if (prev != nullptr) {
                            v0 = ld(prev + o0) * (1.f - qm) + v0 * qm;
                            v1 = ld(prev + o0 + 1) * (1.f - qm) + v1 * qm;
                        }
                        *reinterpret_cast<typename Pair16<T>::type*>(out + o0) = floats2_rn<T>(v0, v1);
                    }
                }
        }
        // ---- pixels with non-consecutive taps: the reference's literal arithmetic, one MMA warp per pixel, all channels.
        // The accumulators are dead by now, so this role has the registers for it.
        for (int i = v; i < nirr; i += 4) {
            const int m = irr[i], qx = gx0 + (m & 15), qy = gy0 + (m >> 4);
            const long long qofs = (long long)qy * W + qx;
            irregular_pixel<T, K, true>(src, logits, out, prev, mask, b, C, Hs, Ws, H, W, qx, qy, flow[(long long)b * 2 * hw + qofs],
                                     flow[(long long)b * 2 * hw + hw + qofs], lane);
        }
    }
}

template <int K, typename T>
static int launch_fwd(const void* src, const void* flow, const void* logits, void* out, void* probs, const void* prev, const void* mask,
                      int B, int C, int Hs, int Ws, int H, int W, cudaStream_t st_) {
    const int gcols = (W + GW - 1) / GW, grows = (H + GH - 1) / GH;
    const long long ngroups = (long long)B * gcols * grows;
    if (ngroups > INT_MAX) return GFLA_E_SHAPE;
    k_local_attn_fwd_tc<K, T><<<(unsigned)ngroups, FT_THREADS, 0, st_>>>((const T*)src, (const float*)flow, (const T*)logits, (T*)out,
                                                                        (T*)probs, (const T*)prev, (const T*)mask, C, Hs, Ws, H, W,
                                                                        gcols, grows);
    return launch_status();
}

template <int K, int CN, typename T>
static int launch_fwd_cl(const void* src, const void* flow, const void* logits, void* out, void* probs, const void* prev,
                         const void* mask, int B, int C, int Hs, int Ws, int H, int W, cudaStream_t st_) {
    const int gcols = (W + GW - 1) / GW, grows = (H + GH - 1) / GH;
    const long long ngroups = (long long)B * gcols * grows;
    if (ngroups > INT_MAX) return GFLA_E_SHAPE;
    auto kern = k_local_attn_fwd_tc_cl<K, CN, T>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, FwdClSmem<CN>::ALLOC);
    if (e != cudaSuccess) return static_cast<int>(e);
    kern<<<(unsigned)ngroups, FC_THREADS, FwdClSmem<CN>::ALLOC, st_>>>((const T*)src, (const float*)flow, (const T*)logits, (T*)out,
                                                                       (T*)probs, (const T*)prev, (const T*)mask, C, Hs, Ws, H, W,
                                                                       gcols, grows);
    return launch_status();
}

}  // namespace tc

bool local_attn_fwd_tc_supported(int C, int Ws, int k, int dtype, int flow_dtype, int layout, const void* src, const void* out) {
    const bool c_ok = C % 256 == 0 || C == 128 || C == 64;
    if (!((dtype == GFLA_BF16 || dtype == GFLA_F16) && flow_dtype == GFLA_F32 && (k == 3 || k == 5) && c_ok && aligned(src, 16))) return false;
    // channels-last: 16-byte cp.async of the source and 4-byte channel-pair stores need aligned pointers
    return layout == GFLA_NHWC ? aligned(out, 16) : (Ws % 8) == 0;
}

template <typename T>
static int local_attn_fwd_tc_t(const void* src, const void* flow, const void* logits, void* out, void* probs, const void* prev,
                               const void* mask, int B, int C, int Hs, int Ws, int H, int W, int k, int layout, cudaStream_t st_) {
    if (layout != GFLA_NHWC) return k == 5 ? tc::launch_fwd<5, T>(src, flow, logits, out, probs, prev, mask, B, C, Hs, Ws, H, W, st_)
                                           : tc::launch_fwd<3, T>(src, flow, logits, out, probs, prev, mask, B, C, Hs, Ws, H, W, st_);
    // channels-last: 128-channel passes wherever C allows them (C = 64 takes one 64-channel pass)
    const bool wide = C % 128 == 0;
#define GFLA_FC_CASE(K_, CN_) \
    if (k == K_ && wide == (CN_ == 128)) return tc::launch_fwd_cl<K_, CN_, T>(src, flow, logits, out, probs, prev, mask, B, C, Hs, Ws, H, W, st_);
    GFLA_FC_CASE(5, 128) GFLA_FC_CASE(5, 64) GFLA_FC_CASE(3, 128) GFLA_FC_CASE(3, 64)
#undef GFLA_FC_CASE
    return GFLA_E_NOTSUP;
}

int local_attn_fwd_tc(const void* src, const void* flow, const void* logits, void* out, void* probs, const void* prev,
                      const void* mask, int B, int C, int Hs, int Ws, int H, int W, int k, int dtype, int flow_dtype,
                      int layout, cudaStream_t st_) {
    if (!local_attn_fwd_tc_supported(C, Ws, k, dtype, flow_dtype, layout, src, out)) return GFLA_E_NOTSUP;
    return dtype == GFLA_F16 ? local_attn_fwd_tc_t<__half>(src, flow, logits, out, probs, prev, mask, B, C, Hs, Ws, H, W, k, layout, st_)
                             : local_attn_fwd_tc_t<__nv_bfloat16>(src, flow, logits, out, probs, prev, mask, B, C, Hs, Ws, H, W, k, layout,
                                                                  st_);
}

}  // namespace gfla
