// Pieces shared by the forward and backward tile kernels: pixel-group geometry, the collapsed (k+1)x(k+1) weight
// window and its scatter into the 16-bit weight slab, and the literal path of pixels whose taps are not consecutive.
// T, the 16-bit element type of the data and of the weight slab, is __nv_bfloat16 or __half.
#pragma once
#include <climits>

#include "local_attn_pixel.cuh"
#include "tc_common.cuh"

namespace gfla {
namespace tc {

constexpr int GW = 16, GH = 8;          // pixel group: 16 x 8 = 128 pixels (= M or K of the MMAs)
constexpr int SEG = 16;                 // source positions per row segment = one MMA K step

// this CTA's pixel group: image b, top-left pixel (gx0, gy0); groups are numbered row-major within each image
__device__ __forceinline__ void group_decode(int gcols, int grows, uint32_t& b, int& gx0, int& gy0) {
    FastDiv fc, fr;
    fc.init(gcols);
    fr.init(grows);
    uint32_t g = blockIdx.x, gc, gr;
    fc.divmod(g, g, gc);
    fr.divmod(g, b, gr);
    gx0 = gc * GW;
    gy0 = gr * GH;
}

// bounding box (clamped tap positions) of one 16x8 pixel group from its flow: warp-collective, lane owns pixels
// lane + 32 i
template <int K>
__device__ __forceinline__ void group_bbox(const float* __restrict__ flow, int b, int gx0, int gy0, int H, int W, int Hs,
                                           int Ws, int lane, int& x0, int& y0, int& x1, int& y1) {
    const long long hw = (long long)H * W;
    float rfx[4], rfy[4];   // all loads first, then the taps: fused into one loop, the backward kernel needs more registers
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = lane + 32 * i, px = gx0 + (m & 15), py = gy0 + (m >> 4);
        const bool valid = px < W && py < H;
        const long long o = (long long)b * 2 * hw + (long long)py * W + px;
        rfx[i] = valid ? flow[o] : 0.f;
        rfy[i] = valid ? flow[o + hw] : 0.f;
    }
    int xmin = INT_MAX, xmax = INT_MIN, ymin = INT_MAX, ymax = INT_MIN;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = lane + 32 * i, px = gx0 + (m & 15), py = gy0 + (m >> 4);
        if (px < W && py < H) {
            xmin = min(xmin, axis_tap<float>(rfx[i], -(K / 2), px, Ws).lo);
            xmax = max(xmax, axis_tap<float>(rfx[i], K - 1 - K / 2, px, Ws).hi);
            ymin = min(ymin, axis_tap<float>(rfy[i], -(K / 2), py, Hs).lo);
            ymax = max(ymax, axis_tap<float>(rfy[i], K - 1 - K / 2, py, Hs).hi);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        xmin = min(xmin, __shfl_xor_sync(0xffffffffu, xmin, o));
        xmax = max(xmax, __shfl_xor_sync(0xffffffffu, xmax, o));
        ymin = min(ymin, __shfl_xor_sync(0xffffffffu, ymin, o));
        ymax = max(ymax, __shfl_xor_sync(0xffffffffu, ymax, o));
    }
    x0 = xmin; y0 = ymin; x1 = xmax; y1 = ymax;
}

// Collapsed window of one (regular) pixel: w[r][s] multiplies source position (Y0 + r, X0 + s).
// p = softmax probabilities (already scaled by whatever the caller wants, e.g. 1/k^2).  Border handling =
// the reference's index clamp: weights of out-of-range columns / rows are folded onto the border position.
// On return X0 / Y0 are shifted so that the mapping also holds for windows lying entirely outside the image.
// The kernels only ever store the weights as T, so the window comes back as T pairs: wp[r (K+1)/2 + s/2] holds w[r][s]
// in its low half for even s, in its high half for odd s.
template <typename T, int K>
__device__ __forceinline__ void build_window(const float* p, const AxisTap<float> (&tx)[K], const AxisTap<float> (&ty)[K],
                                             int Hs, int Ws, float scale, uint32_t (&wp)[(K + 1) * (K + 1) / 2], int& X0, int& Y0) {
    constexpr int K1 = K + 1;
    float w[K1 * K1];
#pragma unroll
    for (int i = 0; i < K1 * K1; ++i) w[i] = 0.f;
#pragma unroll
    for (int i = 0; i < K; ++i) {  // separably: x-weights of row i first, then spread over the two y-taps
        float rowx[K1];
#pragma unroll
        for (int s = 0; s < K1; ++s) rowx[s] = 0.f;
#pragma unroll
        for (int j = 0; j < K; ++j) {
            const float pij = p[i * K + j] * scale;
            rowx[j] += pij * tx[j].wlo;
            rowx[j + 1] += pij * tx[j].whi;
        }
#pragma unroll
        for (int s = 0; s < K1; ++s) {
            w[i * K1 + s] += ty[i].wlo * rowx[s];
            w[(i + 1) * K1 + s] += ty[i].whi * rowx[s];
        }
    }
    X0 = tx[0].fl;
    Y0 = ty[0].fl;
    if (X0 < 0 || X0 + K > Ws - 1 || Y0 < 0 || Y0 + K > Hs - 1) {  // only pixels whose window crosses the image edge
#pragma unroll
        for (int r = 0; r < K1; ++r) {
#pragma unroll
            for (int s = 0; s < K; ++s)
                if (X0 + s < 0) { w[r * K1 + s + 1] += w[r * K1 + s]; w[r * K1 + s] = 0.f; }
#pragma unroll
            for (int s = K; s > 0; --s)
                if (X0 + s > Ws - 1) { w[r * K1 + s - 1] += w[r * K1 + s]; w[r * K1 + s] = 0.f; }
        }
#pragma unroll
        for (int s = 0; s < K1; ++s) {
#pragma unroll
            for (int r = 0; r < K; ++r)
                if (Y0 + r < 0) { w[(r + 1) * K1 + s] += w[r * K1 + s]; w[r * K1 + s] = 0.f; }
#pragma unroll
            for (int r = K; r > 0; --r)
                if (Y0 + r > Hs - 1) { w[(r - 1) * K1 + s] += w[r * K1 + s]; w[r * K1 + s] = 0.f; }
        }
        // a window entirely outside the image has been folded onto its last (first) column / row, which
        // belongs on border position 0 (Ws-1, Hs-1)
        X0 = min(max(X0, -K), Ws - 1);
        Y0 = min(max(Y0, -K), Hs - 1);
    }
#pragma unroll
    for (int i = 0; i < K1 * K1 / 2; ++i) wp[i] = bits16<T>(w[2 * i]) | (bits16<T>(w[2 * i + 1]) << 16);
}

// This pixel's weights for source row y, positions [x, x + NPOS): window row y - Y0 (nothing when the row is outside the
// window), stored as 16-bit values at base + e * stride for position x + e.  The zero entries are the caller's to write.
template <int K, int NPOS = SEG>
__device__ __forceinline__ void scatter_window_row(uint32_t base, uint32_t stride, const uint32_t (&wp)[(K + 1) * (K + 1) / 2],
                                                   int X0, int Y0, int y, int x) {
    constexpr int K1 = K + 1, RW = K1 / 2;   // 16-bit pairs per window row
    const int rr = y - Y0;
    if (rr < 0 || rr > K) return;
    uint32_t wr[RW];
#pragma unroll
    for (int s = 0; s < RW; ++s) wr[s] = 0u;
#pragma unroll
    for (int r = 0; r < K1; ++r)
        if (rr == r) {
#pragma unroll
            for (int s = 0; s < RW; ++s) wr[s] = wp[r * RW + s];
        }
#pragma unroll
    for (int s = 0; s < K1; ++s) {
        const int e = X0 + s - x;
        const uint32_t h = (s & 1) ? wr[s / 2] >> 16 : wr[s / 2] & 0xffffu;
        if (e >= 0 && e < NPOS && (h & 0x7fffu) != 0u) sts16(base + e * stride, h);
    }
}

// Does this pixel's window touch the step at source row y, positions [x, x + SEG)?  Its clamped extent
// [clampi(X0), clampi(X0 + K)] x [clampi(Y0), clampi(Y0 + K)] is the same for the unfolded origin (tx[0].fl, ty[0].fl)
// and the folded one build_window returns.  It holds every position scatter_window_row writes and every clamped position
// the backward's Q pick reads, so a pixel for which this is false adds exact zeros to every MMA of the step.
template <int K>
__device__ __forceinline__ bool window_meets_step(int X0, int Y0, int Hs, int Ws, int y, int x) {
    return clampi(Y0, Hs - 1) <= y && y <= clampi(Y0 + K, Hs - 1) && clampi(X0, Ws - 1) < x + SEG && clampi(X0 + K, Ws - 1) >= x;
}

// warp-collective: bit 0 = some pixel of group row 2 warp (lanes 0-15) is active, bit 1 = the same for row 2 warp + 1
__device__ __forceinline__ uint32_t warp_row_bits(bool active) {
    const uint32_t bal = __ballot_sync(0xffffffffu, active);
    return ((bal & 0xffffu) != 0u ? 1u : 0u) | ((bal >> 16) != 0u ? 2u : 0u);
}

// One "irregular" pixel (taps not consecutive integers: fp32 rounding of (flow+offset)+coord straddling an integer,
// ~1e-5 of all pixels) with the reference's literal 4-taps-per-(i,j) arithmetic (block_extractor_kernel.cu:57-82
// followed by base_function.py:804-810).  One such pixel costs 4*k*k*C dependent loads, so a whole warp shares it:
// every lane evaluates the (identical) softmax and taps, lanes split the channels.  The (i, j) loops stay rolled: an
// unrolled tap table is register-hungry and would raise the pressure of (or spill into) the hot epilogue loop.
template <typename T, int K, bool NHWC>
__device__ __forceinline__ void irregular_pixel(const T* __restrict__ src, const T* __restrict__ logits, T* __restrict__ out,
                                                const T* __restrict__ prev, const T* __restrict__ mask, int b, int C, int Hs, int Ws,
                                                int H, int W,
                                                int qx, int qy, float qfx, float qfy, int lane) {
    constexpr int KK = K * K;
    const long long hw = (long long)H * W, qofs = (long long)qy * W + qx;
    float p[KK];
    pixel_softmax<T, float, KK>(logits + (long long)b * KK * hw + qofs, hw, KK, p);   // every lane: same loads
    const long long spl = (long long)Hs * Ws;
    const long long sc = NHWC ? 1 : spl, sp = NHWC ? C : 1;     // element strides: channel, position
    const T* sb = src + (long long)b * spl * C;
    T* ob = NHWC ? out + ((long long)b * hw + qofs) * C : out + (long long)b * C * hw + qofs;
    for (int c = lane; c < C; c += 32) {
        const T* s = sb + c * sc;
        float acc = 0.f;
#pragma unroll 1
        for (int i = 0; i < K; ++i) {      // rolled on purpose (rare path): keeps the tap table out of the registers
            const AxisTap<float> ty = axis_tap<float>(qfy, i - K / 2, qy, Hs);
#pragma unroll 1
            for (int j = 0; j < K; ++j) {
                const AxisTap<float> tx = axis_tap<float>(qfx, j - K / 2, qx, Ws);
                acc += p[i * K + j] * tap_value(s, tx, ty, Ws, sp);
            }
        }
        acc *= 1.0f / static_cast<float>(KK);
        if (prev != nullptr) {
            const float qm = ld(mask + (long long)b * hw + qofs);
            const T* pb = NHWC ? prev + ((long long)b * hw + qofs) * C : prev + (long long)b * C * hw + qofs;
            acc = ld(pb + (NHWC ? (long long)c : (long long)c * hw)) * (1.f - qm) + acc * qm;
        }
        st(ob + (NHWC ? (long long)c : (long long)c * hw), acc);
    }
}

}  // namespace tc
}  // namespace gfla
