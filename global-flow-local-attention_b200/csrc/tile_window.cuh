// Pieces shared by the forward and backward tile kernels: pixel-group geometry, per-pixel softmax,
// the reference's tap arithmetic and the collapsed (k+1)x(k+1) weight window.
#pragma once
#include <climits>

#include "common.cuh"
#include "tc_common.cuh"

namespace gfla {
namespace tc {

constexpr int GW = 16, GH = 8;          // pixel group: 16 x 8 = 128 pixels (= M or K of the MMAs)
constexpr int SEG = 16;                 // source positions per row segment = one MMA K step

// softmax over the KK logits of one pixel (bf16 planes, stride hw), fp32 arithmetic
template <int KK>
__device__ __forceinline__ void pixel_softmax_f32(const __nv_bfloat16* __restrict__ lg, long long hw, float* p) {
    float mx = -INFINITY;
#pragma unroll
    for (int t = 0; t < KK; ++t) {
        p[t] = __bfloat162float(lg[t * hw]);
        mx = fmaxf(mx, p[t]);
    }
    float sum = 0.f;
#pragma unroll
    for (int t = 0; t < KK; ++t) {
        p[t] = expf(p[t] - mx);
        sum += p[t];
    }
    const float inv = 1.0f / sum;
#pragma unroll
    for (int t = 0; t < KK; ++t) p[t] *= inv;
}

// the same from logits already held in registers (p[t] = logit on entry)
template <int KK>
__device__ __forceinline__ void softmax_inplace_f32(float* p) {
    float mx = -INFINITY;
#pragma unroll
    for (int t = 0; t < KK; ++t) mx = fmaxf(mx, p[t]);
    float sum = 0.f;
#pragma unroll
    for (int t = 0; t < KK; ++t) {
        p[t] = expf(p[t] - mx);
        sum += p[t];
    }
    const float inv = 1.0f / sum;
#pragma unroll
    for (int t = 0; t < KK; ++t) p[t] *= inv;
}

// the k taps per axis, evaluated exactly like the reference; "regular" = consecutive integers
template <int K>
__device__ __forceinline__ bool taps_regular(float flow_x, float flow_y, int x, int y, int Hs, int Ws,
                                             AxisTap<float> (&tx)[K], AxisTap<float> (&ty)[K]) {
    bool regular = true;
#pragma unroll
    for (int j = 0; j < K; ++j) {
        tx[j] = axis_tap<float>(flow_x, j - K / 2, x, Ws);
        ty[j] = axis_tap<float>(flow_y, j - K / 2, y, Hs);
        regular = regular && (tx[j].fl == tx[0].fl + j) && (ty[j].fl == ty[0].fl + j);
    }
    return regular;
}

// Flow of this lane's 4 pixels of a 16x8 pixel group (pixel m = lane + 32 i; zeros outside the image).  Split from
// the reduction below so that a producer can issue the loads a whole tile of work before it needs the box.
struct TileFlow { float fx[4], fy[4]; };

__device__ __forceinline__ void tile_flow_load(const float* __restrict__ flow, int b, int gx0, int gy0, int H, int W, int lane,
                                               TileFlow& r) {
    const long long hw = (long long)H * W;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = lane + 32 * i, px = gx0 + (m & 15), py = gy0 + (m >> 4);
        const bool valid = px < W && py < H;
        const long long o = (long long)b * 2 * hw + (long long)py * W + px;
        r.fx[i] = valid ? flow[o] : 0.f;
        r.fy[i] = valid ? flow[o + hw] : 0.f;
    }
}

// bounding box (clamped tap positions) of one 16x8 pixel group from its flow values: warp-collective.
// align_x8: NCHW tensor maps need the innermost (x) box origin on a 16-byte boundary.
template <int K>
__device__ __forceinline__ void tile_bbox_reduce(const TileFlow& r, int gx0, int gy0, int H, int W, int Hs, int Ws, int lane,
                                                 bool align_x8, int& x0, int& y0, int& x1, int& y1) {
    int xmin = INT_MAX, xmax = INT_MIN, ymin = INT_MAX, ymax = INT_MIN;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = lane + 32 * i, px = gx0 + (m & 15), py = gy0 + (m >> 4);
        if (px < W && py < H) {
            xmin = min(xmin, axis_tap<float>(r.fx[i], -(K / 2), px, Ws).lo);
            xmax = max(xmax, axis_tap<float>(r.fx[i], K - 1 - K / 2, px, Ws).hi);
            ymin = min(ymin, axis_tap<float>(r.fy[i], -(K / 2), py, Hs).lo);
            ymax = max(ymax, axis_tap<float>(r.fy[i], K - 1 - K / 2, py, Hs).hi);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        xmin = min(xmin, __shfl_xor_sync(0xffffffffu, xmin, o));
        xmax = max(xmax, __shfl_xor_sync(0xffffffffu, xmax, o));
        ymin = min(ymin, __shfl_xor_sync(0xffffffffu, ymin, o));
        ymax = max(ymax, __shfl_xor_sync(0xffffffffu, ymax, o));
    }
    if (align_x8) xmin &= ~7;
    x0 = xmin; y0 = ymin; x1 = xmax; y1 = ymax;
}

template <int K>
__device__ __forceinline__ void group_bbox(const float* __restrict__ flow, int b, int gx0, int gy0, int H, int W, int Hs,
                                           int Ws, int lane, bool align_x8, int& x0, int& y0, int& x1, int& y1) {
    TileFlow r;
    tile_flow_load(flow, b, gx0, gy0, H, W, lane, r);
    tile_bbox_reduce<K>(r, gx0, gy0, H, W, Hs, Ws, lane, align_x8, x0, y0, x1, y1);
}

// Collapsed window of one (regular) pixel: w[r][s] multiplies source position (Y0 + r, X0 + s).
// p = softmax probabilities (already scaled by whatever the caller wants, e.g. 1/k^2).  Border handling =
// the reference's index clamp: weights of out-of-range columns / rows are folded onto the border position.
// On return X0 / Y0 are shifted so that the mapping also holds for windows lying entirely outside the image.
template <int K>
__device__ __forceinline__ void build_window(const float* p, const AxisTap<float> (&tx)[K], const AxisTap<float> (&ty)[K],
                                             int Hs, int Ws, float scale, float* w, int& X0, int& Y0) {
    constexpr int K1 = K + 1;
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
}

// One "irregular" pixel (taps not consecutive integers: fp32 rounding of (flow+offset)+coord straddling an integer,
// ~1e-5 of all pixels) with the reference's literal 4-taps-per-(i,j) arithmetic (block_extractor_kernel.cu:57-82
// followed by base_function.py:804-810).  One such pixel costs 4*k*k*CN dependent loads, so a whole warp shares it:
// every lane evaluates the (identical) softmax and taps, lanes split the channels [c0, c0 + CN).  The (i, j) loops stay
// rolled: an unrolled tap table is register-hungry and would raise the pressure of (or spill into) the hot epilogue loop.
template <int K, bool NHWC>
__device__ __forceinline__ void irregular_pixel(const __nv_bfloat16* __restrict__ src, const __nv_bfloat16* __restrict__ logits,
                                                __nv_bfloat16* __restrict__ out, const __nv_bfloat16* __restrict__ prev,
                                                const __nv_bfloat16* __restrict__ mask, int b, int C, int c0, int CN, int Hs,
                                                int Ws, int H, int W, int qx, int qy, float qfx, float qfy, int lane) {
    constexpr int KK = K * K;
    const long long hw = (long long)H * W, qofs = (long long)qy * W + qx;
    float p[KK];
    pixel_softmax_f32<KK>(logits + (long long)b * KK * hw + qofs, hw, p);   // every lane: same loads (broadcast)
    const long long spl = (long long)Hs * Ws;
    const long long sc = NHWC ? 1 : spl, sp = NHWC ? C : 1;     // element strides: channel, position
    const __nv_bfloat16* sb = NHWC ? src + (long long)b * spl * C + c0 : src + ((long long)b * C + c0) * spl;
    __nv_bfloat16* ob = NHWC ? out + ((long long)b * hw + qofs) * C + c0 : out + ((long long)b * C + c0) * hw + qofs;
    for (int c = lane; c < CN; c += 32) {
        const __nv_bfloat16* s = sb + c * sc;
        float acc = 0.f;
#pragma unroll 1
        for (int i = 0; i < K; ++i) {      // rolled on purpose (rare path): keeps the tap table out of the registers
            const AxisTap<float> ty = axis_tap<float>(qfy, i - K / 2, qy, Hs);
#pragma unroll 1
            for (int j = 0; j < K; ++j) {
                const AxisTap<float> tx = axis_tap<float>(qfx, j - K / 2, qx, Ws);
                float v = 0.f;
                v += tx.wlo * ty.wlo * __bfloat162float(s[(ty.lo * Ws + tx.lo) * sp]);
                v += tx.whi * ty.wlo * __bfloat162float(s[(ty.lo * Ws + tx.hi) * sp]);
                v += tx.wlo * ty.whi * __bfloat162float(s[(ty.hi * Ws + tx.lo) * sp]);
                v += tx.whi * ty.whi * __bfloat162float(s[(ty.hi * Ws + tx.hi) * sp]);
                acc += p[i * K + j] * v;
            }
        }
        acc *= 1.0f / static_cast<float>(KK);
        if (prev != nullptr) {
            const float qm = __bfloat162float(mask[(long long)b * hw + qofs]);
            const __nv_bfloat16* pb = NHWC ? prev + ((long long)b * hw + qofs) * C + c0 : prev + ((long long)b * C + c0) * hw + qofs;
            acc = __bfloat162float(pb[NHWC ? (long long)c : (long long)c * hw]) * (1.f - qm) + acc * qm;
        }
        ob[NHWC ? (long long)c : (long long)c * hw] = __float2bfloat16_rn(acc);
    }
}

}  // namespace tc
}  // namespace gfla
