// extern "C" surface of libgfla_warp.so (declared in include/gfla_warp.h): argument validation + dispatch, and the
// process-wide launch counter.
#include "det_accum.cuh"

namespace gfla {
int block_extract_fwd(const void*, const void*, void*, int, int, int, int, int, int, int, int, int, cudaStream_t);
int block_extract_bwd(const void*, const void*, const void*, void*, void*, int, int, int, int, int, int, int, int, int, int, int, cudaStream_t);
int convert(const void*, int, void*, int, long long, cudaStream_t);
int attn_reshape_fwd(const void*, void*, int, int, int, int, int, cudaStream_t);
int attn_reshape_bwd(const void*, void*, int, int, int, int, int, int, cudaStream_t);
int resample2d_fwd(const void*, const void*, void*, int, int, int, int, int, int, int, int, int, cudaStream_t);
int resample2d_bwd(const void*, const void*, const void*, void*, void*, int, int, int, int, int, int, int, int, int, int, cudaStream_t);
int resample2d_cos_fwd(const void*, const void*, const void*, void*, void*, int, int, int, int, int, int, int, int, double, int, cudaStream_t);
int resample2d_cos_bwd(const void*, const void*, const void*, const void*, const void*, void*, void*, void*, void*, int, int, int, int, int,
                       int, int, int, double, int, int, cudaStream_t);
int local_attn_fwd_gather(const void*, const void*, const void*, void*, void*, const void*, const void*, int, int, int, int, int, int, int, int, int, int, cudaStream_t);
int local_attn_bwd_gather(const void*, const void*, const void*, const void*, void*, void*, void*, int, int, int, int, int, int, int, int, int, int, int, cudaStream_t);
bool local_attn_bwd_tc_supported(int C, int k, int dtype, int flow_dtype, int layout, const void* src, const void* gout, const void* gsrc);
int local_attn_bwd_tc(const void* src, const void* flow, const void* logits, const void* gout, void* gsrc, void* gflow, void* glogits, int B, int C, int Hs, int Ws, int H, int W, int k, int dtype, int accumulate, cudaStream_t);
int local_attn_fwd_tc(const void*, const void*, const void*, void*, void*, const void*, const void*, int, int, int, int, int, int, int, int, int, int, cudaStream_t);
int relayout(const void*, void*, int, int, int, int, int, int, cudaStream_t);
bool local_attn_fwd_tc_supported(int C, int Ws, int k, int dtype, int flow_dtype, int layout, const void* src, const void* out);
bool patch_conv_supported(int C, int N, int dtype, int flow_dtype, int layout);
int patch_conv_fwd(const void*, const void*, const void*, void*, int, int, int, int, int, int, int, cudaStream_t);
int patch_conv_bwd(const void*, const void*, const void*, const void*, void*, void*, void*, int, int, int, int, int, int, int, int,
                   cudaStream_t);
int local_attn_bwd_gather_det(const void*, const void*, const void*, const void*, void*, void*, int, int, int, int, int, int, int, int, int,
                              int, int, fx_t*, const int*, cudaStream_t);
int local_attn_bwd_tc_det(const void*, const void*, const void*, const void*, void*, void*, int, int, int, int, int, int, int, int, int,
                          fx_t*, const int*, cudaStream_t);
int block_extract_bwd_det(const void*, const void*, const void*, void*, int, int, int, int, int, int, int, int, int, int, fx_t*, const int*,
                          cudaStream_t);
int patch_conv_bwd_det(const void*, const void*, const void*, const void*, void*, int, int, int, int, int, int, int, int, fx_t*, fx_t*,
                       const int*, cudaStream_t);
}  // namespace gfla

#include <atomic>
#include <initializer_list>

namespace gfla {
static std::atomic<unsigned long long> g_launches{0};
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
}  // namespace gfla

using namespace gfla;

#define REQ_PTR(p) do { if ((p) == nullptr) return GFLA_E_NULL; } while (0)
#define REQ_ALIGN(p, dt) do { if (!aligned((p), elem_size(dt))) return GFLA_E_ALIGN; } while (0)
#define REQ_OK(expr) do { const int r_ = (expr); if (r_ != GFLA_OK) return r_; } while (0)

template <typename... I> static inline bool pos(I... sizes) { return ((sizes > 0) && ...); }
static inline bool k_ok(int k) { return k >= 1 && k <= 9; }
static inline bool dtype_known(int d) { return elem_size(d) != 0; }

// every non-NULL pointer aligned to dtype's element size (NULL: an optional buffer the caller left out)
static inline bool all_aligned(std::initializer_list<const void*> ps, int dtype) {
    for (const void* p : ps)
        if (p != nullptr && !aligned(p, elem_size(dtype))) return false;
    return true;
}

// The two resample2d families: F32 / F64 with every buffer in dtype (half = false), or BF16 / F16 feature maps (`data`)
// next to an fp32 flow, stats, grad_in2, grad_in1 and grad_val (`wide`, half = true).  eps: 0 for the plain ops.
static int resample2d_args(bool half, int B, int C, int Hi, int Wi, int H, int W, int ks, int dilation, double eps, int dtype,
                           std::initializer_list<const void*> data, std::initializer_list<const void*> wide) {
    if (!pos(B, C, Hi, Wi, H, W) || ks < 2 || ks > 9 || dilation < 1 || !(eps >= 0)) return GFLA_E_SHAPE;
    if (half ? (dtype != GFLA_BF16 && dtype != GFLA_F16) : (dtype != GFLA_F32 && dtype != GFLA_F64)) return GFLA_E_DTYPE;
    if (!all_aligned(data, dtype) || !all_aligned(wide, half ? GFLA_F32 : dtype)) return GFLA_E_ALIGN;
    return GFLA_OK;
}

// Layout, shape, dtype and algo checks of the local-attention entry points, and the alignment of their buffers (`data` in
// dtype, `flows` in flow_dtype).  The caller has checked its required pointers.
static int local_attn_args(int B, int C, int Hs, int Ws, int H, int W, int k, int dtype, int flow_dtype, int layout, int algo,
                           std::initializer_list<const void*> data, std::initializer_list<const void*> flows) {
    if (layout != GFLA_NCHW && layout != GFLA_NHWC) return GFLA_E_SHAPE;
    if (!pos(B, C, Hs, Ws, H, W) || !k_ok(k)) return GFLA_E_SHAPE;
    if (!dtypes_ok(dtype, flow_dtype, dtype)) return GFLA_E_DTYPE;
    if (algo < 0 || algo > 2) return GFLA_E_NOTSUP;
    if (!all_aligned(data, dtype) || !all_aligned(flows, flow_dtype)) return GFLA_E_ALIGN;
    return GFLA_OK;
}

// the two local-attention backward passes check the layout before the pointers
static int local_attn_bwd_args(const void* source, const void* flow, const void* logits, const void* grad_out, const void* grad_source,
                               const void* grad_flow, const void* grad_logits, int B, int C, int Hs, int Ws, int H, int W, int k,
                               int dtype, int flow_dtype, int layout, int algo) {
    if (layout != GFLA_NCHW && layout != GFLA_NHWC) return GFLA_E_SHAPE;
    REQ_PTR(source); REQ_PTR(flow); REQ_PTR(logits); REQ_PTR(grad_out); REQ_PTR(grad_source); REQ_PTR(grad_flow); REQ_PTR(grad_logits);
    return local_attn_args(B, C, Hs, Ws, H, W, k, dtype, flow_dtype, layout, algo, {source, logits, grad_out, grad_source, grad_logits},
                           {flow, grad_flow});
}

// shape, dtype and support checks shared by the patch-convolution entry points
static int patch_conv_args(int B, int C, int Hs, int Ws, int H, int W, int k, int N, int dtype, int flow_dtype, int layout) {
    if (layout != GFLA_NCHW && layout != GFLA_NHWC) return GFLA_E_SHAPE;
    if (!pos(B, C, Hs, Ws, H, W, N) || !k_ok(k)) return GFLA_E_SHAPE;
    if (dtype != GFLA_BF16 || flow_dtype != GFLA_F32) return GFLA_E_DTYPE;
    if (!patch_conv_supported(C, N, dtype, flow_dtype, layout)) return GFLA_E_NOTSUP;
    return GFLA_OK;
}

// ------------------------------------------------------------------ deterministic backward passes (det_accum.cuh)
// The workspace of each: the fixed-point sums of every scattered output, the exponents and the maxima (fx_layout).
// Local attention and block_extractor scatter grad_source [B][C][Hs][Ws] only, with one exponent and maximum per image.
static FxLayout scatter_det_layout(int B, int C, int Hs, int Ws) { return fx_layout((long long)B * C * Hs * Ws, B, B); }
static FxLayout pc_det_layout(int B, int C, int Hs, int Ws, int k, int N) {
    return fx_layout((long long)B * Hs * Ws * C + (long long)N * k * k * C, B + 1, B + 2);
}

// NULL workspace: GFLA_E_NULL; not 16-byte aligned: GFLA_E_ALIGN; smaller than needed: GFLA_E_SHAPE
static int ws_check(const void* ws, long long bytes, const FxLayout& l) {
    if (ws == nullptr) return GFLA_E_NULL;
    if (!aligned(ws, 16)) return GFLA_E_ALIGN;
    if (bytes < 0 || (size_t)bytes < l.total) return GFLA_E_SHAPE;
    return GFLA_OK;
}

#define FX_PARTS(ws, l) \
    fx_t* sums = reinterpret_cast<fx_t*>(ws); \
    int* exps = reinterpret_cast<int*>(static_cast<char*>(ws) + (l).exps); \
    fx_t* amax = reinterpret_cast<fx_t*>(static_cast<char*>(ws) + (l).amax)

// The deterministic backward of an op that scatters only grad_source (a checked scatter_det_layout workspace): zero the
// workspace, max|G_b| over the gout_per_image elements of each image of grad_out, E_b from the bound factor * max|G_b|,
// the scatter kernel(sums, exps), and one narrowing pass into grad_source.
template <typename Kernel>
static int det_scatter(void* workspace, const FxLayout& l, const void* grad_out, long long gout_per_image, double factor,
                       void* grad_source, long long src_per_image, int B, int dtype, int accumulate, cudaStream_t st_, Kernel&& kernel) {
    FX_PARTS(workspace, l);
    int r = zero_async(workspace, l.total, st_);
    if (r == GFLA_OK) r = fx_amax(grad_out, dtype, gout_per_image, B, amax, st_);
    if (r == GFLA_OK) r = fx_exponents(amax, B, nullptr, factor, false, exps, st_);
    if (r == GFLA_OK) r = kernel(sums, exps);
    if (r == GFLA_OK) r = fx_narrow(sums, exps, src_per_image, B * src_per_image, grad_source, dtype, accumulate, st_);
    return r;
}

extern "C" {

int gfla_abi_version(void) { return GFLA_ABI_VERSION; }

const char* gfla_error_string(int code) {
    switch (code) {
        case GFLA_OK: return "ok";
        case GFLA_E_NULL: return "gfla: required pointer is NULL";
        case GFLA_E_SHAPE: return "gfla: bad shape / kernel_size";
        case GFLA_E_DTYPE: return "gfla: unsupported dtype combination";
        case GFLA_E_ALIGN: return "gfla: misaligned pointer";
        case GFLA_E_NOTSUP: return "gfla: requested algorithm cannot serve this call";
        default: return code > 0 ? cudaGetErrorString(static_cast<cudaError_t>(code)) : "gfla: unknown error";
    }
}

int gfla_device_check(void) {
    int dev = 0, major = 0, minor = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return static_cast<int>(e);
    cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
    cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
    return (major == 9 && minor == 0) ? GFLA_OK : static_cast<int>(cudaErrorNoKernelImageForDevice);
}

// The tile kernels keep no wait profile and no debug channel; the entry points stay for ABI compatibility.
int gfla_debug_wait_profile(int which, int enable, unsigned long long* out_u64x64) {
    (void)enable; (void)out_u64x64;
    return (which < 0 || which > 2) ? GFLA_E_SHAPE : GFLA_E_NOTSUP;
}

unsigned long long gfla_debug_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

int gfla_debug_set_buffer(void* host_mapped_u64x8) {
    (void)host_mapped_u64x8;
    return GFLA_E_NOTSUP;
}

int gfla_relayout(const void* src, void* dst, int B, int C, int H, int W, int dtype, int to_nhwc, gfla_stream_t stream) {
    REQ_PTR(src); REQ_PTR(dst);
    if (!pos(B, C, H, W)) return GFLA_E_SHAPE;
    if (!dtype_known(dtype)) return GFLA_E_DTYPE;
    if (src == dst) return GFLA_E_NOTSUP;
    REQ_ALIGN(src, dtype); REQ_ALIGN(dst, dtype);
    return relayout(src, dst, B, C, H, W, dtype, to_nhwc, (cudaStream_t)stream);
}

int gfla_block_extract_fwd(const void* source, const void* flow, void* out, int B, int C, int Hs, int Ws, int Hf,
                           int Wf, int k, int dtype, int flow_dtype, gfla_stream_t stream) {
    REQ_PTR(source); REQ_PTR(flow); REQ_PTR(out);
    if (!pos(B, C, Hs, Ws, Hf, Wf) || !k_ok(k)) return GFLA_E_SHAPE;
    if (!dtypes_ok(dtype, flow_dtype, dtype)) return GFLA_E_DTYPE;
    REQ_ALIGN(source, dtype); REQ_ALIGN(out, dtype); REQ_ALIGN(flow, flow_dtype);
    return block_extract_fwd(source, flow, out, B, C, Hs, Ws, Hf, Wf, k, dtype, flow_dtype, (cudaStream_t)stream);
}

int gfla_block_extract_bwd(const void* source, const void* flow, const void* grad_out, void* grad_source,
                           void* grad_flow, int B, int C, int Hs, int Ws, int Hf, int Wf, int k, int dtype,
                           int flow_dtype, int grad_source_dtype, int accumulate, gfla_stream_t stream) {
    REQ_PTR(source); REQ_PTR(flow); REQ_PTR(grad_out); REQ_PTR(grad_source); REQ_PTR(grad_flow);
    if (!pos(B, C, Hs, Ws, Hf, Wf) || !k_ok(k)) return GFLA_E_SHAPE;
    if (!dtypes_ok(dtype, flow_dtype, grad_source_dtype)) return GFLA_E_DTYPE;
    REQ_ALIGN(source, dtype); REQ_ALIGN(grad_out, dtype); REQ_ALIGN(grad_source, grad_source_dtype);
    REQ_ALIGN(flow, flow_dtype); REQ_ALIGN(grad_flow, flow_dtype);
    return block_extract_bwd(source, flow, grad_out, grad_source, grad_flow, B, C, Hs, Ws, Hf, Wf, k, dtype, flow_dtype,
                             grad_source_dtype, accumulate, (cudaStream_t)stream);
}

int gfla_convert(const void* src, int src_dtype, void* dst, int dst_dtype, long long n, gfla_stream_t stream) {
    REQ_PTR(src); REQ_PTR(dst);
    if (n <= 0) return GFLA_E_SHAPE;
    if (!dtype_known(src_dtype) || !dtype_known(dst_dtype)) return GFLA_E_DTYPE;
    REQ_ALIGN(src, src_dtype); REQ_ALIGN(dst, dst_dtype);
    return convert(src, src_dtype, dst, dst_dtype, n, (cudaStream_t)stream);
}

int gfla_attn_reshape_fwd(const void* in, void* out, int B, int H, int W, int k, int dtype, gfla_stream_t stream) {
    REQ_PTR(in); REQ_PTR(out);
    if (!pos(B, H, W) || !k_ok(k)) return GFLA_E_SHAPE;
    if (!dtype_known(dtype)) return GFLA_E_DTYPE;
    REQ_ALIGN(in, dtype); REQ_ALIGN(out, dtype);
    return attn_reshape_fwd(in, out, B, H, W, k, dtype, (cudaStream_t)stream);
}

int gfla_attn_reshape_bwd(const void* grad_out, void* grad_in, int B, int H, int W, int k, int dtype, int accumulate,
                          gfla_stream_t stream) {
    REQ_PTR(grad_out); REQ_PTR(grad_in);
    if (!pos(B, H, W) || !k_ok(k)) return GFLA_E_SHAPE;
    if (!dtype_known(dtype)) return GFLA_E_DTYPE;
    REQ_ALIGN(grad_out, dtype); REQ_ALIGN(grad_in, dtype);
    return attn_reshape_bwd(grad_out, grad_in, B, H, W, k, dtype, accumulate, (cudaStream_t)stream);
}

// ------------------------------------------------------------------ resample2d: the fp32 / fp64 and the 16-bit families
int gfla_resample2d_fwd(const void* in1, const void* in2, void* out, int B, int C, int Hi, int Wi, int H, int W, int ks,
                        int dilation, int dtype, gfla_stream_t stream) {
    REQ_PTR(in1); REQ_PTR(in2); REQ_PTR(out);
    REQ_OK(resample2d_args(false, B, C, Hi, Wi, H, W, ks, dilation, 0.0, dtype, {in1, out}, {in2}));
    return resample2d_fwd(in1, in2, out, B, C, Hi, Wi, H, W, ks, dilation, dtype, (cudaStream_t)stream);
}

int gfla_resample2d_bwd(const void* in1, const void* in2, const void* grad_out, void* grad_in1, void* grad_in2, int B,
                        int C, int Hi, int Wi, int H, int W, int ks, int dilation, int dtype, int accumulate,
                        gfla_stream_t stream) {
    REQ_PTR(in1); REQ_PTR(in2); REQ_PTR(grad_out); REQ_PTR(grad_in1); REQ_PTR(grad_in2);
    REQ_OK(resample2d_args(false, B, C, Hi, Wi, H, W, ks, dilation, 0.0, dtype, {in1, grad_out}, {in2, grad_in1, grad_in2}));
    return resample2d_bwd(in1, in2, grad_out, grad_in1, grad_in2, B, C, Hi, Wi, H, W, ks, dilation, dtype, accumulate,
                          (cudaStream_t)stream);
}

int gfla_resample2d_cosine_fwd(const void* in1, const void* in2, const void* target, void* cos_out, void* stats, int B, int C, int Hi,
                               int Wi, int H, int W, int ks, int dilation, double eps, int dtype, gfla_stream_t stream) {
    REQ_PTR(in1); REQ_PTR(in2); REQ_PTR(target); REQ_PTR(cos_out); REQ_PTR(stats);
    REQ_OK(resample2d_args(false, B, C, Hi, Wi, H, W, ks, dilation, eps, dtype, {in1, target, cos_out}, {in2, stats}));
    return resample2d_cos_fwd(in1, in2, target, cos_out, stats, B, C, Hi, Wi, H, W, ks, dilation, eps, dtype, (cudaStream_t)stream);
}

int gfla_resample2d_cosine_bwd(const void* in1, const void* in2, const void* target, const void* stats, const void* grad_cos,
                               void* grad_in1, void* grad_in2, void* grad_val, void* grad_target, int B, int C, int Hi, int Wi, int H,
                               int W, int ks, int dilation, double eps, int dtype, int accumulate, gfla_stream_t stream) {
    REQ_PTR(in1); REQ_PTR(in2); REQ_PTR(target); REQ_PTR(stats); REQ_PTR(grad_cos); REQ_PTR(grad_in2);
    if (grad_in1 != nullptr && grad_val == nullptr) return GFLA_E_NULL;      // the scatter runs on the materialised d/d(warped)
    REQ_OK(resample2d_args(false, B, C, Hi, Wi, H, W, ks, dilation, eps, dtype, {in1, target, grad_cos, grad_target},
                           {in2, stats, grad_in2, grad_in1, grad_val}));
    return resample2d_cos_bwd(in1, in2, target, stats, grad_cos, grad_in1, grad_in2, grad_val, grad_target, B, C, Hi, Wi, H, W, ks, dilation,
                              eps, dtype, accumulate, (cudaStream_t)stream);
}

int gfla_resample2d16_fwd(const void* in1, const void* in2_f32, void* out, int B, int C, int Hi, int Wi, int H, int W, int ks,
                          int dilation, int dtype, gfla_stream_t stream) {
    REQ_PTR(in1); REQ_PTR(in2_f32); REQ_PTR(out);
    REQ_OK(resample2d_args(true, B, C, Hi, Wi, H, W, ks, dilation, 0.0, dtype, {in1, out}, {in2_f32}));
    return resample2d_fwd(in1, in2_f32, out, B, C, Hi, Wi, H, W, ks, dilation, dtype, (cudaStream_t)stream);
}

int gfla_resample2d16_bwd(const void* in1, const void* in2_f32, const void* grad_out, void* grad_in1_f32, void* grad_in2_f32, int B,
                          int C, int Hi, int Wi, int H, int W, int ks, int dilation, int dtype, int accumulate, gfla_stream_t stream) {
    REQ_PTR(in1); REQ_PTR(in2_f32); REQ_PTR(grad_out); REQ_PTR(grad_in1_f32); REQ_PTR(grad_in2_f32);
    REQ_OK(resample2d_args(true, B, C, Hi, Wi, H, W, ks, dilation, 0.0, dtype, {in1, grad_out}, {in2_f32, grad_in1_f32, grad_in2_f32}));
    return resample2d_bwd(in1, in2_f32, grad_out, grad_in1_f32, grad_in2_f32, B, C, Hi, Wi, H, W, ks, dilation, dtype, accumulate,
                          (cudaStream_t)stream);
}

int gfla_resample2d16_cosine_fwd(const void* in1, const void* in2_f32, const void* target, void* cos_out, void* stats_f32, int B, int C,
                                 int Hi, int Wi, int H, int W, int ks, int dilation, double eps, int dtype, gfla_stream_t stream) {
    REQ_PTR(in1); REQ_PTR(in2_f32); REQ_PTR(target); REQ_PTR(cos_out); REQ_PTR(stats_f32);
    REQ_OK(resample2d_args(true, B, C, Hi, Wi, H, W, ks, dilation, eps, dtype, {in1, target, cos_out}, {in2_f32, stats_f32}));
    return resample2d_cos_fwd(in1, in2_f32, target, cos_out, stats_f32, B, C, Hi, Wi, H, W, ks, dilation, eps, dtype, (cudaStream_t)stream);
}

int gfla_resample2d16_cosine_bwd(const void* in1, const void* in2_f32, const void* target, const void* stats_f32, const void* grad_cos,
                                 void* grad_in1_f32, void* grad_in2_f32, void* grad_val_f32, void* grad_target, int B, int C, int Hi, int Wi,
                                 int H, int W, int ks, int dilation, double eps, int dtype, int accumulate, gfla_stream_t stream) {
    REQ_PTR(in1); REQ_PTR(in2_f32); REQ_PTR(target); REQ_PTR(stats_f32); REQ_PTR(grad_cos); REQ_PTR(grad_in2_f32);
    if (grad_in1_f32 != nullptr && grad_val_f32 == nullptr) return GFLA_E_NULL;
    REQ_OK(resample2d_args(true, B, C, Hi, Wi, H, W, ks, dilation, eps, dtype, {in1, target, grad_cos, grad_target},
                           {in2_f32, stats_f32, grad_in2_f32, grad_in1_f32, grad_val_f32}));
    return resample2d_cos_bwd(in1, in2_f32, target, stats_f32, grad_cos, grad_in1_f32, grad_in2_f32, grad_val_f32, grad_target, B, C, Hi, Wi,
                              H, W, ks, dilation, eps, dtype, accumulate, (cudaStream_t)stream);
}

// ------------------------------------------------------------------ local attention
static int local_attn_fwd_any(const void* source, const void* flow, const void* logits, void* out, void* probs,
                              const void* prev, const void* mask, int B, int C, int Hs, int Ws, int H, int W, int k, int dtype,
                              int flow_dtype, int layout, int algo, gfla_stream_t stream) {
    REQ_PTR(source); REQ_PTR(flow); REQ_PTR(logits); REQ_PTR(out);
    REQ_OK(local_attn_args(B, C, Hs, Ws, H, W, k, dtype, flow_dtype, layout, algo, {source, logits, out, probs, prev, mask}, {flow}));
    const bool tc_ok = local_attn_fwd_tc_supported(C, Ws, k, dtype, flow_dtype, layout, source, out) &&
                       (prev == nullptr || layout == GFLA_NCHW || aligned(prev, 16));
    if (algo == 2 && !tc_ok) return GFLA_E_NOTSUP;
    if (algo == 2 || (algo == 0 && tc_ok))
        return local_attn_fwd_tc(source, flow, logits, out, probs, prev, mask, B, C, Hs, Ws, H, W, k, dtype, flow_dtype, layout, (cudaStream_t)stream);
    return local_attn_fwd_gather(source, flow, logits, out, probs, prev, mask, B, C, Hs, Ws, H, W, k, dtype, flow_dtype, layout, (cudaStream_t)stream);
}

int gfla_local_attn_fwd(const void* source, const void* flow, const void* logits, void* out, void* probs, int B, int C,
                        int Hs, int Ws, int H, int W, int k, int dtype, int flow_dtype, int layout, int algo,
                        gfla_stream_t stream) {
    return local_attn_fwd_any(source, flow, logits, out, probs, nullptr, nullptr, B, C, Hs, Ws, H, W, k, dtype, flow_dtype,
                              layout, algo, stream);
}

int gfla_local_attn_blend_fwd(const void* source, const void* flow, const void* logits, const void* prev, const void* mask,
                              void* out, int B, int C, int Hs, int Ws, int H, int W, int k, int dtype, int flow_dtype,
                              int layout, int algo, gfla_stream_t stream) {
    REQ_PTR(prev); REQ_PTR(mask);
    return local_attn_fwd_any(source, flow, logits, out, nullptr, prev, mask, B, C, Hs, Ws, H, W, k, dtype, flow_dtype, layout,
                              algo, stream);
}

int gfla_local_attn_bwd(const void* source, const void* flow, const void* logits, const void* grad_out,
                        void* grad_source, void* grad_flow, void* grad_logits, int B, int C, int Hs, int Ws, int H, int W,
                        int k, int dtype, int flow_dtype, int layout, int accumulate, int algo, gfla_stream_t stream) {
    REQ_OK(local_attn_bwd_args(source, flow, logits, grad_out, grad_source, grad_flow, grad_logits, B, C, Hs, Ws, H, W, k, dtype,
                               flow_dtype, layout, algo));
    const bool tc_ok = local_attn_bwd_tc_supported(C, k, dtype, flow_dtype, layout, source, grad_out, grad_source);
    if (algo == 2 && !tc_ok) return GFLA_E_NOTSUP;
    if (algo == 2 || (algo == 0 && tc_ok))
        return local_attn_bwd_tc(source, flow, logits, grad_out, grad_source, grad_flow, grad_logits, B, C, Hs, Ws, H, W, k, dtype,
                                 accumulate, (cudaStream_t)stream);
    return local_attn_bwd_gather(source, flow, logits, grad_out, grad_source, grad_flow, grad_logits, B, C, Hs, Ws, H, W,
                                 k, dtype, flow_dtype, accumulate, layout, (cudaStream_t)stream);
}

// ------------------------------------------------------------------ patch convolution
int gfla_patch_conv_fwd(const void* source, const void* flow, const void* weight, void* out, int B, int C, int Hs, int Ws, int H,
                        int W, int k, int N, int dtype, int flow_dtype, int layout, gfla_stream_t stream) {
    REQ_PTR(source); REQ_PTR(flow); REQ_PTR(weight); REQ_PTR(out);
    REQ_OK(patch_conv_args(B, C, Hs, Ws, H, W, k, N, dtype, flow_dtype, layout));
    if (!aligned(source, 16) || !aligned(weight, 16) || !aligned(out, 16)) return GFLA_E_ALIGN;
    REQ_ALIGN(flow, flow_dtype);
    return patch_conv_fwd(source, flow, weight, out, B, C, Hs, Ws, H, W, k, (cudaStream_t)stream);
}

int gfla_patch_conv_bwd(const void* source, const void* flow, const void* weight, const void* grad_out, void* grad_source_f32,
                        void* grad_flow, void* grad_weight_f32, int B, int C, int Hs, int Ws, int H, int W, int k, int N, int dtype,
                        int flow_dtype, int layout, int accumulate, gfla_stream_t stream) {
    REQ_PTR(source); REQ_PTR(flow); REQ_PTR(weight); REQ_PTR(grad_out);
    REQ_PTR(grad_source_f32); REQ_PTR(grad_flow); REQ_PTR(grad_weight_f32);
    REQ_OK(patch_conv_args(B, C, Hs, Ws, H, W, k, N, dtype, flow_dtype, layout));
    if (!aligned(source, 16) || !aligned(weight, 16) || !aligned(grad_out, 16) || !aligned(grad_source_f32, 16) ||
        !aligned(grad_weight_f32, 16))
        return GFLA_E_ALIGN;
    REQ_ALIGN(flow, flow_dtype); REQ_ALIGN(grad_flow, flow_dtype);
    return patch_conv_bwd(source, flow, weight, grad_out, grad_source_f32, grad_flow, grad_weight_f32, B, C, Hs, Ws, H, W, k,
                          accumulate, (cudaStream_t)stream);
}

// ------------------------------------------------------------------ deterministic backward passes
long long gfla_local_attn_bwd_det_workspace_bytes(int B, int C, int Hs, int Ws, int H, int W, int k) {
    if (!pos(B, C, Hs, Ws, H, W) || !k_ok(k)) return GFLA_E_SHAPE;
    return (long long)scatter_det_layout(B, C, Hs, Ws).total;
}

int gfla_local_attn_bwd_det(const void* source, const void* flow, const void* logits, const void* grad_out, void* grad_source,
                            void* grad_flow, void* grad_logits, int B, int C, int Hs, int Ws, int H, int W, int k, int dtype,
                            int flow_dtype, int layout, int accumulate, int algo, void* workspace, long long workspace_bytes,
                            gfla_stream_t stream) {
    REQ_OK(local_attn_bwd_args(source, flow, logits, grad_out, grad_source, grad_flow, grad_logits, B, C, Hs, Ws, H, W, k, dtype,
                               flow_dtype, layout, algo));
    const FxLayout l = scatter_det_layout(B, C, Hs, Ws);
    REQ_OK(ws_check(workspace, workspace_bytes, l));
    // the tile kernel never writes grad_source here (fx_narrow does): its alignment must not change which kernel runs
    const bool tc_ok = local_attn_bwd_tc_supported(C, k, dtype, flow_dtype, layout, source, grad_out, source);
    if (algo == 2 && !tc_ok) return GFLA_E_NOTSUP;
    const bool tile = algo == 2 || (algo == 0 && tc_ok);
    const cudaStream_t st_ = (cudaStream_t)stream;
    // Bound of image b: every pixel spreads g_c times weights that sum to exactly 1/k^2 (softmax probabilities summing to
    // 1, times bilinear weights summing to 1, times 1/k^2) over the source positions, so every grad_source element of the
    // image is at most (H W / k^2) max|G_b| in magnitude, and so is the sum of the magnitudes of its partials.  The tile
    // kernel rounds the weights to the data's 16-bit type first.  bf16: a factor of at most 1 + 2^-8 on a pixel's weight
    // sum.  fp16: a normal weight grows by at most 2^-11 of itself (factor 1 + 2^-11), and a weight below 2^-14 is
    // subnormal and off by at most 2^-25 absolutely, (k+1)^2 2^-25 per pixel at most: against the pixel's weight sum 1/k^2
    // that is k^2 (k+1)^2 2^-25 <= 900 2^-25 < 2^-15 (k <= 5, the only tile sizes).  Together below 1 + 2^-10.  Either
    // factor stays far inside the one bit of margin below 2^62 (det_accum.cuh), which only requires a factor below 2.
    return det_scatter(workspace, l, grad_out, (long long)C * H * W, (double)H * W / ((double)k * k), grad_source,
                       (long long)C * Hs * Ws, B, dtype, accumulate, st_, [&](fx_t* sums, const int* exps) {
        if (tile)
            return local_attn_bwd_tc_det(source, flow, logits, grad_out, grad_flow, grad_logits, B, C, Hs, Ws, H, W, k, dtype, accumulate,
                                         sums, exps, st_);
        return local_attn_bwd_gather_det(source, flow, logits, grad_out, grad_flow, grad_logits, B, C, Hs, Ws, H, W, k, dtype,
                                         flow_dtype, accumulate, layout, sums, exps, st_);
    });
}

long long gfla_block_extract_bwd_det_workspace_bytes(int B, int C, int Hs, int Ws, int Hf, int Wf, int k) {
    if (!pos(B, C, Hs, Ws, Hf, Wf) || !k_ok(k)) return GFLA_E_SHAPE;
    return (long long)scatter_det_layout(B, C, Hs, Ws).total;
}

int gfla_block_extract_bwd_det(const void* source, const void* flow, const void* grad_out, void* grad_source, void* grad_flow,
                               int B, int C, int Hs, int Ws, int Hf, int Wf, int k, int dtype, int flow_dtype, int accumulate,
                               void* workspace, long long workspace_bytes, gfla_stream_t stream) {
    REQ_PTR(source); REQ_PTR(flow); REQ_PTR(grad_out); REQ_PTR(grad_source); REQ_PTR(grad_flow);
    if (!pos(B, C, Hs, Ws, Hf, Wf) || !k_ok(k)) return GFLA_E_SHAPE;
    if (!dtypes_ok(dtype, flow_dtype, dtype)) return GFLA_E_DTYPE;
    REQ_ALIGN(source, dtype); REQ_ALIGN(grad_out, dtype); REQ_ALIGN(grad_source, dtype);
    REQ_ALIGN(flow, flow_dtype); REQ_ALIGN(grad_flow, flow_dtype);
    const FxLayout l = scatter_det_layout(B, C, Hs, Ws);
    REQ_OK(ws_check(workspace, workspace_bytes, l));
    const cudaStream_t st_ = (cudaStream_t)stream;
    // Bound of image b: every grad_out element spreads bilinear weights that sum to 1 over 4 source positions of its
    // channel, so a grad_source element collects at most the k^2 Hf Wf elements of its channel: k^2 Hf Wf max|G_b|.
    return det_scatter(workspace, l, grad_out, (long long)C * k * Hf * k * Wf, (double)k * k * Hf * Wf, grad_source,
                       (long long)C * Hs * Ws, B, dtype, accumulate, st_, [&](fx_t* sums, const int* exps) {
        return block_extract_bwd_det(source, flow, grad_out, grad_flow, B, C, Hs, Ws, Hf, Wf, k, dtype, flow_dtype, accumulate, sums,
                                     exps, st_);
    });
}

long long gfla_patch_conv_bwd_det_workspace_bytes(int B, int C, int Hs, int Ws, int H, int W, int k, int N) {
    if (!pos(B, C, Hs, Ws, H, W, N) || !k_ok(k)) return GFLA_E_SHAPE;
    return (long long)pc_det_layout(B, C, Hs, Ws, k, N).total;
}

int gfla_patch_conv_bwd_det(const void* source, const void* flow, const void* weight, const void* grad_out, void* grad_source,
                            void* grad_flow, void* grad_weight, int B, int C, int Hs, int Ws, int H, int W, int k, int N, int dtype,
                            int flow_dtype, int layout, int accumulate, void* workspace, long long workspace_bytes,
                            gfla_stream_t stream) {
    REQ_PTR(source); REQ_PTR(flow); REQ_PTR(weight); REQ_PTR(grad_out);
    REQ_PTR(grad_source); REQ_PTR(grad_flow); REQ_PTR(grad_weight);
    REQ_OK(patch_conv_args(B, C, Hs, Ws, H, W, k, N, dtype, flow_dtype, layout));
    if (!aligned(source, 16) || !aligned(weight, 16) || !aligned(grad_out, 16)) return GFLA_E_ALIGN;
    REQ_ALIGN(grad_source, dtype); REQ_ALIGN(grad_weight, dtype); REQ_ALIGN(flow, flow_dtype); REQ_ALIGN(grad_flow, flow_dtype);
    const FxLayout l = pc_det_layout(B, C, Hs, Ws, k, N);
    REQ_OK(ws_check(workspace, workspace_bytes, l));
    const cudaStream_t st_ = (cudaStream_t)stream;
    FX_PARTS(workspace, l);
    const long long n_src = (long long)B * Hs * Ws * C, n_w = (long long)N * k * k * C;
    int r = zero_async(workspace, l.total, st_);
    if (r == GFLA_OK) r = fx_amax(grad_out, dtype, (long long)H * W * N, B, amax, st_);     // amax[b] = max|G_b|
    if (r == GFLA_OK) r = fx_amax(weight, dtype, n_w, 1, amax + B, st_);                   // amax[B] = max|W|
    if (r == GFLA_OK) r = fx_amax(source, dtype, n_src, 1, amax + B + 1, st_);             // amax[B+1] = max|source|
    // grad_source of image b: GA[p, tap, c] = sum_n G[p, n] W[n, tap, c] is at most N max|G_b| max|W|, and each (pixel,
    // tap) spreads it with bilinear weights summing to 1, so an element collects at most k^2 H W N max|G_b| max|W|.
    if (r == GFLA_OK) r = fx_exponents(amax, B, amax + B, (double)k * k * H * W * N, false, exps, st_);
    // grad_weight, one exponent for the call: sum over b and p of G[b, p, n] A[b, p, tap, c], where A (a convex blend of
    // source values rounded to bf16) is at most max|source|: B H W max|G| max|source|.
    if (r == GFLA_OK) r = fx_exponents(amax, B, amax + B + 1, (double)B * H * W, true, exps + B, st_);
    if (r == GFLA_OK)
        r = patch_conv_bwd_det(source, flow, weight, grad_out, grad_flow, B, C, Hs, Ws, H, W, k, accumulate, sums, sums + n_src, exps,
                               st_);
    if (r == GFLA_OK) r = fx_narrow(sums, exps, (long long)Hs * Ws * C, n_src, grad_source, dtype, accumulate, st_);
    if (r == GFLA_OK) r = fx_narrow(sums + n_src, exps + B, n_w, n_w, grad_weight, dtype, accumulate, st_);
    return r;
}

long long gfla_local_attn_bwd_workspace_bytes(int B) { (void)B; return 0; }   // the tile backward's scratch: the library's pool

int gfla_local_attn_bwd_ws(const void* source, const void* flow, const void* logits, const void* grad_out,
                           void* grad_source, void* grad_flow, void* grad_logits, int B, int C, int Hs, int Ws, int H, int W,
                           int k, int dtype, int flow_dtype, int layout, int accumulate, int algo, void* workspace,
                           long long workspace_bytes, gfla_stream_t stream) {
    if (workspace != nullptr && workspace_bytes < 0) return GFLA_E_SHAPE;
    return gfla_local_attn_bwd(source, flow, logits, grad_out, grad_source, grad_flow, grad_logits, B, C, Hs, Ws, H, W, k, dtype,
                               flow_dtype, layout, accumulate, algo, stream);
}

}  // extern "C"
