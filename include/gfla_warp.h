/*
 * gfla_warp.h -- C ABI of the H100-native (sm_90a) GFLA warping library.
 *
 * This is the drop-in boundary for the warping hot path of
 * RenYurui/Global-Flow-Local-Attention: the three custom extensions under
 * model/networks/ (block_extractor, local_attn_reshape, resample2d_package)
 * and the local-attention softmax-weighted gather they feed (ExtractorAttn,
 * model/networks/base_function.py:790-818).  Each entry point names the
 * reference interface (pybind function, file:line) it replaces.
 *
 * Conventions (all entry points)
 *   - plain pointers + sizes only: no torch / ATen types cross this boundary.
 *     Pointers are DEVICE pointers to contiguous NCHW tensors on the device
 *     that owns `stream` (the caller's current device).
 *   - `stream` is a cudaStream_t passed as void* (0 = legacy default stream).
 *     The reference launches on at::cuda::getCurrentCUDAStream()
 *     (block_extractor_kernel.cu:197); callers pass that same stream.
 *   - nothing is synchronised inside the library.  It allocates in one place:
 *     the tile backward (gfla_local_attn_bwd, gfla_local_attn_bwd_ws) takes
 *     fp32 border sums, 2*(Hs+Ws)*C floats per image, stream-ordered from a
 *     memory pool that the library creates for each device on first use and
 *     keeps for the life of the process; the call hands them back to the pool
 *     on its stream.  The only other state is a process-wide launch counter
 *     (gfla_debug_launch_count).  Both are thread-safe.
 *   - return value: 0 on success; a negative GFLA_E_* code for argument
 *     errors (nothing was launched); a positive cudaError_t if a launch
 *     failed.  (The reference returns the constant 1 and checks nothing,
 *     block_extractor_cuda.cc:12; see INTEGRATION.md for the shim that maps
 *     this back to the legacy `int` return.)
 *   - dtype codes describe the element type of source / output / logits /
 *     gradient tensors; `flow_dtype` that of the flow field and its gradient.
 *     F32 and F64 mirror the reference's AT_DISPATCH_FLOATING_TYPES
 *     (float, double only).  BF16 / F16 storage is an extension: arithmetic
 *     is fp32, and the flow may stay fp32 (`flow_dtype` = GFLA_F32) so the tap
 *     indices are bit-identical to the fp32 reference.
 *   - every size is an `int` like in the reference, but products are formed
 *     in 64 bits (the reference overflows `int n` above 2^31 elements,
 *     block_extractor_kernel.cu:33,180).
 *   - `accumulate` (backward entry points): 1 = reference semantics -- the
 *     gradients are ADDED into caller-provided (normally zero-filled) buffers
 *     (block_extractor.py:35-36, resample2d.py:32-33); 0 = the library
 *     overwrites them (zero-filling internally where it scatters), so the
 *     caller may pass uninitialised memory.
 */
#ifndef GFLA_WARP_H_
#define GFLA_WARP_H_

#ifdef __cplusplus
extern "C" {
#endif

#define GFLA_ABI_VERSION 1

typedef void* gfla_stream_t; /* cudaStream_t */

enum gfla_dtype { GFLA_F32 = 0, GFLA_F64 = 1, GFLA_BF16 = 2, GFLA_F16 = 3 };

/* storage order of the [B,C,H,W] feature tensors of the fused op (source, out and their gradients);
 * flow / logits / probs are always planar (NCHW).  NHWC = torch.channels_last. */
enum gfla_layout { GFLA_NCHW = 0, GFLA_NHWC = 1 };

enum gfla_error {
    GFLA_OK = 0,
    GFLA_E_NULL = -1,     /* a required pointer is NULL                          */
    GFLA_E_SHAPE = -2,    /* non-positive size, or kernel_size outside [1, 9]    */
    GFLA_E_DTYPE = -3,    /* unknown dtype code / unsupported dtype combination  */
    GFLA_E_ALIGN = -4,    /* pointer not aligned to its element size             */
    GFLA_E_NOTSUP = -5    /* requested fast path cannot serve this call          */
};

int gfla_abi_version(void);
/* static string for any code returned by this library (GFLA_E_* or cudaError_t) */
const char* gfla_error_string(int code);
/* whether the running device can execute the library (built for compute capability 9.0, sm_90a);
 * returns 0 when usable. */
int gfla_device_check(void);

/* Former debug channel of the pipelined tile kernels.  The current kernels have no pipeline barriers that could
 * time out: returns GFLA_E_NOTSUP and does nothing. */
int gfla_debug_set_buffer(void* host_mapped_u64x8);

/* Statistics: number of kernels this library has launched in this process so far (all entry points, all
 * threads; a relaxed counter that nothing inside the library reads).  bench.py reports the difference across
 * its timed region as `gpu_launches`. */
unsigned long long gfla_debug_launch_count(void);

/* Former wait profile of the pipelined tile kernels: returns GFLA_E_SHAPE for `which` outside [0, 2] and
 * GFLA_E_NOTSUP otherwise (the current kernels collect no profile). */
int gfla_debug_wait_profile(int which, int enable, unsigned long long* out_u64x64);

/* Re-layout of a [B,C,H,W] feature tensor between planar NCHW and channels-last NHWC storage
 * (out of place; to_nhwc = 1: NCHW -> NHWC, 0: NHWC -> NCHW).  Not part of the reference's API: the
 * Python layer uses it to serve planar bf16 / fp16 callers with the channels-last tile kernels. */
int gfla_relayout(const void* src, void* dst, int B, int C, int H, int W, int dtype, int to_nhwc,
                  gfla_stream_t stream);

/* ------------------------------------------------------------------------ *
 * block_extractor
 *   replaces block_extractor_cuda.forward(source, flow_field, output, k)
 *            block_extractor_cuda.backward(source, flow_field, grad_output,
 *                                          grad_source, grad_flow_field, k)
 *   (block_extractor/block_extractor_cuda.cc:5-33, kernels
 *    block_extractor_kernel.cu:20-85 and :89-170)
 *   source [B,C,Hs,Ws], flow [B,2,Hf,Wf] (ch0 = x, ch1 = y, in pixels)
 *   out / grad_out [B,C,k*Hf,k*Wf]; Hs,Ws may differ from Hf,Wf
 *   (external_function.py:61-66).
 * ------------------------------------------------------------------------ */
int gfla_block_extract_fwd(const void* source, const void* flow, void* out,
                           int B, int C, int Hs, int Ws, int Hf, int Wf, int k,
                           int dtype, int flow_dtype, gfla_stream_t stream);
/* grad_source_dtype: == dtype (reference contract), or GFLA_F32 when dtype is a 16-bit type: the scatter then
 * uses native fp32 red.global instead of 16-bit compare-and-swap atomics; narrow with gfla_convert(). */
int gfla_block_extract_bwd(const void* source, const void* flow, const void* grad_out,
                           void* grad_source, void* grad_flow,
                           int B, int C, int Hs, int Ws, int Hf, int Wf, int k,
                           int dtype, int flow_dtype, int grad_source_dtype, int accumulate,
                           gfla_stream_t stream);
/* element-wise dtype conversion between fp32 and bf16 / f16 (n elements, contiguous) */
int gfla_convert(const void* src, int src_dtype, void* dst, int dst_dtype, long long n, gfla_stream_t stream);

/* ------------------------------------------------------------------------ *
 * local_attn_reshape  ([B,k*k,H,W] -> [B,1,k*H,k*W], depth-to-space)
 *   replaces local_attn_reshape_cuda.forward(inputs, output, k)
 *            local_attn_reshape_cuda.backward(inputs, grad_output, grad_inputs, k)
 *   (local_attn_reshape/local_attn_reshape_cuda.cc:5-29, kernels
 *    local_attn_reshape_kernel.cu:20-61 and :65-108; `inputs` is unused by
 *    the reference backward and is not part of this signature)
 * ------------------------------------------------------------------------ */
int gfla_attn_reshape_fwd(const void* in, void* out, int B, int H, int W, int k,
                          int dtype, gfla_stream_t stream);
int gfla_attn_reshape_bwd(const void* grad_out, void* grad_in, int B, int H, int W, int k,
                          int dtype, int accumulate, gfla_stream_t stream);

/* ------------------------------------------------------------------------ *
 * resample2d  (Gaussian-weighted ks x ks warp with dilation)
 *   replaces resample2d_cuda.forward(input1, input2, output, ks, dilation)
 *            resample2d_cuda.backward(input1, input2, gradOutput,
 *                                     gradInput1, gradInput2, ks, dilation)
 *   (resample2d_package/resample2d_cuda.cc:6-33, kernels
 *    resample2d_kernel.cu:20-95, :98-202, :204-330)
 *   in1 [B,C,Hi,Wi]; in2 [B,3,H,W] = (dx, dy, sigma) -- the sigma plane is
 *   appended by the Python module (resample2d.py:51-52); out [B,C,H,W];
 *   grad_in2 [B,3,H,W] (all three planes are written, like :328).
 *   in2 / grad_in2 have the same dtype as in1 (F32 or F64 only; 16-bit
 *   feature maps: gfla_resample2d16_*, below).
 * ------------------------------------------------------------------------ */
int gfla_resample2d_fwd(const void* in1, const void* in2, void* out,
                        int B, int C, int Hi, int Wi, int H, int W, int ks, int dilation,
                        int dtype, gfla_stream_t stream);
int gfla_resample2d_bwd(const void* in1, const void* in2, const void* grad_out,
                        void* grad_in1, void* grad_in2,
                        int B, int C, int Hi, int Wi, int H, int W, int ks, int dilation,
                        int dtype, int accumulate, gfla_stream_t stream);

/* ------------------------------------------------------------------------ *
 * resample2d -> cosine similarity, fused  (SURVEY row f4)
 *   replaces, in PerceptualCorrectness.calculate_loss
 *   (model/networks/external_function.py:275-279),
 *       input_sample      = Resample2d(4, 1, sigma=2)(source_vgg, flow)   # resample2d_cuda.forward
 *       correction_sample = F.cosine_similarity(input_sample, target_all) # over the channel axis
 *   and their backward (resample2d_cuda.backward + ATen) by one kernel each
 *   way; the warped feature tensor [B,C,H,W] is never written.
 *   in1 = source features [B,C,Hi,Wi]; in2 [B,3,H,W] as for resample2d;
 *   target [B,C,H,W]; cos_out [B,H,W];
 *   cos = sum_c (v_c / max(|v|,eps)) * (t_c / max(|t|,eps))   (ATen, eps = 1e-8 in the reference call);
 *   stats [B,3,H,W] = (v.t, |v|, |t|), written by the forward and read by the backward.
 *   Backward: grad_cos [B,H,W] -> grad_in2 [B,3,H,W] (always);
 *   grad_target [B,C,H,W] optional (NULL = not wanted);
 *   grad_in1 [B,C,Hi,Wi] optional -- it needs grad_val, a caller-provided
 *   [B,C,H,W] scratch tensor that receives d/d(warped) before the scatter.
 *   accumulate applies to grad_in1 / grad_in2 / grad_target.  F32 or F64.
 * ------------------------------------------------------------------------ */
int gfla_resample2d_cosine_fwd(const void* in1, const void* in2, const void* target,
                               void* cos_out, void* stats,
                               int B, int C, int Hi, int Wi, int H, int W, int ks, int dilation,
                               double eps, int dtype, gfla_stream_t stream);
int gfla_resample2d_cosine_bwd(const void* in1, const void* in2, const void* target,
                               const void* stats, const void* grad_cos,
                               void* grad_in1, void* grad_in2, void* grad_val, void* grad_target,
                               int B, int C, int Hi, int Wi, int H, int W, int ks, int dilation,
                               double eps, int dtype, int accumulate, gfla_stream_t stream);

/* ------------------------------------------------------------------------ *
 * resample2d and resample2d -> cosine on 16-bit feature maps
 *   Same operations, shapes and arguments as the four entry points above, for
 *   dtype = GFLA_BF16 or GFLA_F16 (anything else: GFLA_E_DTYPE).
 *   In dtype: in1, out, grad_out, target, cos_out, grad_cos, grad_target.
 *   In fp32: in2 (dx, dy, sigma), grad_in2, stats, grad_in1 and grad_val.
 *   A call computes exactly what the F32 entry point computes on the widened
 *   16-bit inputs (the taps are decided in fp32, all arithmetic is fp32) and
 *   rounds each dtype output once, at its store.  grad_in1 is scattered with
 *   fp32 atomics into the fp32 buffer, as in the F32 call (no 16-bit atomics);
 *   the caller narrows it once, e.g. with gfla_convert.  With accumulate = 1 a
 *   dtype grad_target is widened, added to in fp32 and rounded once.
 * ------------------------------------------------------------------------ */
int gfla_resample2d16_fwd(const void* in1, const void* in2_f32, void* out,
                          int B, int C, int Hi, int Wi, int H, int W, int ks, int dilation,
                          int dtype, gfla_stream_t stream);
int gfla_resample2d16_bwd(const void* in1, const void* in2_f32, const void* grad_out,
                          void* grad_in1_f32, void* grad_in2_f32,
                          int B, int C, int Hi, int Wi, int H, int W, int ks, int dilation,
                          int dtype, int accumulate, gfla_stream_t stream);
int gfla_resample2d16_cosine_fwd(const void* in1, const void* in2_f32, const void* target,
                                 void* cos_out, void* stats_f32,
                                 int B, int C, int Hi, int Wi, int H, int W, int ks, int dilation,
                                 double eps, int dtype, gfla_stream_t stream);
int gfla_resample2d16_cosine_bwd(const void* in1, const void* in2_f32, const void* target,
                                 const void* stats_f32, const void* grad_cos,
                                 void* grad_in1_f32, void* grad_in2_f32, void* grad_val_f32, void* grad_target,
                                 int B, int C, int Hi, int Wi, int H, int W, int ks, int dilation,
                                 double eps, int dtype, int accumulate, gfla_stream_t stream);

/* ------------------------------------------------------------------------ *
 * fused local attention = the tail of ExtractorAttn.forward
 *   (base_function.py:804-810 with softmax=True, generator.py:112):
 *     out = avg_pool2d( LocalAttnReshape(Softmax_dim1(logits)) *
 *                       BlockExtractor(k)(source, flow), k, k )
 *   computed without materialising the [B,C,k*H,k*W] block tensor.
 *   source [B,C,Hs,Ws]; flow [B,2,H,W]; logits [B,k*k,H,W] (pre-softmax);
 *   out [B,C,H,W]; probs (optional, may be NULL) [B,k*k,H,W] receives the
 *   softmax, i.e. what hook_attn_param returns (base_function.py:812-818).
 *   Backward: grad_source follows `accumulate`; grad_flow [B,2,H,W] and
 *   grad_logits [B,k*k,H,W] likewise.
 *   `layout`: GFLA_NCHW (the reference's contiguous layout) or GFLA_NHWC (channels-last: every
 *           source position is 2*C contiguous bytes -- the layout the tile kernels are fastest on).
 *   `algo`: 0 = automatic choice, 1 = CUDA-core gather kernel,
 *           2 = tensor-core tile kernel (GFLA_E_NOTSUP if it cannot serve the call).
 * ------------------------------------------------------------------------ */
int gfla_local_attn_fwd(const void* source, const void* flow, const void* logits,
                        void* out, void* probs,
                        int B, int C, int Hs, int Ws, int H, int W, int k,
                        int dtype, int flow_dtype, int layout, int algo, gfla_stream_t stream);
/* Same forward with the caller's mask blend fused into the store (SURVEY 8(f2); generator.py:130,
 * `out = out*(1-mask) + out_attn*mask`, and the two-branch sum at generator.py:496-498):
 *     out = prev * (1 - mask) + local_attention(source, flow, logits) * mask
 * prev [B,C,H,W] (same dtype/layout as out; may alias nothing), mask [B,1,H,W] planar, same dtype.
 * Forward only (inference): training code keeps the unfused blend so autograd sees it. */
int gfla_local_attn_blend_fwd(const void* source, const void* flow, const void* logits,
                              const void* prev, const void* mask, void* out,
                              int B, int C, int Hs, int Ws, int H, int W, int k,
                              int dtype, int flow_dtype, int layout, int algo, gfla_stream_t stream);
int gfla_local_attn_bwd(const void* source, const void* flow, const void* logits,
                        const void* grad_out,
                        void* grad_source, void* grad_flow, void* grad_logits,
                        int B, int C, int Hs, int Ws, int H, int W, int k,
                        int dtype, int flow_dtype, int layout, int accumulate, int algo,
                        gfla_stream_t stream);
/* The same backward with a caller-provided scratch buffer (DEVICE memory, >= gfla_local_attn_bwd_workspace_bytes(B) bytes).
 * The size is 0, the buffer is ignored and the call behaves exactly like gfla_local_attn_bwd, whose tile kernel takes its
 * scratch from the library's own pool (see Conventions).  Kept so that callers written against ABI version 1 keep linking. */
long long gfla_local_attn_bwd_workspace_bytes(int B);
int gfla_local_attn_bwd_ws(const void* source, const void* flow, const void* logits,
                           const void* grad_out,
                           void* grad_source, void* grad_flow, void* grad_logits,
                           int B, int C, int Hs, int Ws, int H, int W, int k,
                           int dtype, int flow_dtype, int layout, int accumulate, int algo,
                           void* workspace, long long workspace_bytes, gfla_stream_t stream);

/* ------------------------------------------------------------------------ *
 * patch convolution = the source half of ExtractorAttn's first conv
 *   replaces, in ExtractorAttn.forward (base_function.py:800,805,807),
 *       block_source = BlockExtractor(k)(source, flow)                  # block_extractor_kernel.cu:20-85
 *       conv2d(cat(block_target, block_source), W, stride=k)           # the input channels of block_source
 *   and their backward (block_extractor_kernel.cu:89-170 + the conv's) by an implicit GEMM on the tensor cores:
 *       out = conv2d(BlockExtractor(k)(source, flow), weight, None, stride=k)
 *   computed without writing the [B,C,k*H,k*W] block tensor or its gradient.
 *   source [B,C,Hs,Ws] channels-last (layout must be GFLA_NHWC); flow [B,2,H,W] planar;
 *   weight [N][k][k][C] (the storage of a torch.channels_last [N,C,k,k] tensor); out [B,N,H,W] channels-last.
 *   Served: dtype GFLA_BF16 with flow_dtype GFLA_F32, C % 64 == 0, N == 128 (GFLA_E_DTYPE / GFLA_E_NOTSUP otherwise).
 *   source, weight, out, grad_out and the fp32 buffers must be 16-byte aligned.
 *   Backward: grad_out [B,N,H,W] channels-last; grad_source_f32 [B,C,Hs,Ws] channels-last fp32 and
 *   grad_weight_f32 [N][k][k][C] fp32 (narrow each with gfla_convert); grad_flow [B,2,H,W] fp32, written without
 *   atomics (deterministic).  All three follow `accumulate`.
 * ------------------------------------------------------------------------ */
int gfla_patch_conv_fwd(const void* source, const void* flow, const void* weight, void* out,
                        int B, int C, int Hs, int Ws, int H, int W, int k, int N,
                        int dtype, int flow_dtype, int layout, gfla_stream_t stream);
int gfla_patch_conv_bwd(const void* source, const void* flow, const void* weight, const void* grad_out,
                        void* grad_source_f32, void* grad_flow, void* grad_weight_f32,
                        int B, int C, int Hs, int Ws, int H, int W, int k, int N,
                        int dtype, int flow_dtype, int layout, int accumulate, gfla_stream_t stream);

/* ------------------------------------------------------------------------ *
 * deterministic backward passes  (torch.use_deterministic_algorithms(True))
 *   The same gradients as gfla_local_attn_bwd, gfla_block_extract_bwd and gfla_patch_conv_bwd, bit-identical from call
 *   to call and independent of the batch composition: each scattered gradient (grad_source, and grad_weight of the
 *   patch convolution) is summed as 64-bit fixed point with one power-of-two scale per image (per call for
 *   grad_weight) derived on the device from max|grad_out| and a proved bound, then rounded once to `dtype`.
 *   The other gradients (grad_flow, grad_logits) are written per pixel as in the default entry points.
 *   - workspace: caller-owned DEVICE memory of at least *_det_workspace_bytes(...) bytes, 16-byte aligned; its
 *     contents on entry do not matter (the call zero-fills what it uses).  NULL: GFLA_E_NULL; misaligned:
 *     GFLA_E_ALIGN; too small: GFLA_E_SHAPE (nothing is launched in each case).  The *_workspace_bytes queries
 *     return a negative GFLA_E_* code for bad sizes.
 *   - a non-finite value among the inputs of an image's bound (grad_out; for the patch convolution also the weight and,
 *     for grad_weight, the source) makes every fixed-point output of that image (of the call, for grad_weight) NaN.
 *   - an image whose grad_out is all zero gets exactly zero (plus the caller's value with accumulate = 1).
 *   - a partial that is non-finite for another reason (NaN or Inf logits, flow or source) is not made sticky: it
 *     converts to INT64_MIN and the sums it lands in are meaningless (not necessarily NaN).
 *   - the results do not depend on the SM count: no launch shape of these entry points follows it.
 *   gfla_block_extract_bwd_det: grad_source has the data dtype (no fp32 variant: the sum is rounded once anyway).
 *   gfla_patch_conv_bwd_det: grad_source [B,Hs,Ws,C] and grad_weight [N][k][k][C] in `dtype` (channels-last storage).
 * ------------------------------------------------------------------------ */
long long gfla_local_attn_bwd_det_workspace_bytes(int B, int C, int Hs, int Ws, int H, int W, int k);
int gfla_local_attn_bwd_det(const void* source, const void* flow, const void* logits,
                            const void* grad_out,
                            void* grad_source, void* grad_flow, void* grad_logits,
                            int B, int C, int Hs, int Ws, int H, int W, int k,
                            int dtype, int flow_dtype, int layout, int accumulate, int algo,
                            void* workspace, long long workspace_bytes, gfla_stream_t stream);
long long gfla_block_extract_bwd_det_workspace_bytes(int B, int C, int Hs, int Ws, int Hf, int Wf, int k);
int gfla_block_extract_bwd_det(const void* source, const void* flow, const void* grad_out,
                               void* grad_source, void* grad_flow,
                               int B, int C, int Hs, int Ws, int Hf, int Wf, int k,
                               int dtype, int flow_dtype, int accumulate,
                               void* workspace, long long workspace_bytes, gfla_stream_t stream);
long long gfla_patch_conv_bwd_det_workspace_bytes(int B, int C, int Hs, int Ws, int H, int W, int k, int N);
int gfla_patch_conv_bwd_det(const void* source, const void* flow, const void* weight, const void* grad_out,
                            void* grad_source, void* grad_flow, void* grad_weight,
                            int B, int C, int Hs, int Ws, int H, int W, int k, int N,
                            int dtype, int flow_dtype, int layout, int accumulate,
                            void* workspace, long long workspace_bytes, gfla_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* GFLA_WARP_H_ */
