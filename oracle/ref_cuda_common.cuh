/*
 * TEST INFRASTRUCTURE ONLY.
 * Launch helpers for the reference's CUDA kernel bodies compiled for sm_90a (oracle/_ref/libgfla_ref_cuda.so):
 * the same extracted text as the host build (oracle/Makefile), this time through nvcc, behind plain
 * extern "C" launchers that take device pointers -- no ATen.  Geometry = the reference launchers'
 * <<<ceil(n/256), 256, 0, stream>>> with `int n` (block_extractor_kernel.cu:172-217, 222-278;
 * local_attn_reshape_kernel.cu:110-195; resample2d_kernel.cu:335-454), so callers must keep n < 2^31
 * like the reference does (chunk the batch).  Used as (i) a GPU-side oracle at full cfg2 size and
 * (ii) bench.py's "reference CUDA kernels, recompiled" baseline.  Never linked by the product.
 */
#pragma once
#include <cuda_runtime.h>

static inline long4 contig_stride(long b, long c, long d) { return make_long4(b * c * d, c * d, d, 1); }
static inline int ref_cuda_status() { return (int)cudaGetLastError(); }
#define REF_GRID(n) dim3((unsigned)(((n) + 255) / 256)), dim3(256), 0, (cudaStream_t)stream
#define REF_FITS_INT(n) do { if ((n) <= 0 || (n) > 2147483647L) return -2; } while (0)
