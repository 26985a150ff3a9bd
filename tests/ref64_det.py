"""Per-element error bounds of the deterministic backward mode (csrc/det_accum.cuh), next to ref64's bounds of the
default paths.  Each returns the bound on |y - ref| for one output element, from what that path rounds:

  * the partials, as in the default path minus its per-add roundings: fp32 products and GEMM sums (ref64.FP32_SLACK or
    gamma(n) of the magnitude), the tile kernel's bf16 window;
  * quant(n, E): each of the n partials of an element rounded to a multiple of 2^-E (llrint, det_accum.cuh fx_add):
    n 2^-(E+1);
  * the int64 -> double conversion of the sum (k_fx_narrow): 2^-53 of the magnitude;
  * one rounding to the storage type (k_fx_narrow's st_d): u |r|, plus eta.  It rounds the computed value, so it also
    scales the errors above: the 1.01 pays for that.

E is the exponent det_accum.cu derives, exponent(M) below, from the image's bound M (api.cu).
"""
import math

import numpy as np

import ref64

U_FP32, U_FP64 = 2.0 ** -24, 2.0 ** -53
INT64_TO_DOUBLE = 2.0 ** -53


def exponent(m):
    """fx_exponent (det_accum.cu): 61 - e with m < 2^e; 0 for m == 0"""
    if m == 0:
        return 0
    return max(-2000, min(2000, 61 - math.frexp(m)[1]))


def exponents(M):
    """per-image exponents of the per-image bounds M (array)"""
    return np.array([exponent(float(m)) for m in np.ravel(M)])


def quant(n, E):
    """n partials per element, each rounded to the nearest multiple of 2^-E (E broadcast per image)"""
    return np.asarray(n, np.float64) * 2.0 ** -(np.asarray(E, np.float64) + 1)


def _final(r, err, u, eta):
    return u * np.abs(r) + 1.01 * err + eta


def la_exponents(gout, H, W, k):
    """local attention, tile and gather: M_b = (H W / k^2) max|G_b| (api.cu gfla_local_attn_bwd_det)"""
    g = np.abs(np.asarray(gout, np.float64)).reshape(len(gout), -1).max(axis=1)
    return exponents(H * W / (k * k) * g)


def n_partials_la(H, W, k):
    """partials one grad_source element can receive: at most 4 k^2 per pixel (the literal path's corner taps; the
    collapsed window gives fewer), from every pixel of the image"""
    return 4 * k * k * H * W


def bound_gs_tile(r, Mgs, E, n, u, eta, init=0.0):
    """tile backward, deterministic (k_local_attn_bwd_tc<K, CN, true>): the bf16 window (tile_window.cuh build_window,
    u of each weight: u Mgs) and the fp32 MMA sums of the GS GEMM (ref64.FP32_SLACK Mgs); no per-partial bf16 rounding
    and no bf16 adds (the default path's (n_adds + 1) u Mgs); quantisation and int64 -> double; one rounding of
    r + init"""
    rr = np.asarray(r) + init
    err = (u + ref64.FP32_SLACK) * Mgs + quant(n, E) + INT64_TO_DOUBLE * (Mgs + np.abs(init))
    return _final(rr, err, u, eta)


def bound_gs_gather(r, Mgs, E, n, u, eta, slack=ref64.FP32_SLACK):
    """gather backward, deterministic (k_local_attn_bwd<T, TF, K, true>), every storage type: partials in the arithmetic
    type (fp32: ref64.FP32_SLACK Mgs; fp64: slack = 2^-49), quantisation, int64 -> double, one rounding (u = 2^-24 for
    fp32, 2^-53 for fp64 storage)"""
    err = slack * Mgs + quant(n, E) + INT64_TO_DOUBLE * Mgs
    return _final(r, err, u, eta)


def be_exponents(gout, k, Hf, Wf):
    """block_extract: M_b = k^2 Hf Wf max|G_b| (api.cu gfla_block_extract_bwd_det)"""
    g = np.abs(np.asarray(gout, np.float64)).reshape(len(gout), -1).max(axis=1)
    return exponents(k * k * Hf * Wf * g)


def bound_be_gs(r, Mgs, E, n, u, eta):
    """block_extract backward, deterministic: fp32 products g w (ref64.FP32_SLACK Mgs), n = 4 k^2 Hf Wf partials at
    most, quantisation, int64 -> double, one rounding"""
    return _final(r, ref64.FP32_SLACK * Mgs + quant(n, E) + INT64_TO_DOUBLE * Mgs, u, eta)


def pc_exponents(gout, w, src, k, H, W, n_out):
    """patch convolution: grad_source M_b = k^2 H W N max|G_b| max|W| per image; grad_weight one exponent for the call,
    B H W max|G| max|source| (api.cu gfla_patch_conv_bwd_det)"""
    g = np.abs(np.asarray(gout, np.float64)).reshape(len(gout), -1).max(axis=1)
    mw, ms = float(np.abs(w).max()), float(np.abs(src).max())
    return exponents(k * k * H * W * n_out * g * mw), exponent(len(gout) * H * W * float(g.max()) * ms)


def bound_pc_gs(r, Mgs, E, n, n_out, u, eta):
    """patch convolution grad_source, deterministic: GA = G W^T over N bf16 products in fp32 and the product with the
    corner weight (gamma(N + 1) Mgs, as the default path); no fp32 reductions into a buffer (the default's gamma(n + 1));
    quantisation of n partials, int64 -> double, one rounding"""
    return _final(r, 1.01 * ref64.gamma(n_out + 1) * Mgs + quant(n, E) + INT64_TO_DOUBLE * Mgs, u, eta)


def bound_pc_gw(r, Mgw, E, n_slices, per_slice_px, u, eta):
    """patch convolution grad_weight, deterministic: each partial is an fp32 MMA sum over one slice of per_slice_px
    pixels (gamma(per_slice_px) of its share of Mgw); n_slices partials per element quantised at the call's exponent;
    int64 -> double; one rounding"""
    return _final(r, 1.01 * ref64.gamma(per_slice_px + 1) * Mgw + quant(n_slices, E) + INT64_TO_DOUBLE * Mgw, u, eta)
