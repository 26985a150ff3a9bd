"""Per-element bounds of the 16-bit resample2d and resample2d -> cosine kernels (k_resample2d16_*, csrc/resample2d.cu).

A 16-bit call computes exactly what the fp32 kernel computes on the widened 16-bit inputs and rounds each 16-bit output
once, at its store.  So the fp64 reference is evaluated on the widened inputs (the fp32 flow as given), and an output y16
of the 16-bit kernel satisfies

    |y16 - r| <= |y16 - y32| + |y32 - r| <= u16 |y32| + b32 <= u16 (|r| + b32) + b32 = (1 + u16) b32 + u16 |r|

where y32 is the fp32 kernel's value, b32 its fp32 bound (ref64_resample.bound_*) and u16 the unit roundoff of the
16-bit type.  Outputs the 16-bit kernels keep in fp32 (grad_input2, the cosine stats) have the fp32 bound itself.
"""
import numpy as np

import ref64


def round16(x, kind):
    """x rounded to nearest-even in the 16-bit type ('bf16' or 'fp16'), returned widened to fp32"""
    with np.errstate(over="ignore"):                       # fp16: beyond 65504 the rounding is an infinity
        r = ref64.round_bf16(x) if kind == "bf16" else ref64.round_fp16(x)
    return r.astype(np.float32)


def bound16(b32, r, kind):
    """bound of an fp32 result with bound b32 around the reference r after one rounding to the 16-bit type"""
    u, eta = ref64.storage(kind)
    return ((1 + u) * b32         # the fp32 kernel's own error, and the 16-bit rounding of that error
            + u * np.abs(r)       # the one rounding of the fp32 value: the 16-bit store in rs_fwd / rs_cos_fwd / rs_cos_bwd
            + eta)                # (out, cos, grad_target) or gfla_convert of the fp32 grad_input1 buffer; eta: fp16's
                                  # subnormal range, where a rounding is off by half the spacing, not by u of the value


MAX16 = {"bf16": float(np.finfo(np.float32).max), "fp16": 65504.0}


def check16(name, y, r, b32, kind):
    """ref64.check of a 16-bit output y against bound16.  Where the reference lies beyond the 16-bit type's largest finite
    value (fp16's 65504: where a norm of the cosine is clamped to eps its gradients reach ~1e7), the store overflows:
    there y must be the infinity of the reference's sign, and the element is not checked against the bound."""
    y, r = np.asarray(y, np.float64), np.asarray(r, np.float64)
    over = np.abs(r) * (1 + ref64.storage(kind)[0]) + b32 > MAX16[kind]
    if over.any():
        edge = np.abs(r) > MAX16[kind] * (1 + ref64.storage(kind)[0])      # certainly rounded to infinity
        assert (np.isinf(y[edge]) & (np.sign(y[edge]) == np.sign(r[edge]))).all(), f"{name}: overflow is not an infinity"
    return ref64.check(name, np.where(over, r, y), r, bound16(b32, r, kind))
