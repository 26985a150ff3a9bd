"""TEST / BASELINE INFRASTRUCTURE ONLY.

torch-tensor bindings of ``oracle/_ref/libgfla_ref_cuda.so``: the reference's own CUDA
kernels (block_extractor_kernel.cu:5-170, local_attn_reshape_kernel.cu:5-108,
resample2d_kernel.cu:5-330), extracted at build time and compiled by nvcc for sm_90a
behind the plain launchers in ``ref_cuda_*.cu`` (``make -C oracle refcuda``).

Two uses, both outside the product path:
  * a GPU-side oracle that reaches the full cfg2 size (the host build needs minutes per
    sample; this needs milliseconds) -- ``tests/test_gpu_refcuda.py``;
  * bench.py's second baseline: "the reference's CUDA kernels, recompiled for sm_90"
    (BASELINE.md section 3), i.e. the unfused ExtractorAttn tail exactly as
    base_function.py:804-810 runs it, on the same GPU.

The autograd Functions below mirror block_extractor.py:5-42 and local_attn_reshape.py:5-37
(zero-filled outputs, gradients accumulated into zero-filled buffers) and keep the
reference's limits: float / double only, ``int n`` element counts (callers chunk the batch).
"""
from __future__ import annotations

import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(_HERE, "_ref", "libgfla_ref_cuda.so")
_SFX = {torch.float32: "f32", torch.float64: "f64"}
_lib = None


def available() -> bool:
    return os.path.exists(SO)


def lib():
    global _lib
    if _lib is None:
        if not available():
            raise FileNotFoundError(f"{SO} is not built (make -C oracle refcuda; needs /root/reference)")
        _lib = ctypes.CDLL(SO)
    return _lib


def _call(name, dtype, *args):
    fn = getattr(lib(), f"refcuda_{name}_{_SFX[dtype]}")
    fn.restype = ctypes.c_int
    conv = [ctypes.c_void_p(a.data_ptr()) if isinstance(a, torch.Tensor) else a for a in args]
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    rc = fn(*conv, stream)
    if rc != 0:
        raise RuntimeError(f"refcuda_{name}: error {rc}" + (" (element count exceeds the reference's int)" if rc == -2 else ""))


def _chk(*ts):
    for t in ts:
        assert t.is_cuda and t.is_contiguous() and t.dtype == ts[0].dtype and t.dtype in _SFX


def block_extract_fwd(source, flow, k):
    _chk(source, flow)
    b, c, hs, ws = source.shape
    _, _, hf, wf = flow.shape
    out = source.new_zeros((b, c, k * hf, k * wf))                       # block_extractor.py:21
    _call("block_extract_fwd", source.dtype, source, flow, out, b, c, hs, ws, hf, wf, k)
    return out


def block_extract_bwd(source, flow, grad_out, k):
    _chk(source, flow, grad_out)
    b, c, hs, ws = source.shape
    _, _, hf, wf = flow.shape
    gs, gf = torch.zeros_like(source), torch.zeros_like(flow)            # block_extractor.py:35-36
    _call("block_extract_bwd", source.dtype, source, flow, grad_out, gs, gf, b, c, hs, ws, hf, wf, k)
    return gs, gf


def attn_reshape_fwd(x, k):
    _chk(x)
    b, kk, h, w = x.shape
    assert kk == k * k
    out = x.new_zeros((b, 1, k * h, k * w))                              # local_attn_reshape.py:18
    _call("attn_reshape_fwd", x.dtype, x, out, b, h, w, k)
    return out


def attn_reshape_bwd(x, grad_out, k):
    _chk(x, grad_out)
    b, _, h, w = x.shape
    gi = torch.zeros_like(x)
    _call("attn_reshape_bwd", x.dtype, x, grad_out, gi, b, h, w, k)
    return gi


def resample2d_fwd(in1, in2, ks, dil):
    _chk(in1, in2)
    _, c, hi, wi = in1.shape
    b, _, h, w = in2.shape
    out = in1.new_zeros((b, c, h, w))
    _call("resample2d_fwd", in1.dtype, in1, in2, out, b, c, hi, wi, h, w, ks, dil)
    return out


def resample2d_bwd(in1, in2, grad_out, ks, dil):
    _chk(in1, in2, grad_out)
    _, c, hi, wi = in1.shape
    b, _, h, w = in2.shape
    g1, g2 = torch.zeros_like(in1), torch.zeros_like(in2)
    _call("resample2d_bwd_input1", in1.dtype, in1, in2, grad_out, g1, b, c, hi, wi, h, w, ks, dil)
    _call("resample2d_bwd_input2", in1.dtype, in1, in2, grad_out, g2, b, c, hi, wi, h, w, ks, dil)
    return g1, g2


class ExtractFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, source, flow, k):
        ctx.save_for_backward(source, flow)
        ctx.k = k
        return block_extract_fwd(source, flow, k)

    @staticmethod
    def backward(ctx, g):
        s, f = ctx.saved_tensors
        gs, gf = block_extract_bwd(s, f, g.contiguous(), ctx.k)
        return gs, gf, None


class ReshapeFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, k):
        ctx.save_for_backward(x)
        ctx.k = k
        return attn_reshape_fwd(x, k)

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        return attn_reshape_bwd(x, g.contiguous(), ctx.k), None


class Resample2dFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, in1, in2, ks, dil):
        ctx.save_for_backward(in1, in2)
        ctx.ks, ctx.dil = ks, dil
        return resample2d_fwd(in1, in2, ks, dil)

    @staticmethod
    def backward(ctx, g):
        a, f = ctx.saved_tensors
        g1, g2 = resample2d_bwd(a, f, g.contiguous(), ctx.ks, ctx.dil)
        return g1, g2, None, None


def local_attn_tail(source, flow, logits, k):
    """The reference's ExtractorAttn tail (base_function.py:805,808-809 after Softmax(dim=1), :803) on its own kernels."""
    block = ExtractFn.apply(source, flow, k)
    attn = ReshapeFn.apply(torch.softmax(logits, dim=1), k)
    return torch.nn.functional.avg_pool2d(attn * block, k, k)


def local_attn_fwd_bwd(source, flow, logits, grad_out, k, chunk=None):
    """fp32/fp64 CUDA tensors in -> (out, grad_source, grad_flow, grad_logits); the batch is processed in chunks
    small enough for the reference's `int n` (block_extractor_kernel.cu:180) and for memory."""
    b, c, _, _ = source.shape
    _, _, h, w = flow.shape
    if chunk is None:
        per = c * k * h * k * w
        chunk = max(1, min(b, (2 ** 31 - 1) // per, max(1, (2 << 30) // (per * source.element_size()))))
    outs, gss, gfs, gls = [], [], [], []
    for b0 in range(0, b, chunk):
        s = source[b0:b0 + chunk].detach().clone().requires_grad_()
        f = flow[b0:b0 + chunk].detach().clone().requires_grad_()
        l = logits[b0:b0 + chunk].detach().clone().requires_grad_()
        out = local_attn_tail(s, f, l, k)
        out.backward(grad_out[b0:b0 + chunk].contiguous())
        outs.append(out.detach()); gss.append(s.grad); gfs.append(f.grad); gls.append(l.grad)
    return torch.cat(outs), torch.cat(gss), torch.cat(gfs), torch.cat(gls)
