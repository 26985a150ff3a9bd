"""Thin torch-tensor front end of the C ABI: pointer / size / stream plumbing only.

Every function here checks what the reference's autograd Functions check
(contiguity asserts: block_extractor.py:9-10, local_attn_reshape.py:9,
resample2d.py:10-11; `df == 2`: block_extractor.py:16; `ds == k*k`:
local_attn_reshape.py:13; CPU tensors -> NotImplementedError:
block_extractor.py:23-24, local_attn_reshape.py:20-21) and then hands raw
device pointers to libgfla_warp.so on the caller's current stream.

Under torch.use_deterministic_algorithms(True), read when a backward runs, the backward passes that scatter a gradient
(local attention, block_extractor, patch convolution) run their deterministic variants (the *_det entry points: 64-bit
fixed-point sums, bit-identical from run to run and independent of the batch composition); the resample2d backward,
which has none, raises (warns with warn_only=True) like PyTorch's own ops.
"""
from __future__ import annotations

import contextlib
import threading
import warnings

import torch

from . import _lib

_DT = {torch.float32: _lib.GFLA_F32, torch.float64: _lib.GFLA_F64,
       torch.bfloat16: _lib.GFLA_BF16, torch.float16: _lib.GFLA_F16}


def _dt(t: torch.Tensor) -> int:
    try:
        return _DT[t.dtype]
    except KeyError:
        raise TypeError(f"unsupported dtype {t.dtype} (float32/float64, or bfloat16/float16 storage)") from None


def _need_cuda(*ts: torch.Tensor) -> None:
    for t in ts:
        if not t.is_cuda:
            # same behaviour as the reference ops: there is no CPU implementation
            raise NotImplementedError("GFLA warp ops are CUDA-only (sm_90a); got a CPU tensor")
    dev = ts[0].device
    for t in ts:
        if t.device != dev:
            raise ValueError("all tensors must live on the same CUDA device")


def _stream(t: torch.Tensor) -> int:
    return torch.cuda.current_stream(t.device).cuda_stream


def _p(t):
    return None if t is None else t.data_ptr()


# --------------------------------------------------------------------------- deterministic mode
def alert_not_deterministic(caller: str) -> None:
    """What PyTorch's ops do without a deterministic implementation: raise under torch.use_deterministic_algorithms(True),
    warn instead with warn_only=True, nothing otherwise."""
    if not torch.are_deterministic_algorithms_enabled():
        return
    msg = (f"{caller} does not have a deterministic implementation, but you set 'torch.use_deterministic_algorithms(True)'. "
           "You can turn off determinism just for this operation, or you can use the 'warn_only=True' option, if that's "
           "acceptable for your application.")
    if torch.is_deterministic_algorithms_warn_only_enabled():
        warnings.warn(msg, UserWarning, stacklevel=3)
    else:
        raise RuntimeError(msg)


_FILL_LOCK = threading.Lock()


@contextlib.contextmanager
def _no_fill():
    """In deterministic mode torch.empty fills new memory with NaN (torch.utils.deterministic.fill_uninitialized_memory).
    What is allocated inside is written in full by the library (outputs), or zero-filled by the call that uses it
    (workspaces), so that fill would only cost a pass over memory.  The setting is process-wide and autograd runs
    backward passes on one thread per device: the lock keeps two of these blocks from interleaving, so each restores
    the value it found."""
    ud = torch.utils.deterministic
    with _FILL_LOCK:
        prev = ud.fill_uninitialized_memory
        ud.fill_uninitialized_memory = False
        try:
            yield
        finally:
            ud.fill_uninitialized_memory = prev


def _workspace(nbytes: int, device) -> torch.Tensor:
    """caller-owned workspace of a *_det entry point (torch's caching allocator: 512-byte aligned, and it shows up in
    torch.cuda's memory statistics)"""
    if nbytes < 0:
        raise _lib.GflaError(f"workspace query failed with code {nbytes}: {_lib.lib().gfla_error_string(nbytes).decode()}")
    with _no_fill():
        return torch.empty(nbytes, dtype=torch.uint8, device=device)


# --------------------------------------------------------------------------- block_extractor
def block_extract_fwd(source: torch.Tensor, flow: torch.Tensor, k: int) -> torch.Tensor:
    assert source.is_contiguous() and flow.is_contiguous()
    bs, ds, hs, ws = source.size()
    bf, df, hf, wf = flow.size()
    assert df == 2
    _need_cuda(source, flow)
    out = source.new_empty((bs, ds, k * hf, k * wf))   # fully written by the kernel: no zero fill needed
    with torch.cuda.device_of(source):
        _lib.check(_lib.lib().gfla_block_extract_fwd(_p(source), _p(flow), _p(out), bs, ds, hs, ws, hf, wf, k,
                                                     _dt(source), _dt(flow), _stream(source)), "block_extract_fwd")
    return out


def convert(t: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """fp32 <-> bf16/f16 copy with the library's kernel (contiguous tensors)."""
    assert t.is_contiguous()
    out = torch.empty_like(t, dtype=dtype)
    with torch.cuda.device_of(t):
        _lib.check(_lib.lib().gfla_convert(_p(t), _dt(t), _p(out), _DT[dtype], t.numel(), _stream(t)), "convert")
    return out


def block_extract_bwd(source, flow, grad_out, k, grad_source=None, grad_flow=None):
    """Returns (grad_source, grad_flow).  If buffers are passed, gradients are ADDED
    into them (reference contract, block_extractor.py:35-40)."""
    assert source.is_contiguous() and flow.is_contiguous()
    grad_out = grad_out.contiguous()
    _need_cuda(source, flow, grad_out)
    if torch.are_deterministic_algorithms_enabled():
        return _block_extract_bwd_det(source, flow, grad_out, k, grad_source, grad_flow)
    bs, ds, hs, ws = source.size()
    _, _, hf, wf = flow.size()
    accumulate, narrow, flow_in = 1, False, flow
    if grad_source is None:
        accumulate = 0
        # 16-bit storage: scatter into an fp32 buffer (native red.global.f32; a 16-bit scalar atomicAdd is a
        # compare-and-swap loop, ~50x slower) and narrow afterwards
        narrow = source.dtype in (torch.bfloat16, torch.float16)
        grad_source = torch.empty(source.shape, dtype=torch.float32 if narrow else source.dtype, device=source.device)
        # 16-bit flow: the kernel adds one partial grad_flow per channel slice, and in a 16-bit buffer each add would
        # round.  Run on an fp32 copy of the flow (the kernel widens the flow to fp32 anyway, so the taps are the same)
        # and round the gradient once.
        if flow.dtype in (torch.bfloat16, torch.float16):
            flow_in = convert(flow, torch.float32)
        grad_flow = torch.empty_like(flow_in)
    with torch.cuda.device_of(source):
        _lib.check(_lib.lib().gfla_block_extract_bwd(_p(source), _p(flow_in), _p(grad_out), _p(grad_source), _p(grad_flow),
                                                     bs, ds, hs, ws, hf, wf, k, _dt(source), _dt(flow_in), _dt(grad_source),
                                                     accumulate, _stream(source)), "block_extract_bwd")
    if narrow:
        grad_source = convert(grad_source, source.dtype)
    if flow_in is not flow:
        grad_flow = convert(grad_flow, flow.dtype)
    return grad_source, grad_flow


def _block_extract_bwd_det(source, flow, grad_out, k, grad_source, grad_flow):
    """grad_source summed in fixed point and rounded once to the source dtype (no fp32 buffer to narrow); grad_flow in one
    channel slice, written once per element in the flow's dtype (no fp32 copy of a 16-bit flow needed)"""
    bs, ds, hs, ws = source.size()
    _, _, hf, wf = flow.size()
    accumulate = 1
    if grad_source is None:
        accumulate = 0
        with _no_fill():
            grad_source, grad_flow = torch.empty_like(source), torch.empty_like(flow)
    elif grad_source.dtype != source.dtype or grad_flow.dtype != flow.dtype:
        # the sums are rounded once, into the source's (flow's) dtype: a wider buffer would only add a second rounding
        raise TypeError(f"deterministic block_extract backward: grad_source / grad_flow must have the dtypes of source / "
                        f"flow ({source.dtype} / {flow.dtype}), got {grad_source.dtype} / {grad_flow.dtype}")
    l = _lib.lib()
    nb = l.gfla_block_extract_bwd_det_workspace_bytes(bs, ds, hs, ws, hf, wf, k)
    wsp = _workspace(nb, source.device)
    with torch.cuda.device_of(source):
        _lib.check(l.gfla_block_extract_bwd_det(_p(source), _p(flow), _p(grad_out), _p(grad_source), _p(grad_flow), bs, ds, hs, ws,
                                                hf, wf, k, _dt(source), _dt(flow), accumulate, _p(wsp), nb, _stream(source)),
                   "block_extract_bwd_det")
    return grad_source, grad_flow


# --------------------------------------------------------------------------- local_attn_reshape
def attn_reshape_fwd(inputs: torch.Tensor, k: int) -> torch.Tensor:
    assert inputs.is_contiguous()
    bs, ds, hs, ws = inputs.size()
    assert ds == k * k
    _need_cuda(inputs)
    out = inputs.new_empty((bs, 1, k * hs, k * ws))
    with torch.cuda.device_of(inputs):
        _lib.check(_lib.lib().gfla_attn_reshape_fwd(_p(inputs), _p(out), bs, hs, ws, k, _dt(inputs), _stream(inputs)),
                   "attn_reshape_fwd")
    return out


def attn_reshape_bwd(grad_out: torch.Tensor, k: int, grad_in=None) -> torch.Tensor:
    grad_out = grad_out.contiguous()
    _need_cuda(grad_out)
    bs, _, ho, wo = grad_out.size()
    hs, ws = ho // k, wo // k
    accumulate = 1
    if grad_in is None:
        grad_in, accumulate = grad_out.new_empty((bs, k * k, hs, ws)), 0
    with torch.cuda.device_of(grad_out):
        _lib.check(_lib.lib().gfla_attn_reshape_bwd(_p(grad_out), _p(grad_in), bs, hs, ws, k, _dt(grad_out), accumulate,
                                                    _stream(grad_out)), "attn_reshape_bwd")
    return grad_in


# --------------------------------------------------------------------------- resample2d
def resample2d_fwd(input1: torch.Tensor, input2: torch.Tensor, kernel_size: int, dilation: int) -> torch.Tensor:
    assert input1.is_contiguous() and input2.is_contiguous()
    _need_cuda(input1, input2)
    _, d, hi, wi = input1.size()
    b, three, h, w = input2.size()
    assert three == 3, "input2 must be [B,3,H,W] = (dx, dy, sigma) (resample2d.py:51-52)"
    if input2.dtype != input1.dtype:
        raise TypeError("resample2d: input1 and input2 must share a dtype (float32 or float64)")
    out = input1.new_empty((b, d, h, w))
    with torch.cuda.device_of(input1):
        _lib.check(_lib.lib().gfla_resample2d_fwd(_p(input1), _p(input2), _p(out), b, d, hi, wi, h, w, kernel_size,
                                                  dilation, _dt(input1), _stream(input1)), "resample2d_fwd")
    return out


def resample2d_bwd(input1, input2, grad_out, kernel_size, dilation, grad_input1=None, grad_input2=None):
    alert_not_deterministic("resample2d backward (grad_input1 scatter)")
    assert input1.is_contiguous() and input2.is_contiguous()
    grad_out = grad_out.contiguous()
    _need_cuda(input1, input2, grad_out)
    _, d, hi, wi = input1.size()
    b, _, h, w = input2.size()
    accumulate = 1
    if grad_input1 is None:
        grad_input1, grad_input2, accumulate = torch.empty_like(input1), torch.empty_like(input2), 0
    with torch.cuda.device_of(input1):
        _lib.check(_lib.lib().gfla_resample2d_bwd(_p(input1), _p(input2), _p(grad_out), _p(grad_input1), _p(grad_input2),
                                                  b, d, hi, wi, h, w, kernel_size, dilation, _dt(input1), accumulate,
                                                  _stream(input1)), "resample2d_bwd")
    return grad_input1, grad_input2


def resample2d_cosine_fwd(input1, input2, target, kernel_size: int, dilation: int, eps: float = 1e-8):
    """cos[b,y,x] = cosine_similarity(resample2d(input1, input2)[b,:,y,x], target[b,:,y,x]) without the warped tensor
    (external_function.py:275-279).  -> (cos [B,H,W], stats [B,3,H,W] for the backward)"""
    assert input1.is_contiguous() and input2.is_contiguous() and target.is_contiguous()
    _need_cuda(input1, input2, target)
    _, d, hi, wi = input1.size()
    b, three, h, w = input2.size()
    assert three == 3, "input2 must be [B,3,H,W] = (dx, dy, sigma) (resample2d.py:51-52)"
    assert tuple(target.shape) == (b, d, h, w), "target must be [B,C,H,W] on the flow's grid"
    if input2.dtype != input1.dtype or target.dtype != input1.dtype:
        raise TypeError("resample2d_cosine: input1, input2 and target must share a dtype (float32 or float64)")
    cos = input1.new_empty((b, h, w))
    stats = input1.new_empty((b, 3, h, w))
    with torch.cuda.device_of(input1):
        _lib.check(_lib.lib().gfla_resample2d_cosine_fwd(_p(input1), _p(input2), _p(target), _p(cos), _p(stats), b, d, hi, wi, h, w,
                                                         kernel_size, dilation, float(eps), _dt(input1), _stream(input1)),
                   "resample2d_cosine_fwd")
    return cos, stats


def resample2d_cosine_bwd(input1, input2, target, stats, grad_cos, kernel_size, dilation, eps=1e-8, need_input1=False,
                          need_target=False):
    """-> (grad_input1 | None, grad_input2, grad_target | None)"""
    if need_input1:
        alert_not_deterministic("resample2d_cosine backward (grad_input1 scatter)")
    grad_cos = grad_cos.contiguous()
    _need_cuda(input1, input2, target, stats, grad_cos)
    _, d, hi, wi = input1.size()
    b, _, h, w = input2.size()
    grad_in2 = torch.empty_like(input2)
    grad_in1 = torch.empty_like(input1) if need_input1 else None
    grad_val = torch.empty_like(target) if need_input1 else None
    grad_target = torch.empty_like(target) if need_target else None
    with torch.cuda.device_of(input1):
        _lib.check(_lib.lib().gfla_resample2d_cosine_bwd(
            _p(input1), _p(input2), _p(target), _p(stats), _p(grad_cos), _p(grad_in1) if need_input1 else None, _p(grad_in2),
            _p(grad_val) if need_input1 else None, _p(grad_target) if need_target else None, b, d, hi, wi, h, w, kernel_size, dilation,
            float(eps), _dt(input1), 0, _stream(input1)), "resample2d_cosine_bwd")
    return grad_in1, grad_in2, grad_target


# --------------------------------------------------------------------------- fused local attention
ALGO = {"auto": 0, "gather": 1, "tile": 2}


def _feature_layout(t: torch.Tensor) -> int:
    """GFLA_NCHW for contiguous tensors, GFLA_NHWC for torch.channels_last ones (no copy either way)."""
    if t.is_contiguous():
        return _lib.GFLA_NCHW
    if t.dim() == 4 and t.is_contiguous(memory_format=torch.channels_last):
        return _lib.GFLA_NHWC
    raise AssertionError("feature tensors must be contiguous (NCHW) or channels_last")


def _like_layout(t: torch.Tensor, shape, layout: int) -> torch.Tensor:
    fmt = torch.channels_last if layout == _lib.GFLA_NHWC else torch.contiguous_format
    return torch.empty(shape, dtype=t.dtype, device=t.device, memory_format=fmt)


def local_attn_fwd(source, flow, logits, k, return_probs=False, algo="auto"):
    """source may be contiguous (NCHW) or channels_last; `out` comes back in the same memory format."""
    layout = _feature_layout(source)
    assert flow.is_contiguous() and logits.is_contiguous()
    _need_cuda(source, flow, logits)
    bs, ds, hs, ws = source.size()
    bf, df, h, w = flow.size()
    assert df == 2 and bf == bs
    assert logits.shape == (bs, k * k, h, w) and logits.dtype == source.dtype
    out = _like_layout(source, (bs, ds, h, w), layout)
    probs = torch.empty_like(logits) if return_probs else None
    with torch.cuda.device_of(source):
        _lib.check(_lib.lib().gfla_local_attn_fwd(_p(source), _p(flow), _p(logits), _p(out), _p(probs), bs, ds, hs, ws,
                                                  h, w, k, _dt(source), _dt(flow), layout, ALGO[algo], _stream(source)),
                   "local_attn_fwd")
    return (out, probs) if return_probs else out


def local_attn_blend_fwd(source, flow, logits, prev, mask, k, algo="auto"):
    """out = prev * (1 - mask) + local_attention(source, flow, logits) * mask, in one kernel (forward only).
    prev: [B,C,H,W] in the same memory format as source; mask: [B,1,H,W]."""
    layout = _feature_layout(source)
    assert _feature_layout(prev) == layout or prev.shape[1] == 1, "prev must use the same memory format as source"
    assert flow.is_contiguous() and logits.is_contiguous()
    mask = mask.contiguous()
    _need_cuda(source, flow, logits, prev, mask)
    bs, ds, hs, ws = source.size()
    _, _, h, w = flow.size()
    assert prev.shape == (bs, ds, h, w) and mask.shape == (bs, 1, h, w)
    assert prev.dtype == source.dtype and mask.dtype == source.dtype and logits.dtype == source.dtype
    out = _like_layout(source, (bs, ds, h, w), layout)
    with torch.cuda.device_of(source):
        _lib.check(_lib.lib().gfla_local_attn_blend_fwd(_p(source), _p(flow), _p(logits), _p(prev), _p(mask), _p(out), bs, ds,
                                                        hs, ws, h, w, k, _dt(source), _dt(flow), layout, ALGO[algo],
                                                        _stream(source)), "local_attn_blend_fwd")
    return out


def relayout(t: torch.Tensor, to_channels_last: bool) -> torch.Tensor:
    """Out-of-place NCHW <-> channels_last copy of a [B,C,H,W] tensor with the library's own transpose kernel."""
    _need_cuda(t)
    b, c, h, w = t.shape
    if to_channels_last:
        assert t.is_contiguous()
        out = torch.empty((b, c, h, w), dtype=t.dtype, device=t.device, memory_format=torch.channels_last)
    else:
        assert t.is_contiguous(memory_format=torch.channels_last)
        out = torch.empty((b, c, h, w), dtype=t.dtype, device=t.device)
    with torch.cuda.device_of(t):
        _lib.check(_lib.lib().gfla_relayout(_p(t), _p(out), b, c, h, w, _dt(t), 1 if to_channels_last else 0, _stream(t)),
                   "relayout")
    return out


# --------------------------------------------------------------------------- patch convolution
PATCH_CONV_N = 128


def patch_conv_eligible(source, flow, weight, k) -> bool:
    """what the patch-convolution kernels serve (mirrors patch_conv_supported in csrc/patch_conv_tc.cu; an NCHW source
    is re-laid to channels-last here)"""
    return (source.is_cuda and source.dtype == torch.bfloat16 and weight.dtype == torch.bfloat16
            and flow.dtype == torch.float32 and source.dim() == 4 and source.shape[1] % 64 == 0
            and tuple(weight.shape) == (PATCH_CONV_N, source.shape[1], k, k) and 1 <= k <= 9)


def _pack_weight(weight):
    """[N,C,k,k] -> [N][k][k][C] storage (what a channels_last weight already holds: then no copy)"""
    return weight.permute(0, 2, 3, 1).contiguous()


def patch_conv_fwd(source, flow, weight, k):
    """out = conv2d(BlockExtractor(k)(source, flow), weight, None, stride=k) [B,128,H,W] without the block tensor, in the
    source's memory format.  Only for calls patch_conv_eligible accepts."""
    assert flow.is_contiguous()
    _need_cuda(source, flow, weight)
    planar = _feature_layout(source) == _lib.GFLA_NCHW
    src = relayout(source, True) if planar else source
    bs, ds, hs, ws = source.size()
    _, df, h, w = flow.size()
    assert df == 2 and flow.shape[0] == bs
    n = weight.shape[0]
    wp = _pack_weight(weight)
    out = torch.empty((bs, h, w, n), dtype=source.dtype, device=source.device)       # channels-last storage
    with torch.cuda.device_of(source):
        _lib.check(_lib.lib().gfla_patch_conv_fwd(_p(src), _p(flow), _p(wp), _p(out), bs, ds, hs, ws, h, w, k, n, _dt(source),
                                                  _dt(flow), _lib.GFLA_NHWC, _stream(source)), "patch_conv_fwd")
    out = out.permute(0, 3, 1, 2)
    return relayout(out, False) if planar else out


def patch_conv_bwd(source, flow, weight, grad_out, k):
    """-> (grad_source, grad_flow, grad_weight).  grad_source and grad_weight are summed in fp32 buffers and rounded
    once; grad_source comes back in the source's memory format, grad_weight channels-last."""
    assert flow.is_contiguous()
    _need_cuda(source, flow, weight, grad_out)
    planar = _feature_layout(source) == _lib.GFLA_NCHW
    src = relayout(source, True) if planar else source
    if grad_out.is_contiguous(memory_format=torch.channels_last):
        go = grad_out
    else:
        go = relayout(grad_out.contiguous(), True)
    bs, ds, hs, ws = source.size()
    _, _, h, w = flow.size()
    n = weight.shape[0]
    wp = _pack_weight(weight)
    if torch.are_deterministic_algorithms_enabled():
        # grad_source and grad_weight summed in fixed point and rounded once to bf16 by the library
        with _no_fill():
            gs = torch.empty((bs, hs, ws, ds), dtype=source.dtype, device=source.device)   # channels-last storage
            gw = torch.empty((n, k, k, ds), dtype=weight.dtype, device=source.device)
            gf = torch.empty_like(flow)
        l = _lib.lib()
        nb = l.gfla_patch_conv_bwd_det_workspace_bytes(bs, ds, hs, ws, h, w, k, n)
        wsp = _workspace(nb, source.device)
        with torch.cuda.device_of(source):
            _lib.check(l.gfla_patch_conv_bwd_det(_p(src), _p(flow), _p(wp), _p(go), _p(gs), _p(gf), _p(gw), bs, ds, hs, ws, h, w, k, n,
                                                 _dt(source), _dt(flow), _lib.GFLA_NHWC, 0, _p(wsp), nb, _stream(source)),
                       "patch_conv_bwd_det")
        del wsp
        gs, gw = gs.permute(0, 3, 1, 2), gw.permute(0, 3, 1, 2)
        return (relayout(gs, False) if planar else gs), gf, gw
    gs32 = torch.empty((bs, hs, ws, ds), dtype=torch.float32, device=source.device)   # channels-last storage
    gw32 = torch.empty((n, k, k, ds), dtype=torch.float32, device=source.device)
    gf = torch.empty_like(flow)
    with torch.cuda.device_of(source):
        _lib.check(_lib.lib().gfla_patch_conv_bwd(_p(src), _p(flow), _p(wp), _p(go), _p(gs32), _p(gf), _p(gw32), bs, ds, hs, ws,
                                                  h, w, k, n, _dt(source), _dt(flow), _lib.GFLA_NHWC, 0, _stream(source)),
                   "patch_conv_bwd")
    gs = convert(gs32, source.dtype).permute(0, 3, 1, 2)
    del gs32
    gw = convert(gw32, weight.dtype).permute(0, 3, 1, 2)
    return (relayout(gs, False) if planar else gs), gf, gw


def _tile_bwd_eligible(source, flow, k) -> bool:
    """what the backward tile kernels serve (mirrors local_attn_bwd_tc_supported in csrc/local_attn_bwd_tc.cu)"""
    c = source.shape[1]
    return (source.dtype == torch.bfloat16 and flow.dtype == torch.float32 and k in (3, 5)
            and (c % 256 == 0 or c in (64, 128)))


def local_attn_bwd(source, flow, logits, grad_out, k, algo="auto"):
    layout = _feature_layout(source)
    assert flow.is_contiguous() and logits.is_contiguous()
    _need_cuda(source, flow, logits, grad_out)
    if (layout == _lib.GFLA_NCHW and algo == "auto" and _tile_bwd_eligible(source, flow, k)
            and not source.is_contiguous(memory_format=torch.channels_last)):   # H=W=1 / C=1: both formats at once
        # The backward tile kernel is channels-last only (every operand is staged as channel-contiguous 16-byte chunks).
        # For planar callers, re-lay the two feature tensors (two extra passes over them) instead of falling
        # back to the scalar-atomics kernel: ~100x faster at cfg2.
        go = grad_out if grad_out.is_contiguous() else grad_out.contiguous()
        gs, gf, gl = local_attn_bwd(relayout(source, True), flow, logits, relayout(go, True), k, algo="auto")
        return relayout(gs, False), gf, gl
    fmt = torch.channels_last if layout == _lib.GFLA_NHWC else torch.contiguous_format
    grad_out = grad_out.contiguous(memory_format=fmt)
    if torch.are_deterministic_algorithms_enabled():
        return _local_attn_bwd_det(source, flow, logits, grad_out, k, layout, algo)
    tile = layout == _lib.GFLA_NHWC and _tile_bwd_eligible(source, flow, k)
    if source.dtype in (torch.bfloat16, torch.float16) and (algo == "gather" or (algo == "auto" and not tile)):
        # The CUDA-core backward scatters grad_source with one atomic add per (pixel, tap, channel).  In a 16-bit type every
        # add rounds, and the order-dependent rounding of up to (k+1)^2 adds per element exceeds the bf16 tolerance: run it
        # on fp32 copies and round each gradient once.
        gs, gf, gl = local_attn_bwd(source.float(), flow.float(), logits.float(), grad_out.float(), k, algo="gather")
        return gs.to(source.dtype), gf.to(flow.dtype), gl.to(logits.dtype)
    bs, ds, hs, ws = source.size()
    _, _, h, w = flow.size()
    gs, gf, gl = _like_layout(source, source.shape, layout), torch.empty_like(flow), torch.empty_like(logits)
    with torch.cuda.device_of(source):
        _lib.check(_lib.lib().gfla_local_attn_bwd(_p(source), _p(flow), _p(logits), _p(grad_out), _p(gs), _p(gf), _p(gl),
                                                  bs, ds, hs, ws, h, w, k, _dt(source), _dt(flow), layout, 0, ALGO[algo],
                                                  _stream(source)), "local_attn_bwd")
    return gs, gf, gl


def _local_attn_bwd_det(source, flow, logits, grad_out, k, layout, algo):
    """grad_source summed in fixed point and rounded once to the source dtype, by the tile or the gather kernel: 16-bit
    gather calls need no fp32 copies here"""
    bs, ds, hs, ws = source.size()
    _, _, h, w = flow.size()
    with _no_fill():
        gs, gf, gl = _like_layout(source, source.shape, layout), torch.empty_like(flow), torch.empty_like(logits)
    l = _lib.lib()
    nb = l.gfla_local_attn_bwd_det_workspace_bytes(bs, ds, hs, ws, h, w, k)
    wsp = _workspace(nb, source.device)
    with torch.cuda.device_of(source):
        _lib.check(l.gfla_local_attn_bwd_det(_p(source), _p(flow), _p(logits), _p(grad_out), _p(gs), _p(gf), _p(gl), bs, ds, hs, ws, h,
                                             w, k, _dt(source), _dt(flow), layout, 0, ALGO[algo], _p(wsp), nb, _stream(source)),
                   "local_attn_bwd_det")
    return gs, gf, gl
