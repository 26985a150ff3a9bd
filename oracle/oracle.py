"""TEST INFRASTRUCTURE ONLY -- numpy/ctypes bindings for the two CPU checkers.

* ``Oracle``  : ``oracle/_build/liboracle.so`` -- our C restatement of the
  reference arithmetic (``gfla_oracle_impl.h``; every function cites the
  reference file:line it follows).
* ``Ref``     : ``oracle/_ref/libgfla_ref.so`` -- the reference's own CUDA
  kernel bodies compiled for the host behind ``ref_shim.h`` (built only where
  ``/root/reference`` exists; the built library travels to the GPU box).

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s
``cpu_baseline`` / ``--impl reference`` legs import this module.  Nothing in
the product package (``global-flow-local-attention_b200``) does.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_SO = os.path.join(_HERE, "_build", "liboracle.so")
REF_SO = os.path.join(_HERE, "_ref", "libgfla_ref.so")
_SFX = {np.dtype(np.float32): "f32", np.dtype(np.float64): "f64"}


def build(ref: bool | None = None) -> None:
    """Compile the checkers (``make oracle`` and, where possible, ``make ref``)."""
    subprocess.check_call(["make", "-s", "-C", _HERE, "oracle"])
    if ref is None:
        ref = os.path.isdir("/root/reference/model/networks")
    if ref:
        subprocess.check_call(["make", "-s", "-C", _HERE, "ref"])
        import shutil
        if shutil.which("nvcc") or os.path.exists("/usr/local/cuda/bin/nvcc"):
            # the same extracted text through nvcc (sm_90a): GPU-side oracle + "reference CUDA kernels, recompiled" baseline
            subprocess.check_call(["make", "-s", "-C", _HERE, "refcuda"])


def have_ref() -> bool:
    return os.path.exists(REF_SO)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _chk(*arrs):
    dt = arrs[0].dtype
    for a in arrs:
        assert a.dtype == dt and a.flags["C_CONTIGUOUS"], "oracle wants contiguous arrays of one dtype"
    return _SFX[np.dtype(dt)]


class _Lib:
    prefix = ""

    def __init__(self, path):
        if not os.path.exists(path):
            raise FileNotFoundError(f"{path} is not built (python -c 'import oracle.oracle as o; o.build()')")
        self.lib = ctypes.CDLL(path)

    def _fn(self, name, sfx):
        f = getattr(self.lib, f"{self.prefix}{name}_{sfx}")
        f.restype = None
        return f

    # ---- block_extractor ------------------------------------------------
    def block_extract_fwd(self, source, flow, k):
        sfx = _chk(source, flow)
        B, C, Hs, Ws = source.shape
        _, two, Hf, Wf = flow.shape
        assert two == 2
        out = np.zeros((B, C, k * Hf, k * Wf), source.dtype)
        self._fn("block_extract_fwd", sfx)(_p(source), _p(flow), _p(out), B, C, Hs, Ws, Hf, Wf, k)
        return out

    def block_extract_bwd(self, source, flow, grad_out, k):
        sfx = _chk(source, flow, grad_out)
        B, C, Hs, Ws = source.shape
        _, _, Hf, Wf = flow.shape
        gs, gf = np.zeros_like(source), np.zeros_like(flow)
        self._fn("block_extract_bwd", sfx)(_p(source), _p(flow), _p(grad_out), _p(gs), _p(gf), B, C, Hs, Ws, Hf, Wf, k)
        return gs, gf

    # ---- resample2d -------------------------------------------------------
    def resample2d_fwd(self, in1, in2, ks, dil):
        sfx = _chk(in1, in2)
        B, C, Hi, Wi = in1.shape
        _, three, H, W = in2.shape
        assert three == 3
        out = np.zeros((B, C, H, W), in1.dtype)
        self._fn("resample2d_fwd", sfx)(_p(in1), _p(in2), _p(out), B, C, Hi, Wi, H, W, ks, dil)
        return out

    def resample2d_bwd(self, in1, in2, grad_out, ks, dil):
        sfx = _chk(in1, in2, grad_out)
        B, C, Hi, Wi = in1.shape
        _, _, H, W = in2.shape
        g1, g2 = np.zeros_like(in1), np.zeros_like(in2)
        self._fn("resample2d_bwd_input1", sfx)(_p(in1), _p(in2), _p(grad_out), _p(g1), B, C, Hi, Wi, H, W, ks, dil)
        self._fn("resample2d_bwd_input2", sfx)(_p(in1), _p(in2), _p(grad_out), _p(g2), B, C, Hi, Wi, H, W, ks, dil)
        return g1, g2


class Oracle(_Lib):
    """Our restatement (sequential C)."""
    prefix = "oracle_"

    def __init__(self):
        super().__init__(ORACLE_SO)

    def attn_reshape_fwd(self, x, k):
        sfx = _chk(x)
        B, K, H, W = x.shape
        assert K == k * k
        out = np.zeros((B, 1, k * H, k * W), x.dtype)
        self._fn("attn_reshape_fwd", sfx)(_p(x), _p(out), B, H, W, k)
        return out

    def attn_reshape_bwd(self, x, grad_out, k):
        sfx = _chk(x, grad_out)
        B, K, H, W = x.shape
        gi = np.zeros_like(x)
        self._fn("attn_reshape_bwd", sfx)(_p(grad_out), _p(gi), B, H, W, k)
        return gi

    def local_attn_fwd(self, source, flow, logits, k, return_probs=False):
        sfx = _chk(source, flow, logits)
        B, C, Hs, Ws = source.shape
        _, _, H, W = flow.shape
        assert logits.shape == (B, k * k, H, W)
        out = np.zeros((B, C, H, W), source.dtype)
        probs = np.zeros_like(logits)
        self._fn("local_attn_fwd", sfx)(_p(source), _p(flow), _p(logits), _p(out), _p(probs), B, C, Hs, Ws, H, W, k)
        return (out, probs) if return_probs else out

    def local_attn_bwd(self, source, flow, logits, grad_out, k):
        sfx = _chk(source, flow, logits, grad_out)
        B, C, Hs, Ws = source.shape
        _, _, H, W = flow.shape
        gs, gf, gl = np.zeros_like(source), np.zeros_like(flow), np.zeros_like(logits)
        self._fn("local_attn_bwd", sfx)(_p(source), _p(flow), _p(logits), _p(grad_out), _p(gs), _p(gf), _p(gl),
                                        B, C, Hs, Ws, H, W, k)
        return gs, gf, gl


class Ref(_Lib):
    """The reference's kernel bodies on the host (OpenMP over the thread index)."""
    prefix = "ref_"

    def __init__(self, threads: int | None = None):
        super().__init__(REF_SO)
        if threads is not None:
            self.set_threads(threads)

    def set_threads(self, n: int) -> None:
        self.lib.ref_set_threads(int(n))

    def max_threads(self) -> int:
        return int(self.lib.ref_max_threads())

    def attn_reshape_fwd(self, x, k):
        sfx = _chk(x)
        B, K, H, W = x.shape
        assert K == k * k
        out = np.zeros((B, 1, k * H, k * W), x.dtype)
        self._fn("attn_reshape_fwd", sfx)(_p(x), _p(out), B, H, W, k)
        return out

    def attn_reshape_bwd(self, x, grad_out, k):
        sfx = _chk(x, grad_out)
        B, K, H, W = x.shape
        gi = np.zeros_like(x)
        self._fn("attn_reshape_bwd", sfx)(_p(x), _p(grad_out), _p(gi), B, H, W, k)
        return gi
