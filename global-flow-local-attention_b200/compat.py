"""Legacy import names, so the reference's own Python runs on this library unchanged.

``install()`` registers

* ``block_extractor_cuda``, ``local_attn_reshape_cuda``, ``resample2d_cuda`` --
  modules with the reference pybind surface ``forward(...)`` / ``backward(...)``
  (block_extractor_cuda.cc:31-33, local_attn_reshape_cuda.cc:26-29,
  resample2d_cuda.cc:30-33): caller-allocated, zero-filled outputs, gradients
  accumulated, ``int`` return value 1;
* optionally ``model.networks.{block_extractor.block_extractor,
  local_attn_reshape.local_attn_reshape, resample2d_package.resample2d}`` --
  the module paths imported by base_function.py:10-13 and
  external_function.py:5-7 -- pointing at this package's classes.
"""
import sys
import types

from . import functional as F_


def _mk(name, **fns):
    m = types.ModuleType(name)
    m.__dict__.update(fns)
    m.__doc__ = f"gfla_b200 shim for the reference extension `{name}`"
    return m


def _be_forward(source, flow_field, output, kernel_size):
    F_._need_cuda(source, flow_field, output)
    b, c, hs, ws = source.shape
    _, _, hf, wf = flow_field.shape
    F_._call("block_extract_fwd", source, source.data_ptr(), flow_field.data_ptr(), output.data_ptr(), b, c, hs, ws, hf, wf,
             kernel_size, F_._dt(source), F_._dt(flow_field))
    return 1


def _be_backward(source, flow_field, grad_output, grad_source, grad_flow_field, kernel_size):
    F_.block_extract_bwd(source, flow_field, grad_output, kernel_size, grad_source, grad_flow_field)
    return 1


def _lr_forward(inputs, output, kernel_size):
    F_._need_cuda(inputs, output)
    b, _, h, w = inputs.shape
    F_._call("attn_reshape_fwd", inputs, inputs.data_ptr(), output.data_ptr(), b, h, w, kernel_size, F_._dt(inputs))
    return 1


def _lr_backward(inputs, grad_output, grad_inputs, kernel_size):
    F_.attn_reshape_bwd(grad_output, kernel_size, grad_inputs)
    return 1


def _rs_forward(input1, input2, output, kernel_size, dilation):
    F_._need_cuda(input1, input2, output)
    _, c, hi, wi = input1.shape
    b, _, h, w = input2.shape
    F_._call("resample2d_fwd", input1, input1.data_ptr(), input2.data_ptr(), output.data_ptr(), b, c, hi, wi, h, w, kernel_size,
             dilation, F_._dt(input1))
    return 1


def _rs_backward(input1, input2, grad_output, grad_input1, grad_input2, kernel_size, dilation):
    F_.resample2d_bwd(input1, input2, grad_output, kernel_size, dilation, grad_input1, grad_input2)
    return 1


def install(python_wrappers: bool = True, reference_root: str | None = None, fuse_extractor_attn: bool = True) -> None:
    """Register the legacy names.  With `reference_root` (a checkout of the reference), the stubbed
    `model.networks` package also resolves the reference's own network files (base_function.py, generator.py,
    ...), so `from model.networks.generator import PoseGenerator` works without importing the reference's
    `model/__init__.py` (which drags in datasets / visualisation dependencies); and, if `fuse_extractor_attn`,
    the reference's `ExtractorAttn` class is replaced by the fused drop-in (same parameters / state_dict)."""
    sys.modules["block_extractor_cuda"] = _mk("block_extractor_cuda", forward=_be_forward, backward=_be_backward)
    sys.modules["local_attn_reshape_cuda"] = _mk("local_attn_reshape_cuda", forward=_lr_forward, backward=_lr_backward)
    sys.modules["resample2d_cuda"] = _mk("resample2d_cuda", forward=_rs_forward, backward=_rs_backward)
    if not python_wrappers:
        return
    from . import block_extractor, local_attn_reshape, resample2d
    for pkg in ("model", "model.networks", "model.networks.block_extractor", "model.networks.local_attn_reshape",
                "model.networks.resample2d_package"):
        if pkg not in sys.modules:
            m = types.ModuleType(pkg)
            m.__path__ = []
            sys.modules[pkg] = m
    sys.modules["model.networks.block_extractor.block_extractor"] = block_extractor
    sys.modules["model.networks.local_attn_reshape.local_attn_reshape"] = local_attn_reshape
    sys.modules["model.networks.resample2d_package.resample2d"] = resample2d
    if reference_root is not None:
        import importlib
        import os
        nets = os.path.join(reference_root, "model", "networks")
        if not os.path.isdir(nets):
            raise FileNotFoundError(nets)
        sys.modules["model.networks"].__path__ = [nets]
        if fuse_extractor_attn:
            from .extractor_attn import ExtractorAttn
            base_function = importlib.import_module("model.networks.base_function")
            base_function.ExtractorAttn = ExtractorAttn      # generator.py does `from ...base_function import *`
