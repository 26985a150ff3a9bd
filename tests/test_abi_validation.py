"""CPU: every entry point of the C ABI rejects bad arguments with its exact GFLA_E_* code, including which error wins
when several arguments are bad.

Every call made here is one that argument validation rejects: the pointers are host addresses standing in for device
ones, and nothing may reach a launch (each test checks that the library's launch counter did not move).  No GPU is
needed."""
import ctypes

import pytest

NULL, SHAPE, DTYPE, ALIGN, NOTSUP = -1, -2, -3, -4, -5
F32, F64, BF16, F16, BAD_DT = 0, 1, 2, 3, 7
NCHW, NHWC = 0, 1

_BUF = ctypes.create_string_buffer(1 << 16)
P = (ctypes.addressof(_BUF) + 255) & ~255      # 256-byte aligned stand-in for every device buffer
Q = P + 4096                                    # a second one where two buffers must differ

# what each argument is when a case does not override it: a call that would pass validation (and so is never made as is)
DEFAULTS = dict(B=1, C=64, Hs=8, Ws=8, Hf=8, Wf=8, Hi=8, Wi=8, H=8, W=8, k=3, ks=2, dilation=1, eps=1e-8, N=128, n=64,
                dtype=F32, flow_dtype=F32, grad_source_dtype=F32, src_dtype=F32, dst_dtype=BF16, layout=NCHW, algo=0,
                accumulate=0, to_nhwc=1, workspace=P, workspace_bytes=1 << 20, stream=None, probs=None)

_LA = "B C Hs Ws H W k dtype flow_dtype layout"
_RS = "B C Hi Wi H W ks dilation"
# entry point -> (its arguments in ABI order, defaults that differ from DEFAULTS); an argument not in DEFAULTS is a pointer to P
SPECS = {
    "gfla_debug_set_buffer": ("p", {}),
    "gfla_debug_wait_profile": ("which enable out", {"which": 0, "enable": 1}),
    "gfla_relayout": ("src dst B C H W dtype to_nhwc stream", {"dst": Q}),
    "gfla_block_extract_fwd": ("source flow out B C Hs Ws Hf Wf k dtype flow_dtype stream", {}),
    "gfla_block_extract_bwd": ("source flow grad_out grad_source grad_flow B C Hs Ws Hf Wf k dtype flow_dtype grad_source_dtype "
                               "accumulate stream", {}),
    "gfla_convert": ("src src_dtype dst dst_dtype n stream", {}),
    "gfla_attn_reshape_fwd": ("inp out B H W k dtype stream", {}),
    "gfla_attn_reshape_bwd": ("grad_out grad_in B H W k dtype accumulate stream", {}),
    "gfla_resample2d_fwd": (f"in1 in2 out {_RS} dtype stream", {}),
    "gfla_resample2d_bwd": (f"in1 in2 grad_out grad_in1 grad_in2 {_RS} dtype accumulate stream", {}),
    "gfla_resample2d_cosine_fwd": (f"in1 in2 target cos_out stats {_RS} eps dtype stream", {}),
    "gfla_resample2d_cosine_bwd": (f"in1 in2 target stats grad_cos grad_in1 grad_in2 grad_val grad_target {_RS} eps dtype "
                                   "accumulate stream", {}),
    "gfla_resample2d16_fwd": (f"in1 in2 out {_RS} dtype stream", {"dtype": BF16}),
    "gfla_resample2d16_bwd": (f"in1 in2 grad_out grad_in1 grad_in2 {_RS} dtype accumulate stream", {"dtype": BF16}),
    "gfla_resample2d16_cosine_fwd": (f"in1 in2 target cos_out stats {_RS} eps dtype stream", {"dtype": BF16}),
    "gfla_resample2d16_cosine_bwd": (f"in1 in2 target stats grad_cos grad_in1 grad_in2 grad_val grad_target {_RS} eps dtype "
                                     "accumulate stream", {"dtype": BF16}),
    "gfla_local_attn_fwd": (f"source flow logits out probs {_LA} algo stream", {}),
    "gfla_local_attn_blend_fwd": (f"source flow logits prev mask out {_LA} algo stream", {}),
    "gfla_local_attn_bwd": (f"source flow logits grad_out grad_source grad_flow grad_logits {_LA} accumulate algo stream", {}),
    "gfla_local_attn_bwd_workspace_bytes": ("B", {}),
    "gfla_local_attn_bwd_ws": (f"source flow logits grad_out grad_source grad_flow grad_logits {_LA} accumulate algo workspace "
                               "workspace_bytes stream", {}),
    "gfla_patch_conv_fwd": ("source flow weight out B C Hs Ws H W k N dtype flow_dtype layout stream",
                            {"dtype": BF16, "layout": NHWC}),
    "gfla_patch_conv_bwd": ("source flow weight grad_out grad_source grad_flow grad_weight B C Hs Ws H W k N dtype flow_dtype "
                            "layout accumulate stream", {"dtype": BF16, "layout": NHWC}),
    "gfla_local_attn_bwd_det_workspace_bytes": ("B C Hs Ws H W k", {}),
    "gfla_local_attn_bwd_det": (f"source flow logits grad_out grad_source grad_flow grad_logits {_LA} accumulate algo workspace "
                                "workspace_bytes stream", {}),
    "gfla_block_extract_bwd_det_workspace_bytes": ("B C Hs Ws Hf Wf k", {}),
    "gfla_block_extract_bwd_det": ("source flow grad_out grad_source grad_flow B C Hs Ws Hf Wf k dtype flow_dtype accumulate "
                                   "workspace workspace_bytes stream", {}),
    "gfla_patch_conv_bwd_det_workspace_bytes": ("B C Hs Ws H W k N", {}),
    "gfla_patch_conv_bwd_det": ("source flow weight grad_out grad_source grad_flow grad_weight B C Hs Ws H W k N dtype "
                                "flow_dtype layout accumulate workspace workspace_bytes stream", {"dtype": BF16, "layout": NHWC}),
}
NO_ARGUMENTS = {"gfla_abi_version", "gfla_device_check", "gfla_debug_launch_count"}


def _call(so, name, **over):
    names, own = SPECS[name]
    names = names.split()
    unknown = set(over) - set(names)
    assert not unknown, f"{name} has no argument {unknown}"
    args = [over[a] if a in over else own.get(a, DEFAULTS.get(a, P)) for a in names]
    return getattr(so, name)(*args)


# ------------------------------------------------------------------------------------------------ case builders
def nulls(*ptrs):
    return [({p: None}, NULL) for p in ptrs]


def nonpositive(*sizes):
    return [({s: v}, SHAPE) for s in sizes for v in (0, -1)]


def misaligned(**need):
    """each pointer moved off the alignment it needs (in bytes) by half of it"""
    return [({p: P + b // 2}, ALIGN) for p, b in need.items()]


def k_range(name="k"):
    return [({name: 0}, SHAPE), ({name: 10}, SHAPE)]


def resample_cases(fwd_or_bwd, half):
    """the two resample2d families: 16-bit feature maps with in2, stats, grad_in2, grad_in1 and grad_val in fp32, or
    fp32 / fp64 throughout"""
    d = 2 if half else 4             # the data dtype's size at the family's default dtype (BF16 / F32)
    w = 4 if half else d             # in2, stats, grad_in2, grad_in1, grad_val: fp32 in the 16-bit family
    other = (F32, F64, BAD_DT) if half else (BF16, F16, BAD_DT)
    cases = nonpositive(*_RS.split()[:6]) + k_range("ks") + [({"ks": 1}, SHAPE), ({"dilation": 0}, SHAPE),
                                                             ({"dilation": -1}, SHAPE)]
    cases += [({"dtype": dt}, DTYPE) for dt in other]
    cases += [({"B": 0, "dtype": BAD_DT}, SHAPE), ({"dtype": BAD_DT, "in1": P + 1}, DTYPE)]
    if not half:
        cases += [({"dtype": F64, "in1": P + 4}, ALIGN), ({"dtype": F64, "in2": P + 4}, ALIGN)]
    else:
        cases += [({"dtype": F16, "in1": P + 1}, ALIGN), ({"dtype": F16, "in2": P + 2}, ALIGN)]
    if fwd_or_bwd == "fwd":
        return cases + nulls("in1", "in2", "out") + misaligned(in1=d, in2=w, out=d) + [({"in1": None, "B": 0}, NULL)]
    if fwd_or_bwd == "bwd":
        return (cases + nulls("in1", "in2", "grad_out", "grad_in1", "grad_in2")
                + misaligned(in1=d, in2=w, grad_out=d, grad_in1=w, grad_in2=w))
    eps = [({"eps": -1e-8}, SHAPE), ({"eps": float("nan")}, SHAPE), ({"eps": float("-inf")}, SHAPE)]
    if fwd_or_bwd == "cos_fwd":
        return (cases + eps + nulls("in1", "in2", "target", "cos_out", "stats")
                + misaligned(in1=d, in2=w, target=d, cos_out=d, stats=w))
    return (cases + eps + nulls("in1", "in2", "target", "stats", "grad_cos", "grad_in2")
            + misaligned(in1=d, in2=w, target=d, stats=w, grad_cos=d, grad_in2=w, grad_in1=w, grad_val=w, grad_target=d)
            + [({"grad_val": None}, NULL),                                  # grad_in1 without grad_val
               ({"grad_val": None, "B": 0, "dtype": BAD_DT}, NULL),         # ... wins over shape and dtype
               ({"grad_in1": None, "grad_val": P + 2}, ALIGN),                  # grad_val is checked on its own
               ({"grad_in1": None, "grad_val": None, "grad_target": P + d // 2}, ALIGN),
               ({"in1": None, "grad_val": None}, NULL)])


def local_attn_common(ptrs):
    """shape, dtype and algo checks shared by the local-attention entry points"""
    return (nulls(*ptrs) + nonpositive(*_LA.split()[:6]) + k_range()
            + [({"layout": 2}, SHAPE), ({"layout": -1}, SHAPE),
               ({"dtype": BAD_DT}, DTYPE), ({"dtype": F32, "flow_dtype": F64}, DTYPE), ({"dtype": F64, "flow_dtype": F32}, DTYPE),
               ({"dtype": BF16, "flow_dtype": F16}, DTYPE), ({"flow_dtype": BAD_DT}, DTYPE),
               ({"algo": 3}, NOTSUP), ({"algo": -1}, NOTSUP),
               ({"B": 0, "dtype": BAD_DT}, SHAPE), ({"dtype": BAD_DT, "algo": 3}, DTYPE), ({"algo": 3, "source": P + 2}, NOTSUP),
               ({"source": P + 2, "algo": 2}, ALIGN),
               ({"algo": 2}, NOTSUP)])                                     # the tile kernels serve 16-bit data only


# the tile kernels' support rules, at 16-bit data: each case asks for the tile algorithm where it cannot serve
_TILE = dict(dtype=BF16, layout=NHWC, algo=2)
TILE_FWD = [({**_TILE, **o}, NOTSUP) for o in (
    {"k": 7}, {"C": 96}, {"flow_dtype": BF16}, {"source": P + 2}, {"out": P + 2}, {"dtype": F16, "k": 4},
    {"layout": NCHW, "Ws": 4})]
TILE_BWD = [({**_TILE, **o}, NOTSUP) for o in (
    {"k": 7}, {"C": 96}, {"C": 32}, {"flow_dtype": BF16}, {"layout": NCHW}, {"source": P + 2}, {"grad_out": P + 2},
    {"dtype": F16, "C": 192})]

_LA_BWD_PTRS = ("source", "flow", "logits", "grad_out", "grad_source", "grad_flow", "grad_logits")
LA_BWD = (local_attn_common(_LA_BWD_PTRS) + TILE_BWD
          + misaligned(source=4, logits=4, grad_out=4, grad_source=4, grad_logits=4, flow=4, grad_flow=4)
          + [({"source": None, "layout": 2}, SHAPE),                       # the backward checks the layout first
             ({"dtype": BF16, "flow_dtype": F32, "flow": P + 2}, ALIGN), ({"dtype": F64, "flow_dtype": F64, "grad_flow": P + 4}, ALIGN)])


def det_workspace():
    """workspace NULL, misaligned or too small; the alignment of the data wins over the workspace"""
    return [({"workspace": None}, NULL), ({"workspace": P + 8}, ALIGN), ({"workspace": P + 4}, ALIGN),
            ({"workspace_bytes": -1}, SHAPE), ({"workspace_bytes": 0}, SHAPE), ({"workspace_bytes": ("need", -1)}, SHAPE),
            ({"workspace": None, "source": P + 2}, ALIGN), ({"workspace": None, "B": 0}, SHAPE)]


_PC = ("B", "C", "Hs", "Ws", "H", "W", "N")
PATCH_CONV_COMMON = (nonpositive(*_PC) + k_range()
                     + [({"layout": 2}, SHAPE), ({"dtype": F16}, DTYPE), ({"dtype": F32}, DTYPE), ({"dtype": BAD_DT}, DTYPE),
                        ({"flow_dtype": BF16}, DTYPE), ({"flow_dtype": F64}, DTYPE),
                        ({"layout": NCHW}, NOTSUP), ({"C": 96}, NOTSUP), ({"N": 64}, NOTSUP),
                        ({"source": None, "layout": 2}, NULL), ({"layout": 2, "dtype": F16}, SHAPE), ({"B": 0, "dtype": F16}, SHAPE),
                        ({"dtype": F16, "layout": NCHW}, DTYPE), ({"C": 96, "source": P + 8}, NOTSUP),
                        ({"source": P + 8, "flow": P + 2}, ALIGN)])

CASES = {
    "gfla_debug_set_buffer": [({}, NOTSUP), ({"p": None}, NOTSUP)],
    "gfla_debug_wait_profile": [({"which": -1}, SHAPE), ({"which": 3}, SHAPE), ({"which": 0}, NOTSUP), ({"which": 2}, NOTSUP)],
    "gfla_relayout": (nulls("src", "dst") + nonpositive("B", "C", "H", "W") + misaligned(src=4, dst=4)
                      + [({"dtype": BAD_DT}, DTYPE), ({"dtype": -1}, DTYPE), ({"dst": P}, NOTSUP), ({"src": P + 2, "dst": P + 2}, NOTSUP),
                         ({"dtype": BF16, "src": P + 1}, ALIGN), ({"dtype": F64, "dst": Q + 4}, ALIGN),
                         ({"src": None, "B": 0}, NULL), ({"B": 0, "dtype": BAD_DT}, SHAPE), ({"dtype": BAD_DT, "dst": P}, DTYPE)]),
    "gfla_block_extract_fwd": (nulls("source", "flow", "out") + nonpositive("B", "C", "Hs", "Ws", "Hf", "Wf") + k_range()
                               + misaligned(source=4, out=4, flow=4)
                               + [({"dtype": BAD_DT, "flow_dtype": BAD_DT}, DTYPE), ({"flow_dtype": F64}, DTYPE),
                                  ({"dtype": F64}, DTYPE), ({"dtype": BF16, "flow_dtype": F16}, DTYPE),
                                  ({"dtype": F64, "flow_dtype": F64, "flow": P + 4}, ALIGN),
                                  ({"dtype": BF16, "flow_dtype": F32, "flow": P + 2}, ALIGN),
                                  ({"dtype": BF16, "flow_dtype": BF16, "source": P + 1}, ALIGN),
                                  ({"out": None, "k": 0}, NULL), ({"k": 0, "dtype": BAD_DT}, SHAPE), ({"flow_dtype": F64, "out": P + 2}, DTYPE)]),
    "gfla_block_extract_bwd": (nulls("source", "flow", "grad_out", "grad_source", "grad_flow")
                               + nonpositive("B", "C", "Hs", "Ws", "Hf", "Wf") + k_range()
                               + misaligned(source=4, flow=4, grad_out=4, grad_source=4, grad_flow=4)
                               + [({"grad_source_dtype": BF16}, DTYPE), ({"grad_source_dtype": F64}, DTYPE),
                                  ({"dtype": F64, "flow_dtype": F64}, DTYPE), ({"dtype": BAD_DT}, DTYPE),
                                  ({"dtype": BF16, "flow_dtype": BF16, "grad_source_dtype": F16}, DTYPE),
                                  ({"dtype": BF16, "flow_dtype": BF16, "grad_source_dtype": F32, "grad_source": P + 2}, ALIGN),
                                  ({"dtype": BF16, "flow_dtype": F32, "grad_source_dtype": BF16, "grad_flow": P + 2}, ALIGN),
                                  ({"dtype": F16, "flow_dtype": F16, "grad_source_dtype": F16, "grad_out": P + 1}, ALIGN),
                                  ({"grad_flow": None, "B": 0}, NULL), ({"B": 0, "grad_source_dtype": BF16}, SHAPE)]),
    "gfla_convert": (nulls("src", "dst") + nonpositive("n") + misaligned(src=4, dst=2)
                     + [({"src_dtype": BAD_DT}, DTYPE), ({"dst_dtype": BAD_DT}, DTYPE), ({"src_dtype": -1}, DTYPE),
                        ({"src_dtype": F64, "src": P + 4}, ALIGN), ({"n": 0, "src_dtype": BAD_DT}, SHAPE),
                        ({"dst_dtype": BAD_DT, "src": P + 2}, DTYPE), ({"src": None, "n": 0}, NULL)]),
    "gfla_attn_reshape_fwd": (nulls("inp", "out") + nonpositive("B", "H", "W") + k_range() + misaligned(inp=4, out=4)
                              + [({"dtype": BAD_DT}, DTYPE), ({"dtype": BF16, "out": P + 1}, ALIGN), ({"k": 0, "dtype": BAD_DT}, SHAPE)]),
    "gfla_attn_reshape_bwd": (nulls("grad_out", "grad_in") + nonpositive("B", "H", "W") + k_range()
                              + misaligned(grad_out=4, grad_in=4)
                              + [({"dtype": BAD_DT}, DTYPE), ({"dtype": F64, "grad_in": P + 4}, ALIGN),
                                 ({"grad_in": None, "k": 10}, NULL)]),
    "gfla_resample2d_fwd": resample_cases("fwd", False),
    "gfla_resample2d_bwd": resample_cases("bwd", False),
    "gfla_resample2d_cosine_fwd": resample_cases("cos_fwd", False),
    "gfla_resample2d_cosine_bwd": resample_cases("cos_bwd", False),
    "gfla_resample2d16_fwd": resample_cases("fwd", True),
    "gfla_resample2d16_bwd": resample_cases("bwd", True),
    "gfla_resample2d16_cosine_fwd": resample_cases("cos_fwd", True),
    "gfla_resample2d16_cosine_bwd": resample_cases("cos_bwd", True),
    "gfla_local_attn_fwd": (local_attn_common(("source", "flow", "logits", "out")) + TILE_FWD
                            + misaligned(source=4, logits=4, out=4, flow=4, probs=4)
                            + [({"source": None, "layout": 2}, NULL),       # the forward checks the pointers first
                               ({"dtype": BF16, "flow_dtype": F32, "logits": P + 1}, ALIGN)]),
    "gfla_local_attn_blend_fwd": (local_attn_common(("source", "flow", "logits", "prev", "mask", "out")) + TILE_FWD
                                  + misaligned(source=4, logits=4, out=4, flow=4, prev=4, mask=4)
                                  + [({"prev": None, "layout": 2}, NULL), ({"mask": None, "source": None}, NULL),
                                     ({**_TILE, "prev": P + 2}, NOTSUP)]),       # channels-last tile: prev 16-byte aligned
    "gfla_local_attn_bwd": LA_BWD + [({**_TILE, "grad_source": P + 2}, NOTSUP)],
    "gfla_local_attn_bwd_workspace_bytes": [({"B": 0}, 0), ({"B": 1}, 0)],
    "gfla_local_attn_bwd_ws": (LA_BWD + [({**_TILE, "grad_source": P + 2}, NOTSUP),
                                         ({"workspace_bytes": -1}, SHAPE), ({"workspace_bytes": -1, "source": None}, SHAPE),
                                         ({"workspace": None, "workspace_bytes": -1, "source": None}, NULL)]),
    "gfla_patch_conv_fwd": (nulls("source", "flow", "weight", "out") + PATCH_CONV_COMMON
                            + misaligned(source=16, weight=16, out=16, flow=4) + [({"out": P + 2}, ALIGN)]),
    "gfla_patch_conv_bwd": (nulls("source", "flow", "weight", "grad_out", "grad_source", "grad_flow", "grad_weight")
                            + PATCH_CONV_COMMON
                            + misaligned(source=16, weight=16, grad_out=16, grad_source=16, grad_weight=16, flow=4, grad_flow=4)),
    "gfla_local_attn_bwd_det_workspace_bytes": nonpositive(*_LA.split()[:6]) + k_range(),
    "gfla_local_attn_bwd_det": (LA_BWD + det_workspace()
                                + [({"workspace": None, "algo": 2}, NULL),   # the workspace is checked before the tile's support
                                   ({"workspace_bytes": ("need", -1), "algo": 2}, SHAPE)]),
    "gfla_block_extract_bwd_det_workspace_bytes": nonpositive("B", "C", "Hs", "Ws", "Hf", "Wf") + k_range(),
    "gfla_block_extract_bwd_det": (nulls("source", "flow", "grad_out", "grad_source", "grad_flow")
                                   + nonpositive("B", "C", "Hs", "Ws", "Hf", "Wf") + k_range()
                                   + misaligned(source=4, flow=4, grad_out=4, grad_source=4, grad_flow=4)
                                   + [({"dtype": BAD_DT}, DTYPE), ({"flow_dtype": F64}, DTYPE), ({"dtype": BF16, "flow_dtype": F16}, DTYPE),
                                      ({"dtype": BF16, "flow_dtype": F32, "grad_source": P + 1}, ALIGN)]
                                   + det_workspace()),
    "gfla_patch_conv_bwd_det_workspace_bytes": nonpositive(*_PC) + k_range(),
    "gfla_patch_conv_bwd_det": (nulls("source", "flow", "weight", "grad_out", "grad_source", "grad_flow", "grad_weight")
                                + PATCH_CONV_COMMON
                                + misaligned(source=16, weight=16, grad_out=16, grad_source=2, grad_weight=2, flow=4, grad_flow=4)
                                + det_workspace() + [({"workspace": None, "grad_weight": P + 1}, ALIGN)]),
}
# the size a deterministic entry point's workspace needs at the default arguments
NEED = {"gfla_local_attn_bwd_det": "gfla_local_attn_bwd_det_workspace_bytes",
        "gfla_block_extract_bwd_det": "gfla_block_extract_bwd_det_workspace_bytes",
        "gfla_patch_conv_bwd_det": "gfla_patch_conv_bwd_det_workspace_bytes"}


@pytest.fixture(scope="module")
def so():
    import __graft_entry__ as ge
    ge.build_cuda()
    import gfla_b200
    return gfla_b200._lib.lib()


@pytest.fixture
def no_launch(so):
    before = so.gfla_debug_launch_count()
    yield
    assert so.gfla_debug_launch_count() == before, "an argument check let a call through to a launch"


def test_cases_cover_every_entry_point():
    from gfla_b200 import _lib
    assert set(SPECS) == set(CASES) == set(_lib.SIGNATURES) - NO_ARGUMENTS
    for name, (names, own) in SPECS.items():
        assert len(names.split()) == len(_lib.SIGNATURES[name]), name
        assert set(own) <= set(names.split()), name


_PARAMS = [pytest.param(name, over, code, id=f"{name[5:]}-{i}") for name, cases in CASES.items() for i, (over, code) in enumerate(cases)]


@pytest.mark.parametrize("name,over,code", _PARAMS)
def test_rejected(so, no_launch, name, over, code):
    over = dict(over)
    if isinstance(over.get("workspace_bytes"), tuple):         # ("need", d): the size the query reports, plus d
        need = _call(so, NEED[name])
        assert need > 0
        over["workspace_bytes"] = need + over["workspace_bytes"][1]
    assert _call(so, name, **over) == code, over


def test_abi_rejects_other_dtypes(so, no_launch):
    """the 16-bit resample2d entry points take BF16 / F16 feature maps only, with an fp32 flow"""
    from gfla_b200 import _lib
    l = so
    buf = (ctypes.c_float * 64)()
    p = ctypes.addressof(buf)
    for dt in (_lib.GFLA_F32, _lib.GFLA_F64, 7):
        assert l.gfla_resample2d16_fwd(p, p, p, 1, 1, 2, 2, 2, 2, 2, 1, dt, None) == -3
        assert l.gfla_resample2d16_cosine_fwd(p, p, p, p, p, 1, 1, 2, 2, 2, 2, 2, 1, 1e-8, dt, None) == -3
    assert l.gfla_resample2d16_fwd(p, p + 2, p, 1, 1, 2, 2, 2, 2, 2, 1, _lib.GFLA_BF16, None) == -4    # fp32 flow alignment
    assert l.gfla_resample2d16_cosine_bwd(p, p, p, p, p, p, p, None, None, 1, 1, 2, 2, 2, 2, 2, 1, 1e-8, _lib.GFLA_F16, 0,
                                          None) == -1                                                  # grad_in1 without grad_val
