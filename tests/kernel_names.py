"""Kernel names of one profiled run, taken in a child process.

The tests that check which kernels a module launches profile a whole training step: convolutions, the first cuDNN and
cuBLAS work of the process, the backward on autograd's device thread.  Run inside the pytest process ahead of the other
GPU test modules, such sessions were followed by profiler sessions in those modules that recorded none of the library's
kernels.  So these profiles run in a fresh interpreter of their own and hand back the names only: the pytest process
sees no profiler session from them.
"""
import json
import subprocess
import sys

from conftest import ROOT

_PRELUDE = r"""
import json, sys
import torch
from torch.profiler import ProfilerActivity, profile


def profiled(fn):
    fn()                                  # first launches and algorithm choices outside the session
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.key for e in prof.key_averages()]
"""


def kernel_names(body, tmp_path):
    """run `body` (Python source that sets NAMES, typically NAMES = profiled(step)) in a child interpreter started in the
    repository root; -> NAMES"""
    out = tmp_path / "kernel_names.json"
    code = _PRELUDE + body + "\njson.dump(NAMES, open(sys.argv[1], 'w'))\n"
    subprocess.run([sys.executable, "-c", code, str(out)], cwd=ROOT, check=True)
    with open(out) as f:
        return json.load(f)
