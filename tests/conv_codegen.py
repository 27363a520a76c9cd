"""Shared plumbing of the CPU codegen tests of the wgmma convolution kernels (test_halo_codegen, test_prog_codegen,
test_gemm_codegen): the CUDA tools, one compile per csrc file and test session however many modules check its kernels,
the SASS of one kernel and the ptxas stack / spill report."""
import functools
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "comfyui_propainter_nodes_b200", "csrc")

_OBJDIR = tempfile.TemporaryDirectory(prefix="pp_codegen_")   # removed when the session ends


def _cuda_tool(name):
    path = shutil.which(name)
    if path is None:
        cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)
        path = cand if os.path.exists(cand) else None
    return path


@functools.lru_cache(maxsize=None)
def _build(source):
    nvcc = _cuda_tool("nvcc")
    if nvcc is None:
        return None
    obj = os.path.join(_OBJDIR.name, source.replace(".cu", ".o"))
    # the library's flags (csrc/Makefile) plus the ptxas report
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--use_fast_math", "-Xptxas", "-v",
           "-c", os.path.join(CSRC, source), "-o", obj]
    res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    return obj, res.returncode, res.stdout + res.stderr


def compile_csrc(source):
    """(object file, ptxas log) of csrc/`source`, compiled once per session."""
    built = _build(source)
    if built is None:
        pytest.skip("nvcc not found")
    obj, rc, log = built
    assert rc == 0, log[-4000:]
    return obj, log


def sass_functions(obj, kernel):
    """SASS of every function of `obj` whose mangled name contains `kernel`."""
    cuobjdump = _cuda_tool("cuobjdump")
    if cuobjdump is None:
        pytest.skip("cuobjdump not found")
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)
    return [f for f in funcs if f.startswith("_Z") and kernel in f.split("\n", 1)[0]]


def stack_and_spills(log, kernel):
    """(stack frame, spill stores, spill loads) bytes of every function in the ptxas report whose name contains
    `kernel`."""
    lines = log.splitlines()
    out = []
    for i, ln in enumerate(lines):
        if "Function properties for" in ln and kernel in ln:
            m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", lines[i + 1])
            assert m is not None, lines[i + 1]
            out.append(tuple(int(v) for v in m.groups()))
    return out
