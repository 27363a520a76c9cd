"""CPU test: the multi-layer program kernel (conv_prog_kernel, one flow-completion propagation step per launch) compiles
to unserialized, spill-free wgmma groups for sm_90a.

Its consumer warpgroups hold the accumulators of every tile width the program layers use, next to the deformable
sampler and the epilogue.  When they do not fit, ptxas spills to local memory and serializes the wgmmas (C7512), or
injects `warpgroup.arrive` waits (C7519 / C7520); neither changes any output, only the step's speed, so the compiler's
own report and the SASS are checked here."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "comfyui_propainter_nodes_b200", "csrc")
KERNEL = "16conv_prog_kernelENS_10ProgParamsE"     # mangled conv_prog_kernel(ProgParams), anonymous namespace


def _cuda_tool(name):
    path = shutil.which(name)
    if path is None:
        cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)
        path = cand if os.path.exists(cand) else None
    return path


@pytest.fixture(scope="module")
def prog_build(tmp_path_factory):
    nvcc = _cuda_tool("nvcc")
    if nvcc is None:
        pytest.skip("nvcc not found")
    obj = str(tmp_path_factory.mktemp("prog") / "conv_halo.o")
    # the library's flags (csrc/Makefile) plus the ptxas report
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--use_fast_math", "-Xptxas", "-v",
           "-c", os.path.join(CSRC, "conv_halo.cu"), "-o", obj]
    res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]
    return obj, res.stdout + res.stderr


def test_prog_kernel_has_no_wgmma_serialization_warnings(prog_build):
    _, log = prog_build
    bad = [ln for ln in log.splitlines() if re.search(r"\(C75\d\d\)", ln) and KERNEL in ln]
    assert not bad, "\n".join(bad[:8])


def test_prog_kernel_has_no_stack_or_spills(prog_build):
    _, log = prog_build
    lines = log.splitlines()
    idx = next((i for i, ln in enumerate(lines) if "Function properties for" in ln and KERNEL in ln), None)
    assert idx is not None, "no ptxas report for conv_prog_kernel"
    props = lines[idx + 1]
    m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", props)
    assert m is not None, props
    assert tuple(int(v) for v in m.groups()) == (0, 0, 0), props


def test_prog_kernel_sass_waits_once_per_commit_group(prog_build):
    cuobjdump = _cuda_tool("cuobjdump")
    if cuobjdump is None:
        pytest.skip("cuobjdump not found")
    obj, _ = prog_build
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)
    body = next((f for f in funcs if f.startswith("_Z") and KERNEL in f.split("\n", 1)[0]), None)
    assert body is not None, "conv_prog_kernel not found in the SASS"
    hgmma = len(re.findall(r"\bHGMMA\.", body))
    depbar = len(re.findall(r"\bWARPGROUP\.DEPBAR", body))
    assert hgmma > 0
    assert not re.search(r"\bSTL\b", body), "local-memory stores (spills) in conv_prog_kernel"
    # a commit group holds at least 4 HGMMAs (one 64-channel chunk of one filter tap); one wait per group
    assert 4 * depbar <= hgmma, (hgmma, depbar)
