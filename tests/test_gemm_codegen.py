"""CPU test: the flat-layer GEMM kernel (conv_gemm.cu) compiles to unserialized wgmma sequences for sm_90a.

ptxas reports C7519 / C7520 when it has to inject `warpgroup.arrive` waits into a wgmma sequence (each wgmma then
waits for the previous one), and C7512 when it serializes them for lack of registers.  Neither shows up in any output,
only in the kernel's speed, so the compiler's own report and the SASS are checked here, together with the stack and
spill report of both tile shapes (the 128 accumulator registers per thread must stay in registers)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "comfyui_propainter_nodes_b200", "csrc")
KERNEL = "16conv_gemm_kernel"     # mangled conv_gemm_kernel<MB>(GemmParams), anonymous namespace


def _cuda_tool(name):
    path = shutil.which(name)
    if path is None:
        cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)
        path = cand if os.path.exists(cand) else None
    return path


@pytest.fixture(scope="module")
def gemm_build(tmp_path_factory):
    nvcc = _cuda_tool("nvcc")
    if nvcc is None:
        pytest.skip("nvcc not found")
    obj = str(tmp_path_factory.mktemp("gemm") / "conv_gemm.o")
    # the library's flags (csrc/Makefile) plus the ptxas report
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--use_fast_math", "-Xptxas", "-v",
           "-c", os.path.join(CSRC, "conv_gemm.cu"), "-o", obj]
    res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]
    return obj, res.stdout + res.stderr


def test_gemm_kernel_has_no_wgmma_serialization_warnings(gemm_build):
    _, log = gemm_build
    bad = [ln for ln in log.splitlines() if re.search(r"\(C75(19|20|12)\)", ln)]
    assert not bad, "\n".join(bad[:8])


def test_gemm_kernel_has_no_stack_or_spills(gemm_build):
    _, log = gemm_build
    lines = log.splitlines()
    found = 0
    for i, ln in enumerate(lines):
        if "Function properties for" in ln and KERNEL in ln:
            found += 1
            props = lines[i + 1]
            m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", props)
            assert m is not None, props
            assert m.groups() == ("0", "0", "0"), (ln, props)
    assert found == 2, "expected the two tile shapes (MB = 1, 2) of conv_gemm_kernel"


def test_gemm_kernel_sass_waits_once_per_commit_group(gemm_build):
    cuobjdump = _cuda_tool("cuobjdump")
    if cuobjdump is None:
        pytest.skip("cuobjdump not found")
    obj, _ = gemm_build
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)
    bodies = [f for f in funcs if f.startswith("_Z") and KERNEL in f.split("\n", 1)[0]]
    assert len(bodies) == 2, "conv_gemm_kernel<1> / <2> not found in the SASS"
    for body in bodies:
        # a commit group holds 4 * MB HGMMAs (one 64-channel K chunk); a serialized sequence has a wait after each one.
        # The code between two waits (the chunk loop's body; the wait for the last group after the loop closes an
        # empty run) must hold at least 4 HGMMAs.
        runs = [len(re.findall(r"\bHGMMA\.", seg)) for seg in re.split(r"\bWARPGROUP\.DEPBAR", body)]
        runs = [n for n in runs if n > 0]
        assert runs and min(runs) >= 4, runs
