"""CPU test: the halo-tile convolution's main loop compiles to unserialized wgmma sequences for sm_90a.

ptxas reports C7519 / C7520 when it has to inject `warpgroup.arrive` waits into a wgmma sequence (each wgmma then
waits for the previous one), and C7512 when it serializes them for lack of registers.  Neither shows up in any output,
only in the kernel's speed, so the compiler's own report and the SASS are checked here."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "comfyui_propainter_nodes_b200", "csrc")
KERNEL = "16conv_halo_kernelENS_10HaloParamsE"     # mangled conv_halo_kernel(HaloParams), anonymous namespace


def _cuda_tool(name):
    path = shutil.which(name)
    if path is None:
        cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)
        path = cand if os.path.exists(cand) else None
    return path


@pytest.fixture(scope="module")
def halo_build(tmp_path_factory):
    nvcc = _cuda_tool("nvcc")
    if nvcc is None:
        pytest.skip("nvcc not found")
    obj = str(tmp_path_factory.mktemp("halo") / "conv_halo.o")
    # the library's flags (csrc/Makefile) plus the ptxas report
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--use_fast_math", "-Xptxas", "-v",
           "-c", os.path.join(CSRC, "conv_halo.cu"), "-o", obj]
    res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]
    return obj, res.stdout + res.stderr


def test_halo_kernel_has_no_wgmma_serialization_warnings(halo_build):
    _, log = halo_build
    bad = [ln for ln in log.splitlines() if re.search(r"\(C75(19|20|12)\)", ln) and KERNEL in ln]
    assert not bad, "\n".join(bad[:8])


def test_conv_halo_kernel_sass_waits_once_per_commit_group(halo_build):
    cuobjdump = _cuda_tool("cuobjdump")
    if cuobjdump is None:
        pytest.skip("cuobjdump not found")
    obj, _ = halo_build
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)
    body = next((f for f in funcs if f.startswith("_Z") and KERNEL in f.split("\n", 1)[0]), None)
    assert body is not None, "conv_halo_kernel not found in the SASS"
    hgmma = len(re.findall(r"\bHGMMA\.", body))
    depbar = len(re.findall(r"\bWARPGROUP\.DEPBAR", body))
    assert hgmma > 0
    # a commit group holds at least 4 HGMMAs (one 64-channel chunk of one filter tap); one wait per group
    assert 4 * depbar <= hgmma, (hgmma, depbar)
