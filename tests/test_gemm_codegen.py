"""CPU test: the flat-layer GEMM kernel (conv_gemm.cu) compiles to unserialized wgmma sequences for sm_90a.

ptxas reports C7519 / C7520 when it has to inject `warpgroup.arrive` waits into a wgmma sequence (each wgmma then
waits for the previous one), and C7512 when it serializes them for lack of registers.  Neither shows up in any output,
only in the kernel's speed, so the compiler's own report and the SASS are checked here, together with the stack and
spill report of both tile shapes (the 128 accumulator registers per thread must stay in registers)."""
import re

import pytest

from tests.conv_codegen import compile_csrc, sass_functions, stack_and_spills

KERNEL = "16conv_gemm_kernel"     # mangled conv_gemm_kernel<MB>(GemmParams), anonymous namespace


@pytest.fixture(scope="module")
def gemm_build():
    return compile_csrc("conv_gemm.cu")


def test_gemm_kernel_has_no_wgmma_serialization_warnings(gemm_build):
    _, log = gemm_build
    bad = [ln for ln in log.splitlines() if re.search(r"\(C75(19|20|12)\)", ln)]
    assert not bad, "\n".join(bad[:8])


def test_gemm_kernel_has_no_stack_or_spills(gemm_build):
    _, log = gemm_build
    props = stack_and_spills(log, KERNEL)
    assert len(props) == 2, "expected the two tile shapes (MB = 1, 2) of conv_gemm_kernel"
    assert all(p == (0, 0, 0) for p in props), props


def test_gemm_kernel_sass_waits_once_per_commit_group(gemm_build):
    obj, _ = gemm_build
    bodies = sass_functions(obj, KERNEL)
    assert len(bodies) == 2, "conv_gemm_kernel<1> / <2> not found in the SASS"
    for body in bodies:
        # a commit group holds 4 * MB HGMMAs (one 64-channel K chunk); a serialized sequence has a wait after each one.
        # The code between two waits (the chunk loop's body; the wait for the last group after the loop closes an
        # empty run) must hold at least 4 HGMMAs.
        runs = [len(re.findall(r"\bHGMMA\.", seg)) for seg in re.split(r"\bWARPGROUP\.DEPBAR", body)]
        runs = [n for n in runs if n > 0]
        assert runs and min(runs) >= 4, runs
