"""CPU test: the halo-tile convolution's main loop compiles to unserialized wgmma sequences for sm_90a, without stack
or spills, and its TMA epilogue really leaves by TMA stores (UTMASTG) with its operands TMA-loaded.

ptxas reports C7519 / C7520 when it has to inject `warpgroup.arrive` waits into a wgmma sequence (each wgmma then
waits for the previous one), and C7512 when it serializes them for lack of registers.  Neither shows up in any output,
only in the kernel's speed, so the compiler's own report and the SASS are checked here.  The TMA epilogue is a
per-launch branch of conv_halo_kernel next to the drain epilogue, so the checks of the commit groups cover both."""
import re

import pytest

from tests.conv_codegen import compile_csrc, sass_functions, stack_and_spills

KERNEL = "16conv_halo_kernelENS_10HaloParamsE"     # mangled conv_halo_kernel(HaloParams), anonymous namespace


@pytest.fixture(scope="module")
def halo_build():
    return compile_csrc("conv_halo.cu")


def test_halo_kernel_has_no_wgmma_serialization_warnings(halo_build):
    _, log = halo_build
    bad = [ln for ln in log.splitlines() if re.search(r"\(C75(19|20|12)\)", ln) and KERNEL in ln]
    assert not bad, "\n".join(bad[:8])


def test_conv_halo_kernel_sass_waits_once_per_commit_group(halo_build):
    obj, _ = halo_build
    bodies = sass_functions(obj, KERNEL)
    assert bodies, "conv_halo_kernel not found in the SASS"
    hgmma = len(re.findall(r"\bHGMMA\.", bodies[0]))
    depbar = len(re.findall(r"\bWARPGROUP\.DEPBAR", bodies[0]))
    assert hgmma > 0
    # a commit group holds at least 4 HGMMAs (one 64-channel chunk of one filter tap); one wait per group
    assert 4 * depbar <= hgmma, (hgmma, depbar)


def test_conv_halo_kernel_has_no_stack_or_spills(halo_build):
    _, log = halo_build
    reports = stack_and_spills(log, KERNEL)
    assert reports, "conv_halo_kernel not in the ptxas report"
    assert all(r == (0, 0, 0) for r in reports), reports


def test_conv_halo_kernel_stores_with_tma(halo_build):
    obj, _ = halo_build
    bodies = sass_functions(obj, KERNEL)
    assert bodies, "conv_halo_kernel not found in the SASS"
    assert re.search(r"\bUTMASTG\b", bodies[0]), "no TMA store in conv_halo_kernel"
    # patch loads and the epilogue's operand loads
    assert len(re.findall(r"\bUTMALDG\b", bodies[0])) >= 2
