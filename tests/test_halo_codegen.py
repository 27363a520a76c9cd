"""CPU test: the halo-tile convolution's main loop compiles to unserialized wgmma sequences for sm_90a.

ptxas reports C7519 / C7520 when it has to inject `warpgroup.arrive` waits into a wgmma sequence (each wgmma then
waits for the previous one), and C7512 when it serializes them for lack of registers.  Neither shows up in any output,
only in the kernel's speed, so the compiler's own report and the SASS are checked here."""
import re

import pytest

from tests.conv_codegen import compile_csrc, sass_functions

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
