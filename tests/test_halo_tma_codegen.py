"""CPU test: conv_halo_kernel with its TMA-store epilogue compiles for sm_90a without stack or spills, and the epilogue
really leaves by TMA stores (UTMASTG) with its operands TMA-loaded.

The TMA epilogue is a per-launch branch of conv_halo_kernel, next to the drain epilogue; test_halo_codegen checks the
kernel's commit groups (no C7519 / C7520 / C7512, at least 4 HGMMA per WARPGROUP.DEPBAR) over both."""
import re

import pytest

from tests.conv_codegen import compile_csrc, sass_functions, stack_and_spills

KERNEL = "16conv_halo_kernelENS_10HaloParamsE"


@pytest.fixture(scope="module")
def halo_build():
    return compile_csrc("conv_halo.cu")


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
