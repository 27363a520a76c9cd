"""CPU test: the multi-layer program kernel (conv_prog_kernel, one flow-completion propagation step per launch) compiles
to unserialized, spill-free wgmma groups for sm_90a.

Its consumer warpgroups hold the accumulators of every tile width the program layers use, next to the deformable
sampler and the epilogue.  When they do not fit, ptxas spills to local memory and serializes the wgmmas (C7512), or
injects `warpgroup.arrive` waits (C7519 / C7520); neither changes any output, only the step's speed, so the compiler's
own report and the SASS are checked here."""
import re

import pytest

from tests.conv_codegen import compile_csrc, sass_functions, stack_and_spills

KERNEL = "16conv_prog_kernelENS_10ProgParamsE"     # mangled conv_prog_kernel(ProgParams), anonymous namespace


@pytest.fixture(scope="module")
def prog_build():
    return compile_csrc("conv_halo.cu")   # the object test_halo_codegen checks: compiled once per session


def test_prog_kernel_has_no_wgmma_serialization_warnings(prog_build):
    _, log = prog_build
    bad = [ln for ln in log.splitlines() if re.search(r"\(C75\d\d\)", ln) and KERNEL in ln]
    assert not bad, "\n".join(bad[:8])


def test_prog_kernel_has_no_stack_or_spills(prog_build):
    _, log = prog_build
    props = stack_and_spills(log, KERNEL)
    assert props, "no ptxas report for conv_prog_kernel"
    assert props[0] == (0, 0, 0), props


def test_prog_kernel_sass_waits_once_per_commit_group(prog_build):
    obj, _ = prog_build
    bodies = sass_functions(obj, KERNEL)
    assert bodies, "conv_prog_kernel not found in the SASS"
    body = bodies[0]
    hgmma = len(re.findall(r"\bHGMMA\.", body))
    depbar = len(re.findall(r"\bWARPGROUP\.DEPBAR", body))
    assert hgmma > 0
    assert not re.search(r"\bSTL\b", body), "local-memory stores (spills) in conv_prog_kernel"
    # a commit group holds at least 4 HGMMAs (one 64-channel chunk of one filter tap); one wait per group
    assert 4 * depbar <= hgmma, (hgmma, depbar)
