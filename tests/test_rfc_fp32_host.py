"""CPU tests of the fp32 flow completion: its C-ABI entry points, the precision the inference layer picks from the
node's fp16 switch, the codegen of the new fp32 kernels (no fp16 rounding, no hardware tanh), and proof that the
sampler's operator bound in tests/test_rfc_fp32_ops.py rejects the precision losses it is there to catch."""
import os
import re
import subprocess
import types

import pytest
import torch

from comfyui_propainter_nodes_b200 import engine as E
from comfyui_propainter_nodes_b200 import parallel as PAR
from comfyui_propainter_nodes_b200 import propainter_inference as PI
from tests import test_raft_fp32_ops as OPS
from tests import test_rfc_fp32_ops as RFC
from tests.conv_codegen import CSRC, _cuda_tool

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ("pp_flow_complete_fp32", "pp_flow_complete_dist_fp32", "pp_op_dcn_sample_f32", "pp_op_upsample2x_f32")


def test_fp32_flow_completion_entry_points_are_declared_and_exported():
    import ctypes
    hdr = open(os.path.join(ROOT, "include", "propainter_b200.h")).read()
    lib = ctypes.CDLL(E.LIB_PATH)
    for name in NEW_SYMBOLS:
        assert re.search(r"PP_API int " + name + r"\(", hdr), name
        assert name in E.exported_symbols()
        getattr(lib, name)
    # pp_op_conv_tf32 takes the dilation and replicate padding the flow-completion layers need
    decl = re.search(r"PP_API int pp_op_conv_tf32\(([^;]*)\);", hdr).group(1)
    assert re.search(r"int dh,\s*int dw,\s*int replicate", decl), decl
    assert len(decl.split(",")) == len(E._SIGNATURES["pp_op_conv_tf32"][1])


class _StubEngine:
    """Records the precision of every flow_complete call; returns the flows unchanged."""

    world = 1

    def __init__(self):
        self.calls = []

    def flow_complete(self, flows_f, flows_b, flow_masks, fp32=False):
        self.calls.append((flows_f.shape[0], fp32))
        return flows_f.float().clone(), flows_b.float().clone()


@pytest.mark.parametrize("fp16,fp32", [("disable", True), ("enable", False)])
@pytest.mark.parametrize("T,sub", [(6, 80), (26, 12)])
@pytest.mark.parametrize("distributed", [False, True])
def test_flow_completion_picks_precision_from_the_fp16_switch(fp16, fp32, T, sub, distributed):
    """process_inpainting hands complete_flow float32 flows for fp16="disable" and float16 ones for "enable"."""
    dt = torch.float32 if fp16 == "disable" else torch.float16
    eng = _StubEngine()
    ff, fb = torch.rand(1, T - 1, 2, 8, 16).to(dt), torch.rand(1, T - 1, 2, 8, 16).to(dt)
    masks = (torch.rand(1, T, 1, 8, 16) > 0.5).to(dt)
    model = types.SimpleNamespace(engine=eng)
    if distributed:   # an engine without a communicator: every rank computes the whole clip
        of, ob = PAR.complete_flow_distributed(model, (ff, fb), masks, sub, 0, 1)
    else:
        of, ob = PI.complete_flow(model, (ff, fb), masks, sub)
    assert eng.calls and all(p == fp32 for _, p in eng.calls), eng.calls
    assert len(eng.calls) == (1 if T - 1 <= sub else -(-(T - 1) // sub))   # the chunked branch passes it on every chunk
    assert of.dtype == dt and torch.equal(of, ff) and torch.equal(ob, fb)


# ---- codegen: the fp32 kernels never round to fp16 and use no hardware tanh ---------------------------------------------
@pytest.fixture(scope="module")
def sass(tmp_path_factory):
    """SASS of kernels_prop.cu and kernels_basic.cu built with the library's flags (csrc/Makefile)"""
    nvcc, cuobjdump = _cuda_tool("nvcc"), _cuda_tool("cuobjdump")
    if nvcc is None or cuobjdump is None:
        pytest.skip("nvcc / cuobjdump not found")
    d = tmp_path_factory.mktemp("rfc_sass")
    out = {}
    for src in ("kernels_prop.cu", "kernels_basic.cu"):
        obj = str(d / (src + ".o"))
        res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--use_fast_math",
                              "-c", os.path.join(CSRC, src), "-o", obj], cwd=CSRC, capture_output=True, text=True)
        assert res.returncode == 0, res.stderr[-4000:]
        out[src] = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    return out


@pytest.mark.parametrize("src,kernel", [("kernels_prop.cu", "14dcn_sample_f32"), ("kernels_prop.cu", "18rfc_pack_input_f32"),
                                        ("kernels_prop.cu", "15rfc_combine_f32"), ("kernels_basic.cu", "16upsample2x_split")])
def test_fp32_rfc_kernels_have_no_fp16_conversion_and_no_hardware_tanh(sass, src, kernel):
    funcs = re.split(r"\n\s*Function : ", sass[src])
    body = next((f for f in funcs if kernel in f.split("\n", 1)[0]), None)
    assert body is not None, f"{kernel} not found in the SASS of {src}"
    assert not re.findall(r"\b(?:F2FP\.F16|HADD2\.F32|F2F\.F16)", body), kernel
    assert not re.findall(r"\bMUFU\.TANH\b", body), kernel


def test_fp16_sampler_keeps_its_fp16_conversions(sass):
    """the codegen check can fail: the fp16 sampler it sits next to does round to fp16"""
    funcs = re.split(r"\n\s*Function : ", sass["kernels_prop.cu"])
    body = next(f for f in funcs if "10dcn_sampleILi16E" in f.split("\n", 1)[0])
    assert re.findall(r"\bF2FP\.F16", body)


# ---- the sampler's operator bound can fail ------------------------------------------------------------------------------
def _sampler_excess(**emulate):
    x, o = RFC.sampler_case(21, H=12, W=16, N=1)
    ref = RFC.im2col_reference(x, o, torch.float64)
    yard = RFC.im2col_reference(x, o, torch.float32)
    got = RFC.im2col_reference(x, o, torch.float64, **emulate) if emulate else yard
    return OPS.excess(OPS.errors(got, ref, yard))


def test_sampler_bound_accepts_an_fp32_sampler():
    assert _sampler_excess() <= 1.0


def test_sampler_bound_rejects_columns_without_their_lo_part():
    assert _sampler_excess(lo=False) > 10.0


def test_sampler_bound_rejects_a_tanh_with_2_to_minus_11_error():
    assert _sampler_excess(tanh=lambda v: torch.tanh(v) * (1 + 2.0 ** -11)) > 1.0
