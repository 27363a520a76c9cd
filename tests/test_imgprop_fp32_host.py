"""CPU tests of the fp32 image propagation: its C-ABI entry points, the precision the inference layer picks from the
node's fp16 switch, and the codegen of the fp32 kernels (no fp16 rounding anywhere in them)."""
import os
import re
import subprocess
import types

import pytest
import torch

from comfyui_propainter_nodes_b200 import engine as E
from comfyui_propainter_nodes_b200 import propainter_inference as PI
from tests.conv_codegen import CSRC, _cuda_tool

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_fp32_imgprop_entry_points_are_declared_and_exported():
    import ctypes
    hdr = open(os.path.join(ROOT, "include", "propainter_b200.h")).read()
    lib = ctypes.CDLL(E.LIB_PATH)
    for name in ("pp_image_propagate_fp32", "pp_op_imgprop_step_f32"):
        assert re.search(r"PP_API int " + name + r"\(", hdr), name
        assert name in E.exported_symbols()
        getattr(lib, name)


class _StubEngine:
    """Records the precision of every image_propagate call; returns the frames and masks unchanged."""

    def __init__(self):
        self.calls = []

    def image_propagate(self, frames, masks, flows_f, flows_b, fp32=False):
        self.calls.append((frames.shape[0], fp32))
        return frames.clone(), masks.clone()


@pytest.mark.parametrize("fp16,device,fp32", [("disable", "cuda", True), ("enable", "cuda", False),
                                              ("disable", "cpu", True)])
@pytest.mark.parametrize("T,sub", [(6, 80), (26, 12)])
def test_image_propagation_picks_precision_from_the_fp16_switch(fp16, device, fp32, T, sub):
    cfg = PI.ProPainterConfig(3, 4, sub, 2, fp16, T, torch.device(device), (16, 8))
    eng = _StubEngine()
    frames, masks = torch.rand(1, T, 3, 8, 16), (torch.rand(1, T, 1, 8, 16) > 0.5).float()
    flows = (torch.zeros(1, T - 1, 2, 8, 16), torch.zeros(1, T - 1, 2, 8, 16))
    uf, um = PI.image_propagation(types.SimpleNamespace(engine=eng), frames, masks, flows, cfg)
    assert eng.calls and all(p == fp32 for _, p in eng.calls), eng.calls
    assert len(eng.calls) == (1 if T <= sub else -(-T // sub))          # the chunked branch passes it on every chunk
    assert torch.equal(uf, frames) and torch.equal(um, masks)


def test_bilinear_weights_equal_atens_cuda_form_on_every_in_range_corner():
    """bilin_setup (kernels_prop.cu) weighs a corner as ATen's CPU grid_sample does: w = sx - floor(sx), west 1 - w,
    east w.  ATen's CUDA form is west (floor(sx) + 1) - sx, east sx - floor(sx).  In fp32 the two agree on every corner
    inside the image; they differ only on column -1 (floor(sx) = -1), which is out of range and weighted 0."""
    W = 64
    g = torch.Generator().manual_seed(0)
    n = 1 << 18
    k = torch.randint(-1, W + 1, (n,), generator=g).float()
    sx = torch.cat([
        torch.rand(n, generator=g) * (W + 2) - 1.5,                                  # anywhere, incl. beyond the border
        k + torch.randn(n, generator=g) * 1e-6,                                      # just either side of a texel
        k - torch.rand(n, generator=g) * 2.0 ** -20,
        -torch.rand(n, generator=g) * torch.exp2(-torch.randint(1, 40, (n,), generator=g).float()),   # (-1, 0), tiny
    ]).float()
    fx = torch.floor(sx)
    ax = sx - fx
    west, east = 1 - ax, ax                          # the kernel (and ATen CPU)
    west_c, east_c = (fx + 1) - sx, sx - fx          # ATen CUDA
    west_in, east_in = (fx >= 0) & (fx < W), (fx + 1 >= 0) & (fx + 1 < W)
    assert torch.equal(west[west_in], west_c[west_in])
    assert torch.equal(east[east_in], east_c[east_in])
    assert (west != west_c)[fx == -1].any()          # where they do differ, the corner is column -1


# ---- codegen: the fp32 kernels never round to fp16 -------------------------------------------------------------------
@pytest.fixture(scope="module")
def prop_sass(tmp_path_factory):
    """SASS of kernels_prop.cu built with the library's flags (csrc/Makefile)"""
    nvcc, cuobjdump = _cuda_tool("nvcc"), _cuda_tool("cuobjdump")
    if nvcc is None or cuobjdump is None:
        pytest.skip("nvcc / cuobjdump not found")
    obj = str(tmp_path_factory.mktemp("prop_sass") / "kernels_prop.o")
    res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--use_fast_math", "-c",
                          os.path.join(CSRC, "kernels_prop.cu"), "-o", obj], cwd=CSRC, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]
    return subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout


@pytest.mark.parametrize("kernel", ["imgprop_persistent", "imgprop_step", "imgprop_pack", "imgprop_finish",
                                    "flow_to_nhwc2"])
@pytest.mark.parametrize("storage", ["ImgF32", "ImgF16"])
def test_fp32_imgprop_kernels_have_no_fp16_conversions(prop_sass, kernel, storage):
    funcs = re.split(r"\n\s*Function : ", prop_sass)
    head = f"{len(kernel)}{kernel}INS_6{storage}E"
    body = next((f for f in funcs if head in f.split("\n", 1)[0]), None)
    assert body is not None, f"{head} not found in the SASS of kernels_prop.cu"
    n = len(re.findall(r"\b(?:F2FP\.F16|HADD2\.F32|F2F\.F16)", body))
    assert (n == 0) if storage == "ImgF32" else (n > 0), (kernel, storage, n)
