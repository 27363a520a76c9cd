"""CPU tests of the fp32 RAFT path: the split-tf32 weight images and the codegen of the tf32 halo-tile kernel.

The fp32 path stores every RAFT activation and weight as a pair hi = tf32(x), lo = x - hi and runs each GEMM as
hi*W_hi + lo*W_hi + hi*W_lo on the tf32 tensor cores (3xTF32).  That is only fp32-accurate if the split is exact, and
only fast if the tf32 halo kernel keeps the fp16 kernel's unserialized wgmma commit groups."""
import os
import re
import subprocess

import pytest
import torch

from comfyui_propainter_nodes_b200 import engine as E
from tests.test_halo_codegen import CSRC, _cuda_tool

TF32_KERNEL = "21conv_halo_tf32_kernelENS_10HaloParamsE"    # mangled conv_halo_tf32_kernel(HaloParams)


def _seeded(shape, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g) * torch.exp(4 * torch.randn(*shape, generator=g))


def test_split_tf32_is_exact():
    w = _seeded((256, 384, 1, 5), 0)
    hi, lo = E.split_tf32(w)
    assert torch.all((hi.view(torch.int32) & 0x1FFF) == 0)           # low 13 mantissa bits of hi are zero
    assert torch.equal(hi + lo, w)                                    # hi + lo == w exactly in fp32
    assert float((lo.abs() / w.abs().clamp_min(1e-30)).max()) <= 2.0 ** -11
    # round to nearest, ties away from zero (cvt.rna.tf32.f32)
    one_ulp = 2.0 ** -10
    t = torch.tensor([1 + one_ulp / 2, -(1 + one_ulp / 2), 1 + one_ulp / 2 - 2.0 ** -23])
    assert E.split_tf32(t)[0].tolist() == [1 + one_ulp, -(1 + one_ulp), 1.0]


@pytest.mark.parametrize("shape,cin_map", [((128, 384, 1, 5), None), ((64, 3, 7, 7), [0, 1, 2, -1]),
                                           ((256, 324, 1, 1), list(range(324)) + [-1] * 28), ((2, 256, 3, 3), None)])
def test_tf32_weight_image_holds_hi_hi_lo_rows(shape, cin_map):
    w = _seeded(shape, 1)
    packed, meta = E.pack_conv_weight_tf32(w, cin_map)
    cout, cin, kh, kw = shape
    cin_k = len(cin_map) if cin_map is not None else cin
    assert meta["cin_g"] == 2 * 3 * cin_k and meta["kh"] == kh and meta["kw"] == kw and meta["cout_g"] == cout
    num_kc, rows = packed.shape[0], packed.shape[1]
    assert rows == meta["cout_g_pad"] and packed.shape[2:] == (8, 4) and packed.dtype == torch.float32
    # undo the 128B swizzle: position p of row r holds unit p ^ (r & 7)
    pos = torch.arange(8).view(1, 8) ^ (torch.arange(rows).view(-1, 1) & 7)
    inv = torch.argsort(pos, dim=1)
    flat = torch.gather(packed, 2, inv.view(1, rows, 8, 1).expand(num_kc, rows, 8, 4))
    flat = flat.permute(1, 0, 2, 3).reshape(rows, num_kc * 32)
    idx = torch.tensor([max(i, 0) for i in cin_map]) if cin_map is not None else torch.arange(cin)
    keep = torch.tensor([float(i >= 0) for i in cin_map]) if cin_map is not None else torch.ones(cin)
    wk = w[:, idx] * keep.view(1, -1, 1, 1)
    hi, lo = E.split_tf32(wk)
    want = torch.cat([hi, hi, lo], 1).permute(0, 2, 3, 1).reshape(cout, -1)   # K = (ky, kx, pass, ci)
    K = want.shape[1]
    assert torch.equal(flat[:cout, :K], want)
    assert not flat[:cout, K:].any() and not flat[cout:].any()


@pytest.fixture(scope="module")
def halo_build(tmp_path_factory):
    nvcc = _cuda_tool("nvcc")
    if nvcc is None:
        pytest.skip("nvcc not found")
    obj = str(tmp_path_factory.mktemp("halo_tf32") / "conv_halo.o")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--use_fast_math", "-Xptxas", "-v",
           "-c", os.path.join(CSRC, "conv_halo.cu"), "-o", obj]
    res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]
    return obj, res.stdout + res.stderr


def test_tf32_halo_kernel_has_no_wgmma_serialization_warnings(halo_build):
    _, log = halo_build
    bad = [ln for ln in log.splitlines() if re.search(r"\(C75(19|20|12)\)", ln) and TF32_KERNEL in ln]
    assert not bad, "\n".join(bad[:8])


def test_tf32_halo_kernel_sass_waits_once_per_commit_group(halo_build):
    cuobjdump = _cuda_tool("cuobjdump")
    if cuobjdump is None:
        pytest.skip("cuobjdump not found")
    obj, _ = halo_build
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)
    body = next((f for f in funcs if f.startswith("_Z") and TF32_KERNEL in f.split("\n", 1)[0]), None)
    assert body is not None, "conv_halo_tf32_kernel not found in the SASS"
    hgmma = len(re.findall(r"\bHGMMA\.", body))
    depbar = len(re.findall(r"\bWARPGROUP\.DEPBAR", body))
    assert hgmma > 0 and re.search(r"HGMMA\.64x\d+x8\.F32\.TF32", body), "no tf32 HGMMA in conv_halo_tf32_kernel"
    assert 4 * depbar <= hgmma, (hgmma, depbar)
