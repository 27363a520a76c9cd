"""CPU tests of the fp32 RAFT path: the split-tf32 weight images, the codegen of the tf32 kernels, and proof that the
operator bounds of tests/test_raft_fp32_ops.py reject the precision losses they are there to catch.

The fp32 path stores every RAFT activation and weight as a pair hi = tf32(x), lo = x - hi and runs each GEMM as
hi*W_hi + lo*W_hi + hi*W_lo on the tf32 tensor cores (3xTF32).  That is only fp32-accurate if the split is exact, and
only fast if the tf32 halo kernel keeps the fp16 kernel's unserialized wgmma commit groups."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from comfyui_propainter_nodes_b200 import engine as E
from tests.conv_codegen import CSRC, _cuda_tool

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


# ---- the operator bounds of tests/test_raft_fp32_ops.py can fail ----------------------------------------------------
# Each GPU operator test accepts kernel_err <= 8 x yardstick_err + 2^-24 max|ref| against float64 (a factor growing with
# K for the tensor-core GEMMs).  These emulations show that the bounds accept an exact 3xTF32 GEMM and reject the
# mistakes the fp32 path can make.
from tests import test_raft_fp32_ops as OPS   # noqa: E402

ALL_TERMS = ("hi_hi", "lo_hi", "hi_lo")


def _worst_excess(outs, ref, yard, bound):
    return max(OPS.excess(OPS.errors(outs[k].float(), ref[k], yard[k]), bound) for k in ref)


@pytest.mark.parametrize("name", OPS.GEMM_CASES)
def test_conv_bound_accepts_3xtf32_and_rejects_a_dropped_term(name):
    """Rejection by >= 3x: at K = 2304 the kernel's own tensor-core accumulation error is already ~1/9 of a dropped
    term's, so no bound it passes can reject a dropped term by 10x there; at small K the margin is far larger."""
    c, _, xin, w, b, pad, aux = OPS.conv_case(name)
    ref = OPS.conv_reference(c, xin, w, b, pad, aux, torch.float64)
    yard = OPS.conv_reference(c, xin, w, b, pad, aux, torch.float32)
    bound = OPS.gemm_bound(c["K"])
    full = OPS.conv_reference(c, xin, w, b, pad, aux, torch.float64, terms=ALL_TERMS)
    assert _worst_excess(full, ref, yard, bound) <= 1.0
    for dropped in ("lo_hi", "hi_lo"):
        emu = OPS.conv_reference(c, xin, w, b, pad, aux, torch.float64, terms=[t for t in ALL_TERMS if t != dropped])
        assert _worst_excess(emu, ref, yard, bound) >= 3.0, dropped


def test_epilogue_bound_rejects_a_gru_tanh_with_fp16_level_error():
    """The epilogue-only GRU case against the plain fp32 bound: a tanh that is off by 2^-16 relative (32x below the
    worst case of tanh.approx.f32) already fails it."""
    c, _, xin, w, b, pad, aux = OPS.conv_case("halo_5x1_gru_h_epilogue")
    ref = OPS.conv_reference(c, xin, w, b, pad, aux, torch.float64)
    yard = OPS.conv_reference(c, xin, w, b, pad, aux, torch.float32)
    full = OPS.conv_reference(c, xin, w, b, pad, aux, torch.float64, terms=ALL_TERMS)
    assert _worst_excess(full, ref, yard, OPS.fp32_bound) <= 1.0
    emu = OPS.conv_reference(c, xin, w, b, pad, aux, torch.float64, terms=ALL_TERMS,
                             tanh=lambda v: torch.tanh(v) * (1 + 2.0 ** -16))
    assert _worst_excess(emu, ref, yard, OPS.fp32_bound) > 1.0


def _instnorm_sums(x, C, centre=None):
    """instnorm_stats' summation order in fp32 on one image x [HW, C]: 1024-pixel blocks, in a block lane l of
    256 / (C/2) lanes takes pixels l, l + lanes, ...; lanes are added in order, then blocks.  -> (sum, sum of squares)"""
    HW = x.shape[0]
    lanes = 256 // (C // 2)
    nblk = -(-HW // 1024)
    d = x if centre is None else (x - centre).astype(np.float32)
    xb = np.zeros((nblk * 1024, C), np.float32)
    xb[:HW] = d
    rows = -(-1024 // lanes)
    blk = np.zeros((nblk, rows * lanes, C), np.float32)      # zero pixels past the block end add nothing
    blk[:, :1024] = xb.reshape(nblk, 1024, C)
    blk = blk.reshape(nblk, rows, lanes, C)
    s = np.zeros((nblk, lanes, C), np.float32)
    q = np.zeros((nblk, lanes, C), np.float32)
    for r in range(rows):
        v = blk[:, r]
        s += v
        q += v * v
    bs, bq = np.zeros((nblk, C), np.float32), np.zeros((nblk, C), np.float32)
    for lane in range(lanes):
        bs += s[:, lane]
        bq += q[:, lane]
    ts, tq = np.zeros(C, np.float32), np.zeros(C, np.float32)
    for blk_i in range(nblk):
        ts += bs[blk_i]
        tq += bq[blk_i]
    return ts, tq


def _instnorm_emulated(x, two_pass):
    """the fp32 instance norm in the kernels' order: one-pass E[x^2] - mean^2, or the corrected two-pass statistics"""
    N, HW, C = x.shape
    inv = np.float32(1.0) / np.float32(HW)
    out = np.empty_like(x)
    for n in range(N):
        s, q = _instnorm_sums(x[n], C)
        m = s * inv
        if two_pass:
            ds, dq = _instnorm_sums(x[n], C, centre=m)
            dm = ds * inv
            m, var = m + dm, np.maximum(dq * inv - dm * dm, np.float32(0))
        else:
            var = np.maximum(q * inv - m * m, np.float32(0))
        r = (np.float32(1) / np.sqrt(var + np.float32(1e-5))).astype(np.float32)
        out[n] = (x[n] - m) * r
    return torch.from_numpy(out)


@pytest.mark.parametrize("C", [64, 96, 128])
def test_instnorm_bound_rejects_the_one_pass_variance(C):
    x, ratio, _ = OPS.instnorm_case(C, 57600)
    ref = OPS.instnorm_reference(x, False, None, torch.float64)
    yard = OPS.instnorm_reference(x, False, None, torch.float32)
    one, two = _instnorm_emulated(x.numpy(), False), _instnorm_emulated(x.numpy(), True)
    for rt in OPS.IN_RATIOS:
        sel = ratio == rt
        assert OPS.excess(OPS.errors(two[..., sel], ref[..., sel], yard[..., sel])) <= 1.0, rt
    sel = ratio == 30.0
    assert OPS.excess(OPS.errors(one[..., sel], ref[..., sel], yard[..., sel])) > 1.0


# ---- no hardware tanh on the fp32 path --------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def raft_sass(tmp_path_factory, halo_build):
    """SASS of conv_igemm.cu, conv_halo.cu and kernels_raft.cu built with the library's flags (csrc/Makefile)"""
    nvcc, cuobjdump = _cuda_tool("nvcc"), _cuda_tool("cuobjdump")
    if nvcc is None or cuobjdump is None:
        pytest.skip("nvcc / cuobjdump not found")
    objs = {"conv_halo.cu": halo_build[0]}
    d = tmp_path_factory.mktemp("raft_sass")
    for src in ("conv_igemm.cu", "kernels_raft.cu"):
        obj = str(d / (src + ".o"))
        res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--use_fast_math",
                              "-c", os.path.join(CSRC, src), "-o", obj], cwd=CSRC, capture_output=True, text=True)
        assert res.returncode == 0, res.stderr[-4000:]
        objs[src] = obj
    return {src: subprocess.run([cuobjdump, "-sass", o], capture_output=True, text=True, check=True).stdout
            for src, o in objs.items()}


# (source, mangled kernel name, hardware tanh expected): the fp16 kernels keep tanhf, whose error is below fp16 storage
@pytest.mark.parametrize("src,kernel,fast", [
    ("conv_igemm.cu", "22conv_igemm_tf32_kernelE", False), ("conv_halo.cu", "21conv_halo_tf32_kernelE", False),
    ("kernels_raft.cu", "14cnet_split_f32E", False), ("conv_igemm.cu", "17conv_igemm_kernelE", True),
    ("conv_halo.cu", "16conv_halo_kernelE", True), ("kernels_raft.cu", "10cnet_splitE", True)])
def test_fp32_path_kernels_have_no_hardware_tanh(raft_sass, src, kernel, fast):
    funcs = re.split(r"\n\s*Function : ", raft_sass[src])
    body = next((f for f in funcs if kernel in f.split("\n", 1)[0]), None)
    assert body is not None, f"{kernel} not found in the SASS of {src}"
    n = len(re.findall(r"\bMUFU\.TANH\b", body))
    assert (n > 0) if fast else (n == 0), (kernel, n)
