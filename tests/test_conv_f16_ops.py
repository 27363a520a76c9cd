"""Operator tests of the fp16 convolution kernels (conv_halo_kernel, conv_gemm_kernel, conv_igemm_kernel), -m gpu on an
H100.

Every case runs one convolution through Engine.op_conv_segs, which builds the layer with PPConvCall as the stages do
(input segments, cvalid zero extension, groups, geometry, epilogue, kernel dispatch), and compares each output element
with a float64 evaluation of the same operation on the same operands: the fp16 inputs, the weights as packed (rounded to
fp16), the fp32 bias, the fp16 residual / h / z, exact activations in the epilogue's order (act1 -> scale -> + residual
-> act2; GRU z | r; (1 - z) h + z tanh q).

An fp16 output passes when |out - ref| <= 1/2 ulp16(|ref| + E) + E, E the error the kernel's fp32 value may carry before
the store (epilogue() and fp16_bound() below):
  * accumulation: 2^-22 sqrt(K) S, S = conv(|x|, |w|) + |b| in float64, K = taps x real input channels;
  * one fp32 rounding (2^-24 relative) for the bias add, the scale, the leaky slope, the residual add and the GRU blends;
  * the activations' own error: tanh.approx.f32 (tanhf under --use_fast_math) 2^-10.987 relative (PTX ISA), sigmoidf_
    and gelu_erf the terms sigmoid_err / gelu_err, whose size tests/test_conv_f16_host.py justifies by emulating the
    fast-math forms;
  * each term carried through the later epilogue steps with the activation's Lipschitz constant and |scale|.
The 1/2 ulp is the one fp16 rounding of the store.  tests/test_conv_f16_host.py shows on the CPU that this bound accepts
fp32 accumulation in the kernels' K order (round-to-nearest or round-toward-zero per k16 group) with an fp16 store, and
rejects an fp16 accumulator, a double rounding around the residual add, a dropped or repeated tap, a neighbour's bias, a
truncating store and the scale applied after the residual.

An fp32 output passes the fp32 operator tests' yardstick bound (test_raft_fp32_ops.gemm_bound).

Beyond the bound: every output tensor is prefilled with NaN, every input segment is a slice of a wider tensor whose other
channels are NaN (a read outside a segment shows as NaN in the output), nothing outside the written channel slices
changes, bit for bit, and nothing inside them is NaN.  test_plan_coverage shows that the cases reach every kernel branch
they are meant to (plans depend on the SM count: asserted on 132-SM parts).
"""
import math

import pytest
import torch
import torch.nn.functional as F

from comfyui_propainter_nodes_b200 import engine as E
from tests.test_raft_fp32_ops import errors, excess, fp16_ulp, gemm_bound

DEV = "cuda:0"
U32 = 2.0 ** -24                   # fp32 unit roundoff
ACC_C = 2.0 ** -22                 # accumulation error per sqrt(K) and unit of S
TANH_REL = 2.0 ** -10.987          # tanh.approx.f32, PTX ISA
GELU_LIP = 1.13                    # max |GELU'| = 1.1289
RATIOS = {}                        # case -> (plan label, max |d| / bound)


def sigmoid_err(v, s):
    """error of sigmoidf_ = 1 / (1 + __expf(-v)) at v (s = sigmoid(v)): ex2.approx of a rounded v log2(e), 1 + e and the
    approximate division, about 2^-21 relative, plus the rounding of the exponent, 1.5 |v| 2^-24 times the slope s (1 - s);
    both doubled"""
    return s * 2.0 ** -20 + s * (1 - s) * v.abs() * 2.0 ** -22


def gelu_err(v):
    """error of gelu_erf = 0.5 v (1 + erff(v / sqrt 2)): erff's 2 ulp, the roundings of its argument, of 1 + erf and of
    the product, 2^-22 |v| in all (absolute: 1 + erf cancels for v < 0)"""
    return 2.0 ** -22 * v.abs()


def act_exact(v, a, slope, err=None):
    """act(v) in float64, and (given err, the error of v) the error of the kernel's value of it"""
    if a == E.ACT_NONE:
        return v, err
    if a == E.ACT_RELU:
        return torch.relu(v), err
    if a == E.ACT_LRELU:
        y = torch.where(v > 0, v, v * slope)
        return y, None if err is None else max(1.0, abs(slope)) * err + U32 * torch.where(v > 0, 0 * v, y.abs())
    if a == E.ACT_SIGMOID:
        s = torch.sigmoid(v)
        return s, None if err is None else err / 4 + sigmoid_err(v, s)
    if a == E.ACT_TANH:
        t = torch.tanh(v)
        return t, None if err is None else err + TANH_REL * t.abs()
    if a == E.ACT_GELU:
        y = 0.5 * v * (1 + torch.erf(v / math.sqrt(2)))
        return y, None if err is None else GELU_LIP * err + gelu_err(v)
    raise ValueError(a)


def epilogue(c, acc, S, bias, aux, acc_err=None):
    """The layer's epilogue on float64 accumulators acc [N,OH,OW,Cout] (bias not yet added) -> dict of outputs ("out",
    and "rh" for GRU z|r), each (value, error bound E of the kernel's fp32 value before the store).  S: the accumulation
    magnitude conv(|x|, |w|) + |b|; acc_err: the accumulation error (default 2^-22 sqrt(K) S)."""
    v = acc + bias
    Ea = ACC_C * math.sqrt(c["K"]) * S if acc_err is None else acc_err
    E0 = Ea + U32 * (v.abs() + Ea)
    if c["epi"] == "zr":
        half = v.shape[-1] // 2
        s, Es = act_exact(v, E.ACT_SIGMOID, 0.0, E0)
        h = aux["h"]
        rh = s[..., half:] * h
        return dict(out=(s[..., :half], Es[..., :half]),
                    rh=(rh, h.abs() * Es[..., half:] + U32 * (rh.abs() + h.abs() * Es[..., half:])))
    if c["epi"] == "h":
        q, Eq = act_exact(v, E.ACT_TANH, 0.0, E0)
        z, h = aux["z"], aux["h"]
        o = (1 - z) * h + z * q
        return dict(out=(o, z * Eq + U32 * ((1 - z) * h.abs() + z * q.abs() + o.abs() + z * Eq)))
    y, Ey = act_exact(v, c["act"], c["slope"], E0)
    if c["scale"] != 1.0:
        y = y * c["scale"]
        Ey = abs(c["scale"]) * Ey + U32 * (y.abs() + abs(c["scale"]) * Ey)
    if "res" in aux:
        y = y + aux["res"]
        Ey = Ey + U32 * (y.abs() + Ey)
    y, Ey = act_exact(y, c["act2"], c["slope"], Ey)
    return dict(out=(y, Ey))


def fp16_bound(ref, E):
    """|out - ref| <= 1/2 ulp16(|ref| + E) + E"""
    return 0.5 * fp16_ulp(ref.abs() + E) + E


# ------------------------------------------------------------------------------------------------ cases
# Tensors: name -> channels (pixel stride); their spatial size is the input's (segments, in-place outputs) or the
# output's.  segs: (tensor, first channel, channels, gstep) -- group g reads channels co + g * gstep ...; zero: kernel
# input channels (of one group's concatenated segments) that are zero padding, weights registered with -1 there; cin_pad:
# weights registered with their input channels zero-padded to this count (the last segment then reads zero-extended,
# PPConvSeg.cvalid).  out: (tensor, co, gstep) or with out_f32 a float32 tensor.  epi "std": act / slope / scale / res
# (tensor, co) / act2; "zr": h = (tensor, co), rh = (tensor, co); "h": h = (tensor, co), z = (tensor, co).  bias "sat":
# +-60 in channels 0 / 1 mod 16; scaling "cancel": input channels scaled by 2^8 and 2^-8 in alternation.  plan: the tile
# plan the case is meant to run on a 132-SM H100 (kernel, MT / MB, BN, taps per weight stage, epilogue path, panel width).
SMALL = dict(N=2, H=37, W=29)       # < 132 tiles: MT = 1, N tiles narrowed
MT2 = dict(N=4, H=90, W=100)        # 7 x 6 x 4 = 168 tiles of 16 x 16 pixels: MT = 2
WIDE = dict(N=4, H=45, W=130)       # 204 tiles of 16 x 8 but 108 of 16 x 16: MT = 1 at the full N tile width
RAFT = dict(N=2, H=23, W=41)
BIG_FLAT = dict(N=1, H=181, W=187)  # 33,847 pixels: 133 tiles of 256 rows (conv_gemm MB = 2)

CASES = {
    # ---- conv_halo_kernel: tile widths, ragged tap groups, both epilogue paths
    "halo_bn16_tps8_tma": dict(**SMALL, t=dict(x=72, o=24, r=16), segs=[("x", 8, 64, 0)], cout=16, k=(3, 3),
                             out=("o", 8, 0), act=E.ACT_LRELU, slope=0.2, scale=0.5, res=("r", 0), act2=E.ACT_RELU,
                             plan="h MT1 BN16 taps 8+1 TMA pw16"),
    "halo_bn16_tps8_drain": dict(**SMALL, t=dict(x=72, o=24, r=20), segs=[("x", 8, 64, 0)], cout=16, k=(3, 3),
                               out=("o", 3, 0), act=E.ACT_LRELU, slope=0.1, res=("r", 1), plan="h MT1 BN16 8+1 drain"),
    "halo_bn16_mt2_tma": dict(**MT2, t=dict(x=64, o=16), segs=[("x", 0, 64, 0)], cout=16, k=(3, 3), out=("o", 0, 0),
                            act=E.ACT_RELU, plan="h MT2 BN16 8+1 TMA pw16"),
    "halo_bn16_mt2_drain_sigmoid": dict(**MT2, t=dict(x=64, o=20), segs=[("x", 0, 64, 0)], cout=16, k=(3, 3),
                                      out=("o", 2, 0), act=E.ACT_SIGMOID, bias="sat", plan="h MT2 BN16 drain"),
    "halo_bn32_tps4_tma": dict(**SMALL, t=dict(x=64, o=32), segs=[("x", 0, 64, 0)], cout=32, k=(3, 3), out=("o", 0, 0),
                             scale=2.0, plan="h MT1 BN32 taps 4+4+1 TMA pw32"),
    "halo_bn32_mt2_drain_tanh": dict(**MT2, t=dict(x=64, o=40), segs=[("x", 0, 64, 0)], cout=32, k=(3, 3),
                                   out=("o", 4, 0), act=E.ACT_TANH, bias="sat", plan="h MT2 BN32 4+4+1 drain"),
    "halo_bn48_tps2_tma": dict(**SMALL, t=dict(x=64, o=48), segs=[("x", 0, 64, 0)], cout=48, k=(3, 3), out=("o", 0, 0),
                             act=E.ACT_LRELU, slope=0.2, plan="h MT1 BN48 taps 2+2+2+2+1 TMA pw16"),
    "halo_bn64_tps2_tma_res": dict(**WIDE, t=dict(x=64, o=64, r=64), segs=[("x", 0, 64, 0)], cout=64, k=(3, 3),
                                 out=("o", 0, 0), scale=0.25, res=("r", 0), act2=E.ACT_RELU,
                                 plan="h MT1 BN64 taps 2+2+2+2+1 TMA pw64"),
    "halo_1x5_bn64_tma": dict(**WIDE, t=dict(x=64, o=64), segs=[("x", 0, 64, 0)], cout=64, k=(1, 5), out=("o", 0, 0),
                            act=E.ACT_RELU, plan="h MT1 BN64 taps 2+2+1 TMA pw64"),
    "halo_5x1_bn64_drain_gelu": dict(**WIDE, t=dict(x=64, o=72), segs=[("x", 0, 64, 0)], cout=64, k=(5, 1),
                                   out=("o", 5, 0), act=E.ACT_GELU, plan="h MT1 BN64 taps 2+2+1 drain"),
    "halo_bn96_mt2_tma": dict(**MT2, t=dict(x=64, o=96), segs=[("x", 0, 64, 0)], cout=96, k=(3, 3), out=("o", 0, 0),
                            act=E.ACT_LRELU, slope=0.1, plan="h MT2 BN96 TMA pw32"),
    "halo_bn96_mt1_drain_res": dict(**WIDE, t=dict(x=64, o=100, r=100), segs=[("x", 0, 64, 0)], cout=96, k=(3, 3),
                                  out=("o", 1, 0), scale=-0.5, res=("r", 3), plan="h MT1 BN96 drain"),
    "halo_bn128_mt2_tma": dict(**MT2, t=dict(x=64, o=128), segs=[("x", 0, 64, 0)], cout=128, k=(3, 3), out=("o", 0, 0),
                             act=E.ACT_RELU, plan="h MT2 BN128 TMA pw64"),
    "halo_bn128_mt2_drain_res": dict(**MT2, t=dict(x=64, o=136, r=136), segs=[("x", 0, 64, 0)], cout=128, k=(3, 3),
                                   out=("o", 4, 0), act=E.ACT_LRELU, slope=0.2, scale=0.5, res=("r", 2),
                                   act2=E.ACT_RELU, plan="h MT2 BN128 drain"),
    # deep halos, images smaller than one tile in one axis
    "halo_5x5_dil2": dict(**SMALL, t=dict(x=64, o=64), segs=[("x", 0, 64, 0)], cout=64, k=(5, 5), dil=2,
                        out=("o", 0, 0), act=E.ACT_RELU, plan="h MT1 BN32 taps 4x6+1 TMA, 24 x 16 patch"),
    "halo_3x3_dil3": dict(**SMALL, t=dict(x=136, o=68), segs=[("x", 8, 128, 0)], cout=64, k=(3, 3), dil=3,
                        out=("o", 2, 0), act=E.ACT_LRELU, slope=0.2, plan="h MT1 BN32 drain, 22 x 14 patch"),
    "halo_7_rows": dict(N=3, H=7, W=200, t=dict(x=64, o=64), segs=[("x", 0, 64, 0)], cout=64, k=(3, 3), out=("o", 0, 0),
                      act=E.ACT_RELU, plan="h MT1 BN32 TMA, 7 of 16 tile rows"),
    "halo_5_cols": dict(N=3, H=200, W=5, t=dict(x=64, o=72), segs=[("x", 0, 64, 0)], cout=64, k=(3, 3),
                      out=("o", 1, 0), plan="h MT1 BN32 drain, 5 of 8 tile columns"),
    # groups: packed outputs (gstep == Cout_g) take the TMA path, others the drain
    "halo_groups2_packed": dict(N=2, H=37, W=53, t=dict(x=136, o=128), segs=[("x", 8, 64, 64)], groups=2, cout=64,
                              k=(3, 3), out=("o", 0, 64), act=E.ACT_LRELU, slope=0.2, plan="h MT1 BN32 TMA groups 2"),
    "halo_groups2_unpacked": dict(N=2, H=37, W=53, t=dict(x=136, o=160), segs=[("x", 8, 64, 64)], groups=2, cout=64,
                                k=(3, 3), out=("o", 0, 80), plan="h MT1 BN32 drain groups 2"),
    "halo_groups4_packed": dict(N=2, H=37, W=53, t=dict(x=264, o=128), segs=[("x", 8, 64, 64)], groups=4, cout=32,
                              k=(3, 3), out=("o", 0, 32), act=E.ACT_RELU, plan="h MT1 BN32 TMA groups 4"),
    "halo_groups4_unpacked": dict(N=2, H=37, W=53, t=dict(x=264, o=168), segs=[("x", 8, 64, 64)], groups=4, cout=32,
                                k=(3, 3), out=("o", 8, 40), plan="h MT1 BN32 drain groups 4"),
    # flat mode (1x1 layers of less than one conv_gemm wave): partial last tile, last segment ends inside a K chunk
    "halo_flat_ragged_tma": dict(N=1, H=37, W=61, t=dict(x0=136, x1=56, o=128, r=128),
                               segs=[("x0", 8, 128, 0), ("x1", 8, 40, 0)], cout=128, k=(1, 1), out=("o", 0, 0),
                               res=("r", 0), plan="h flat MT1 BN32 TMA"),
    "halo_flat_ragged_drain": dict(N=1, H=37, W=61, t=dict(x0=136, x1=56, o=136),
                                 segs=[("x0", 8, 128, 0), ("x1", 8, 40, 0)], cout=128, k=(1, 1), out=("o", 3, 0),
                                 act=E.ACT_GELU, plan="h flat MT1 BN32 drain"),
    # GRU epilogues
    "halo_gru_zr_tma_sat": dict(**RAFT, t=dict(x=136, hx=392, z=136, rh=136), segs=[("x", 8, 128, 0)], cout=256,
                              k=(1, 5), epi="zr", out=("z", 0, 0), h=("hx", 0), rh=("rh", 8), bias="sat",
                              plan="h MT1 BN32 taps 4+1 TMA"),
    "halo_gru_zr_half48_bn96_drain": dict(**WIDE, t=dict(x=128, hx=64, z=48, rh=56), segs=[("x", 0, 128, 0)], cout=96,
                                        k=(1, 5), epi="zr", out=("z", 0, 0), h=("hx", 8), rh=("rh", 8),
                                        plan="h MT1 BN96 drain: the z | r boundary inside an N tile"),
    "halo_gru_h_drain_sat": dict(**RAFT, t=dict(x=384, hh=136, zz=136, o=136), segs=[("x", 0, 384, 0)], cout=128,
                               k=(5, 1), epi="h", out=("o", 3, 0), h=("hh", 1), z=("zz", 2), bias="sat",
                               plan="h MT1 BN32 drain"),
    # ---- input segments as the stages lay them out
    "seg_gen_encoder10": dict(N=1, H=19, W=37, t=dict(x0=272, b8=400, o=528),
                            segs=[("x0", 8, 128, 128), ("b8", 8, 192, 192)], groups=2, cout=256, k=(3, 3),
                            out=("o", 8, 256), act=E.ACT_LRELU, slope=0.2, plan="h MT1 BN32 TMA groups 2, 2 segments"),
    "seg_backbone0_cvalid": dict(**RAFT, t=dict(cur=136, prop=136, m2=16, o=128),
                               segs=[("cur", 8, 128, 0), ("prop", 0, 128, 0), ("m2", 8, 8, 0)], cin_pad=320,
                               cout=128, k=(3, 3), out=("o", 0, 0), act=E.ACT_LRELU, slope=0.2,
                               plan="h MT1 BN32 TMA, 8-channel segment zero-extended to 64"),
    "seg_fnet_layer2_cvalid": dict(N=2, H=37, W=53, t=dict(x=112, o=96, r=96), segs=[("x", 8, 96, 0)], cin_pad=128,
                                 cout=96, k=(3, 3), out=("o", 0, 0), act=E.ACT_RELU, res=("r", 0), act2=E.ACT_RELU,
                                 plan="h MT1 BN48 TMA, 96 channels zero-extended to 128"),
    "seg_gru_q_inplace": dict(**RAFT, t=dict(rh=144, hx=392, z=136), segs=[("rh", 8, 128, 0), ("hx", 128, 256, 0)],
                            cout=128, k=(5, 1), epi="h", out=("hx", 0, 0), h=("hx", 0), z=("z", 8),
                            plan="h MT1 BN32 TMA, GRU h in place over hx[:128]"),
    "seg_rfc_c0": dict(**RAFT, t=dict(a=136, b=136, c=136, o=136),
                     segs=[("a", 8, 128, 0), ("b", 8, 128, 0), ("c", 8, 128, 0)], cout=128, k=(3, 3),
                     out=("o", 5, 0), act=E.ACT_LRELU, slope=0.1, plan="h MT1 BN32 drain, 3 segments"),
    # ---- conv_igemm_kernel
    "igemm_3x3_s2": dict(N=2, H=37, W=53, t=dict(x=72, o=96), segs=[("x", 8, 64, 0)], cout=96, k=(3, 3), stride=2,
                       out=("o", 0, 0), act=E.ACT_RELU, plan="i BN96"),
    "igemm_7x7_s2_cin3": dict(N=2, H=37, W=53, t=dict(x=8, o=64), segs=[("x", 0, 8, 0)], zero=(3, 4, 5, 6, 7), cout=64,
                            k=(7, 7), stride=2, out=("o", 0, 0), act=E.ACT_LRELU, slope=0.2, plan="i BN64"),
    "igemm_5x5_s2_replicate": dict(N=2, H=37, W=53, t=dict(x=72, o=64), segs=[("x", 8, 64, 0)], cout=64, k=(5, 5),
                                 stride=2, replicate=True, out=("o", 0, 0), plan="i BN64, replicate padding"),
    "igemm_7x7_s3_40_512": dict(N=1, H=37, W=53, t=dict(x=48, o=512), segs=[("x", 8, 40, 0)], cout=512, k=(7, 7),
                              stride=3, out=("o", 0, 0), act=E.ACT_RELU, plan="i BN256"),
    "igemm_cin261_cout126": dict(N=1, H=19, W=23, t=dict(x=272, o=128), segs=[("x", 8, 264, 0)], zero=(261, 262, 263),
                               cout=126, k=(3, 3), out=("o", 0, 0), act=E.ACT_LRELU, slope=0.2,
                               plan="i BN128, Cin 261 -> 264, N tail"),
    "igemm_cin96_dil2": dict(N=2, H=37, W=53, t=dict(x=104, o=64), segs=[("x", 8, 96, 0)], cout=64, k=(3, 3), dil=2,
                           out=("o", 0, 0), act=E.ACT_RELU, plan="i BN64, Cin 96 not a multiple of 64"),
    "igemm_cout2": dict(N=2, H=37, W=53, t=dict(x=64, o=8), segs=[("x", 0, 64, 0)], cout=2, k=(3, 3), stride=2,
                      out=("o", 2, 0), plan="i BN16, N tail"),
    "igemm_cout432": dict(N=1, H=37, W=53, t=dict(x=64, o=432), segs=[("x", 0, 64, 0)], cout=432, k=(3, 3), stride=2,
                        out=("o", 0, 0), plan="i BN144"),
    "igemm_m77_tanh": dict(N=1, H=7, W=11, t=dict(x=128, o=64), segs=[("x", 0, 128, 0)], cout=64, k=(3, 3),
                         out=("o", 0, 0), act=E.ACT_TANH, plan="i BN64, M = 77 < 128"),
    "igemm_f32": dict(N=2, H=37, W=53, t=dict(x=64, o=40), segs=[("x", 0, 64, 0)], cout=30, k=(3, 3), stride=2,
                    out=("o", 2, 0), out_f32=True, plan="i BN32, fp32 output"),
    # ---- conv_gemm_kernel
    "gemm_mb1_tails": dict(N=1, H=67, W=131, t=dict(x=208, o=384), segs=[("x", 8, 200, 0)], cout=384, k=(1, 1),
                         out=("o", 0, 0), act=E.ACT_RELU, plan="g MB1: M, N and K tails"),
    "gemm_mb2_gelu": dict(**BIG_FLAT, t=dict(x=80, o=128), segs=[("x", 8, 72, 0)], cout=120, k=(1, 1), out=("o", 0, 0),
                        act=E.ACT_GELU, plan="g MB2: M, N and K tails"),
    "gemm_k1152_res": dict(N=1, H=131, W=131, t=dict(x=1152, o=136, r=136), segs=[("x", 0, 1152, 0)], cout=136,
                         k=(1, 1), out=("o", 0, 0), act=E.ACT_GELU, scale=0.5, res=("r", 0), plan="g MB1, K = 1152"),
    # ---- fp32 outputs
    "halo_fh2_f32": dict(**RAFT, t=dict(x=256, o=2), segs=[("x", 0, 256, 0)], cout=2, k=(3, 3), out=("o", 0, 0),
                       out_f32=True, plan="h MT1 BN16 drain, fp32 output"),
    # ---- cancellation: S >> |ref|, the accumulation term is what is tested
    "cancel_halo": dict(**SMALL, t=dict(x=128, o=64), segs=[("x", 0, 128, 0)], cout=64, k=(3, 3), out=("o", 0, 0),
                      scaling="cancel", plan="h MT1 BN32 TMA"),
    "cancel_igemm": dict(N=2, H=37, W=53, t=dict(x=128, o=64), segs=[("x", 0, 128, 0)], cout=64, k=(3, 3), stride=2,
                       out=("o", 0, 0), scaling="cancel", plan="i BN64"),
    "cancel_gemm": dict(**BIG_FLAT, t=dict(x=512, o=64), segs=[("x", 0, 512, 0)], cout=64, k=(1, 1), out=("o", 0, 0),
                      scaling="cancel", plan="g MB2"),
}
# A flat layer writing Cout_g channels into a slice of a wider 16-byte aligned tensor, with a wave of conv_gemm tiles.
# conv_gemm_kernel's TMA stores wrote up to the next multiple of 8 channels, over the slice's neighbours: a channel
# count that is not a multiple of 8 now runs on the halo kernel's drain epilogue, 120 stays on conv_gemm_kernel
for _co in (0, 8):
    for _n in (2, 10, 120, 126):
        CASES[f"gemm_slice_{_n}_at_{_co}"] = dict(**BIG_FLAT, t=dict(x=64, o=(_co + _n + 16 + 7) // 8 * 8),
                                                segs=[("x", 0, 64, 0)], cout=_n, k=(1, 1), out=("o", _co, 0),
                                                act=E.ACT_RELU, plan="g MB2" if _n % 8 == 0 else "h flat MT2 drain")
GPU_CASES = list(CASES)


def case(name):
    """-> (c, host tensors {name: fp16 / fp32 tensor}, float64 reference pieces).  The reference pieces: x [N,H,W,
    groups*cin] (real channels), w [cout*groups, cin, kh, kw] fp16-valued, bias, aux operands, pad."""
    c = dict(CASES[name])
    for k, v in dict(groups=1, stride=1, dil=1, replicate=False, act=E.ACT_NONE, act2=E.ACT_NONE, slope=0.0,
                     scale=1.0, epi="std", out_f32=False, zero=(), cin_pad=None).items():
        c.setdefault(k, v)
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    N, H, W, G = c["N"], c["H"], c["W"], c["groups"]
    kh, kw = c["k"]
    ph, pw = (kh - 1) // 2 * c["dil"], (kw - 1) // 2 * c["dil"]
    OH = (H + 2 * ph - c["dil"] * (kh - 1) - 1) // c["stride"] + 1
    OW = (W + 2 * pw - c["dil"] * (kw - 1) - 1) // c["stride"] + 1
    c.update(pad=(ph, pw), OH=OH, OW=OW)
    in_names = {s[0] for s in c["segs"]}
    T = {}
    for t, C in c["t"].items():
        sp = (H, W) if t in in_names else (OH, OW)
        T[t] = torch.full((N, *sp, C), float("nan"), dtype=torch.float32 if (c["out_f32"] and t == c["out"][0])
                          else torch.float16)
    # the layer input: per group, the concatenation of the segments' slices
    cin_seg = sum(s[2] for s in c["segs"])
    real = [i for i in range(cin_seg) if i not in c["zero"]]
    xs = []
    for gi in range(G):
        parts = []
        for t, co, ch, gs in c["segs"]:
            v = torch.randn(N, H, W, ch, generator=g)
            parts.append(v)
        xg = torch.cat(parts, -1)
        if c.get("scaling") == "cancel":
            xg = xg * torch.tensor([2.0 ** 8 if i % 2 == 0 else 2.0 ** -8 for i in range(cin_seg)])
        xg[..., list(c["zero"])] = 0
        xg = xg.half()
        off = 0
        for t, co, ch, gs in c["segs"]:
            T[t][..., co + gi * gs:co + gi * gs + ch] = xg[..., off:off + ch]
            off += ch
        xs.append(xg[..., real])
    x = torch.cat(xs, -1).double()
    cin = len(real)
    c["K"] = kh * kw * cin
    cout = c["cout"] * G
    rms = float(x.pow(2).mean().sqrt())
    w = (torch.randn(cout, cin, kh, kw, generator=g) / (math.sqrt(cin * kh * kw) * rms)).half().float()
    b = torch.randn(cout, generator=g) * 0.5
    if c.get("bias") == "sat":
        b[0::16], b[1::16] = -60.0, 60.0
    cin_map = [real.index(i) if i in real else -1 for i in range(cin_seg)]
    if c["cin_pad"]:
        cin_map += [-1] * (c["cin_pad"] - cin_seg)
    c["cin_map"] = cin_map
    aux = {}

    def fill(role, spec, values):
        t, co = spec
        T[t][..., co:co + values.shape[-1]] = values.to(T[t].dtype)
        aux[role] = T[t][..., co:co + values.shape[-1]].double()

    if "res" in c:
        fill("res", c["res"], torch.randn(N, OH, OW, cout, generator=g))
    if c["epi"] == "zr":
        fill("h", c["h"], torch.tanh(torch.randn(N, OH, OW, cout // 2, generator=g)))
    if c["epi"] == "h":
        fill("h", c["h"], torch.tanh(torch.randn(N, OH, OW, cout, generator=g)))
        fill("z", c["z"], torch.sigmoid(2 * torch.randn(N, OH, OW, cout, generator=g)))
    return c, T, x, w, b, aux


def conv64(c, x, w):
    """float64 convolution NHWC -> NHWC (no bias)"""
    xi = x.permute(0, 3, 1, 2)
    pad = c["pad"]
    if c["replicate"]:
        xi = F.pad(xi, (pad[1], pad[1], pad[0], pad[0]), mode="replicate")
        pad = (0, 0)
    y = F.conv2d(xi, w.to(x.dtype), None, c["stride"], pad, c["dil"], c["groups"])
    return y.permute(0, 2, 3, 1)


def reference(c, x, w, b, aux):
    """dict of output name -> (float64 value, bound E of the kernel's error before the fp16 store)"""
    acc = conv64(c, x, w.double())
    S = conv64(c, x.abs(), w.double().abs()) + b.double().abs()
    return epilogue(c, acc, S, b.double(), aux)


def written(c):
    """{tensor: list of (first channel, channels)} the layer writes"""
    G, n = c["groups"], c["cout"]
    t, co, gs = c["out"]
    if c["epi"] == "zr":
        return {t: [(co, n // 2)], c["rh"][0]: [(c["rh"][1], n // 2)]}
    return {t: [(co + gi * gs, n) for gi in range(G)] if gs else [(co, n * G)]}


def run(eng, name):
    """Launch case `name` on the GPU -> (c, host inputs before, device tensors after, plan, reference inputs)"""
    c, T, x, w, b, aux = case(name)
    eng.register_conv("f16." + name, w, b, c["groups"], c["cin_map"])
    D = {t: v.to(DEV) for t, v in T.items()}
    kw = dict(stride=(c["stride"],) * 2, pad=c["pad"], dilation=(c["dil"],) * 2, replicate=c["replicate"],
              out_f32=c["out_f32"])
    if c["epi"] == "zr":
        kw["gru_zr"] = (D[c["h"][0]], c["h"][1], D[c["rh"][0]], c["rh"][1])
    elif c["epi"] == "h":
        kw["gru_h"] = (D[c["h"][0]], c["h"][1], D[c["z"][0]], c["z"][1])
    else:
        kw.update(act=c["act"], slope=c["slope"], scale=c["scale"], act2=c["act2"])
        if "res" in c:
            kw["residual"] = (D[c["res"][0]], c["res"][1])
    segs = [(D[t], co, ch, gs) for t, co, ch, gs in c["segs"]]
    eng.op_conv_segs("f16." + name, segs, D[c["out"][0]], out_co=c["out"][1], out_gstep=c["out"][2], **kw)
    plan = eng.op_conv_last_plan()
    torch.cuda.synchronize()
    return c, T, {t: v.cpu() for t, v in D.items()}, plan, (x, w, b, aux)


def plan_label(p):
    if p["kernel"] == "h":
        return (f"h MT{p['m']} BN{p['bn']} tps{p['tps']}{' flat' if p['flat'] else ''} "
                f"{'TMA' if p['tma_out'] else 'drain'} SA{p['sa']} SB{p['sb']}")
    if p["kernel"] == "g":
        return f"g MB{p['m']} BN{p['bn']}"
    return f"{p['kernel']} BN{p['bn']} stages{p['sa']}"


def _bits(t):
    return t.contiguous().view(torch.int32 if t.dtype == torch.float32 else torch.int16)


# ------------------------------------------------------------------------------------------------ GPU tests
@pytest.fixture(scope="module")
def eng():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    e = E.Engine(DEV, workspace_gb=1.0)
    yield e
    e.close()
    if RATIOS:
        print("\nfp16 conv max |d| / bound:")
        for k, (lbl, r) in RATIOS.items():
            print(f"  {k:34s} {lbl:36s} {r:.3f}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", GPU_CASES)
def test_conv_f16_matches_float64(eng, name):
    c, before, after, plan, (x, w, b, aux) = run(eng, name)
    wr = written(c)
    # nothing outside the written channel slices changes, bit for bit; nothing inside them is NaN
    for t in before:
        keep = torch.ones(before[t].shape[-1], dtype=torch.bool)
        for co, n in wr.get(t, []):
            keep[co:co + n] = False
            assert not torch.isnan(after[t][..., co:co + n]).any(), f"{name}: NaN in {t}[{co}:{co + n}]"
        assert torch.equal(_bits(after[t][..., keep]), _bits(before[t][..., keep])), \
            f"{name}: channels of {t} outside the written slice changed ({plan_label(plan)})"
    ref = reference(c, x, w, b, aux)
    worst = 0.0
    for key, (val, Eb) in ref.items():
        t, co = (c["rh"][0], c["rh"][1]) if key == "rh" else (c["out"][0], c["out"][1])
        G, gs = c["groups"], c["out"][2]
        n = val.shape[-1] // (G if gs else 1)
        got = torch.cat([after[t][..., co + gi * gs:co + gi * gs + n] for gi in range(G)], -1) if gs else \
            after[t][..., co:co + val.shape[-1]]
        got = got.double()
        if c["out_f32"]:
            yard = reference_f32(c, x, w, b)
            e = errors(got, val, yard)
            r = excess(e, gemm_bound(c["K"]))
        else:
            r = float(((got - val).abs() / fp16_bound(val, Eb)).max())
        worst = max(worst, r)
        assert r <= 1.0, (name, key, plan_label(plan), r)
    RATIOS[name] = (plan_label(plan), worst)
    print(f"{name}: {plan_label(plan)} (meant: {c['plan']}), max |d| / bound {worst:.3f}")


def reference_f32(c, x, w, b):
    """the yardstick of an fp32 output: the layer in torch fp32 on the CPU (plain epilogue)"""
    y = conv64(c, x.float(), w.float()) + b.float()
    assert c["epi"] == "std" and c["act"] == E.ACT_NONE and "res" not in c
    return y


@pytest.mark.gpu
def test_plan_coverage(eng):
    """The cases above reach every branch of the tile heuristics they are meant to: each kernel; halo MT 1 / 2 x TMA /
    drain epilogue x panel width 64 / 32 / 16; taps per weight stage > 1 with a ragged last group; flat mode; gemm MB 1
    / 2.  A change to the heuristics that empties one of them fails here."""
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    if sms != 132:
        pytest.skip(f"the case shapes are chosen for 132 SMs; this device has {sms}")
    seen = set()
    for name in GPU_CASES:
        c, _, _, p, _ = run(eng, name)
        seen.add(p["kernel"])
        if p["kernel"] == "g":
            seen.add(("gemm MB", p["m"]))
        if p["kernel"] == "h":
            pw = 64 if p["bn"] % 64 == 0 else 32 if p["bn"] % 32 == 0 else 16
            seen.add(("halo", p["m"], "TMA" if p["tma_out"] else "drain", pw))
            taps = c["k"][0] * c["k"][1]
            if p["tps"] > 1 and taps % p["tps"] != 0:
                seen.add("ragged tap group")
            if p["flat"]:
                seen.add("flat")
    want = {"g", "h", "i", "ragged tap group", "flat", ("gemm MB", 1), ("gemm MB", 2)}
    want |= {("halo", m, path, pw) for m in (1, 2) for path in ("TMA", "drain") for pw in (64, 32, 16)}
    assert not want - seen, sorted(map(str, want - seen))
