"""Operator tests of the fp32 RAFT path (pp_raft_bidir_fp32), -m gpu on an H100.

Each CUDA operator of the fp32 path is compared with a float64 evaluation of the same operation on the same fp32 inputs.
The yardstick is that operation in torch fp32 on the CPU, on the same inputs; the bound for both max |d| and mean |d|
against float64 is

    kernel_err <= 8 x yardstick_err + 2^-24 * max|ref|

so an operator passes only if it is as accurate as a plain fp32 evaluation up to accumulation order.  The exception is
the GEMMs (the convolutions and the correlation volume), whose sums run on the tf32 tensor cores: their factor grows
with the length K of the sums (gemm_bound below).  The fp16 forms
of the same operators are checked against float64 on fp16-rounded inputs with 1 fp16 ulp of the reference in place of
the 2^-24 term.  tests/test_raft_fp32_host.py shows on the CPU that these bounds reject a 3xTF32 GEMM that drops one of
its terms, a tanh with fp16-level error and the one-pass instance-norm variance.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from comfyui_propainter_nodes_b200 import engine as E

DEV = "cuda:0"
RATIOS = {}      # op -> (kernel_err / yardstick_err) on max and mean |d|, printed at the end of each test


# ------------------------------------------------------------------------------------------------ bounds
def errors(out, ref, yard):
    """-> dict of max / mean |d| of the kernel and the yardstick against the float64 reference."""
    out, ref, yard = out.double(), ref.double(), yard.double()
    dk, dy = (out - ref).abs(), (yard - ref).abs()
    return dict(k_max=float(dk.max()), k_mean=float(dk.mean()), y_max=float(dy.max()), y_mean=float(dy.mean()),
                ref_max=float(ref.abs().max()))


def fp32_bound(e, factor=8):
    """(max bound, mean bound) of fp32 accuracy"""
    floor = 2.0 ** -24 * e["ref_max"]
    return factor * e["y_max"] + floor, factor * e["y_mean"] + floor


# The H100's tensor cores add each wgmma's products into the fp32 accumulator without round-to-nearest, so a tf32 GEMM's
# error grows faster with the length K of its sums than the CPU's fp32 does.  Measured on an H100 80GB HBM3 (700 W),
# kernel_err / yardstick_err of the 3xTF32 convolutions and the correlation volume is 0.45-0.69 sqrt(K) on mean |d| and
# at most 0.92 sqrt(K) on max |d| (K = filter taps x real input channels, 64..2304), so the factor is 1.25 sqrt(K), and
# never below the 8 of the other operators.  A GEMM that drops one of its three split terms is rejected by at least 3x
# at K = 2304 and by far more at small K (tests/test_raft_fp32_host.py).
GEMM_C = 1.25


def gemm_bound(K):
    return lambda e: fp32_bound(e, max(8.0, GEMM_C * math.sqrt(K)))


def excess(e, bound=fp32_bound):
    """max over (max, mean) of kernel_err / bound: <= 1 passes"""
    bmax, bmean = bound(e)
    return max(e["k_max"] / bmax if bmax > 0 else (math.inf if e["k_max"] > 0 else 0.0),
               e["k_mean"] / bmean if bmean > 0 else (math.inf if e["k_mean"] > 0 else 0.0))


def fp16_ulp(x):
    """one fp16 ulp of |x| (normal range; 2^-24 in the subnormal range)"""
    e = torch.floor(torch.log2(x.double().abs().clamp_min(2.0 ** -14)))
    return torch.pow(2.0, e - 10)


def fp16_bound_for(ref):
    u = fp16_ulp(ref)
    return lambda e: (float(u.max()) + 8 * e["y_max"], float(u.mean()) + 8 * e["y_mean"])


def assert_within(op, out, ref, yard, bound=fp32_bound):
    e = errors(out, ref, yard)
    r = (e["k_max"] / max(e["y_max"], 1e-300), e["k_mean"] / max(e["y_mean"], 1e-300))
    RATIOS[op] = r
    print(f"{op}: kernel max/mean {e['k_max']:.3e}/{e['k_mean']:.3e}  yardstick {e['y_max']:.3e}/{e['y_mean']:.3e}  "
          f"ratio {r[0]:.2f}/{r[1]:.2f}")
    assert excess(e, bound) <= 1.0, (op, e, bound(e))


# ------------------------------------------------------------------------------------------------ split tensors
def split(x):
    """fp32 [..., C] -> split tensor [..., 2C] (hi channels, then lo)"""
    hi, lo = E.split_tf32(x.float())
    return torch.cat([hi, lo], -1)


def unsplit(t):
    C = t.shape[-1] // 2
    return t[..., :C].double() + t[..., C:].double()


def check_split(t, what):
    """hi = tf32(x): low 13 mantissa bits zero; |lo| <= 2^-11 |hi| (so hi = 0 forces lo = 0)"""
    t = t.cpu()
    C = t.shape[-1] // 2
    hi, lo = t[..., :C].contiguous(), t[..., C:].contiguous()
    assert not torch.any(hi.view(torch.int32) & 0x1FFF), what + ": hi is not tf32"
    assert torch.all(lo.abs() <= 2.0 ** -11 * hi.abs()), what + ": |lo| > 2^-11 |hi|"


def wide(shape, g):
    """wide dynamic range: randn * exp(2 randn)"""
    return torch.randn(*shape, generator=g) * torch.exp(2 * torch.randn(*shape, generator=g))


# ------------------------------------------------------------------------------------------------ conv cases
# The RAFT layer shapes at odd sizes.  ins: (tensor channels, first channel read, channels read) per input; out: (tensor
# channels, first channel written) of a split output, or "fp32"; cin: real input channels when the tensor has zero
# padding channels (weights registered with a cin_map); epi: "std" / "zr" / "h".
CONV_CASES = {
    "halo_3x3_64": dict(kind="halo", N=2, H=37, W=53, ins=[(64, 0, 64)], cout=64, k=(3, 3), out=(64, 0)),
    "halo_3x3_96_res_relu": dict(kind="halo", N=2, H=23, W=41, ins=[(96, 0, 96)], cout=96, k=(3, 3), act=E.ACT_RELU,
                                 act2=E.ACT_RELU, residual=True, out=(96, 0)),
    "halo_3x3_256_192": dict(kind="halo", N=1, H=23, W=41, ins=[(256, 0, 256)], cout=192, k=(3, 3), act=E.ACT_RELU,
                             out=(192, 0)),
    "halo_3x3_256_126_hx": dict(kind="halo", N=2, H=23, W=41, ins=[(256, 0, 256)], cout=126, k=(3, 3), act=E.ACT_RELU,
                                out=(384, 256)),
    "halo_1x5_gru_zr": dict(kind="halo", N=2, H=23, W=41, ins=[(384, 0, 384)], cout=256, k=(1, 5), epi="zr",
                            out=(128, 0)),
    "halo_5x1_gru_h": dict(kind="halo", N=2, H=23, W=41, ins=[(128, 0, 128), (384, 128, 256)], cout=128, k=(5, 1),
                           epi="h", out=(384, 0)),
    "halo_3x3_256_2_fp32out": dict(kind="halo", N=2, H=23, W=41, ins=[(256, 0, 256)], cout=2, k=(3, 3), out="fp32"),
    "halo_1x1_256_576_scale": dict(kind="halo", N=2, H=23, W=41, ins=[(256, 0, 256)], cout=576, k=(1, 1), scale=0.25,
                                   out=(576, 0)),
    "halo_1x1_352_256": dict(kind="halo", N=2, H=23, W=41, ins=[(352, 0, 352)], cin=324, cout=256, k=(1, 1),
                             act=E.ACT_RELU, out=(256, 0)),
    "halo_flat_convf1": dict(kind="halo", N=1, H=1, W=2 * 23 * 41, ins=[(128, 0, 128)], cout=128, k=(1, 1),
                             act=E.ACT_RELU, out=(128, 0)),
    "igemm_7x7_s2_3": dict(kind="igemm", N=2, H=37, W=53, ins=[(4, 0, 4)], cin=3, cout=64, k=(7, 7), stride=2,
                           out=(64, 0)),
    "igemm_3x3_s2_64_96": dict(kind="igemm", N=2, H=37, W=53, ins=[(64, 0, 64)], cout=96, k=(3, 3), stride=2,
                               act=E.ACT_RELU, out=(96, 0)),
    "igemm_1x1_s2_downsample": dict(kind="igemm", N=2, H=37, W=53, ins=[(64, 0, 64)], cout=96, k=(1, 1), stride=2,
                                    out=(96, 0)),
    # output channel offset 2: not 16-byte aligned, the scalar split epilogue (vec_ok = 0)
    "igemm_scalar_epilogue": dict(kind="igemm", N=2, H=37, W=53, ins=[(64, 0, 64)], cout=30, k=(3, 3), stride=2,
                                  act=E.ACT_RELU, out=(40, 2)),
    # gate pre-activations of +-100 in every 16th channel: sigmoid and tanh must saturate, not overflow into NaN
    "halo_1x5_gru_zr_saturated": dict(kind="halo", N=2, H=23, W=41, ins=[(384, 0, 384)], cout=256, k=(1, 5), epi="zr",
                                      out=(128, 0), bias="saturate"),
    "halo_5x1_gru_h_saturated": dict(kind="halo", N=2, H=23, W=41, ins=[(128, 0, 128), (384, 128, 256)], cout=128,
                                     k=(5, 1), epi="h", out=(384, 0), bias="saturate"),
    # the epilogue alone: conv contributions ~2^-12 of the bias, so the GEMM's error is negligible and the gates' own
    # error shows against the plain fp32 bound
    "halo_1x5_gru_zr_epilogue": dict(kind="halo", N=2, H=23, W=41, ins=[(384, 0, 384)], cout=256, k=(1, 5), epi="zr",
                                     out=(128, 0), bias="epilogue"),
    "halo_5x1_gru_h_epilogue": dict(kind="halo", N=2, H=23, W=41, ins=[(128, 0, 128), (384, 128, 256)], cout=128,
                                    k=(5, 1), epi="h", out=(384, 0), bias="epilogue"),
}
GEMM_CASES = [n for n, c in CONV_CASES.items() if c.get("bias") != "epilogue"]


def conv_case(name):
    """Host inputs of a conv case: split input tensors (fp32 [N,H,W,2C]), weights, bias, epilogue operands."""
    c = dict(CONV_CASES[name])
    c.setdefault("stride", 1), c.setdefault("act", E.ACT_NONE), c.setdefault("act2", E.ACT_NONE)
    c.setdefault("scale", 1.0), c.setdefault("epi", "std"), c.setdefault("residual", False)
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    N, H, W = c["N"], c["H"], c["W"]
    tensors = []
    for C, _, _ in c["ins"]:
        x = wide((N, H, W, C), g)
        if "cin" in c:
            x[..., c["cin"]:] = 0
        tensors.append(x)
    if c["epi"] == "h":         # the GRU's hx: channels 0..127 are h, a tanh output
        tensors[1][..., :128] = torch.tanh(torch.randn(N, H, W, 128, generator=g))
    xin = torch.cat([t[..., co:co + ch] for t, (_, co, ch) in zip(tensors, c["ins"])], -1)
    cin = c.get("cin", xin.shape[-1])
    xin = xin[..., :cin]
    kh, kw = c["k"]
    # outputs of O(1) despite the wide inputs, so that the activations are neither linear nor saturated
    w = torch.randn(c["cout"], cin, kh, kw, generator=g) / (math.sqrt(cin * kh * kw) * float(xin.pow(2).mean().sqrt()))
    b = torch.randn(c["cout"], generator=g) * 0.5
    if c.get("bias") == "saturate":
        b[0::16], b[1::16] = -100.0, 100.0
    if c.get("bias") == "epilogue":
        w = w * 2.0 ** -12
        b = (torch.rand(c["cout"], generator=g) * 2 - 1) * 4
    c["K"] = cin * kh * kw
    pad = ((kh - 1) // 2, (kw - 1) // 2)
    OH = (H + 2 * pad[0] - kh) // c["stride"] + 1
    OW = (W + 2 * pad[1] - kw) // c["stride"] + 1
    aux = {}
    if c["residual"]:
        aux["res"] = torch.randn(N, OH, OW, c["cout"], generator=g)    # the scale of the conv output: it must not hide it
    if c["epi"] == "zr":
        aux["h"] = tensors[0][..., :128]
    if c["epi"] == "h":
        aux["h"] = tensors[1][..., :128]
        aux["z"] = torch.sigmoid(2 * torch.randn(N, OH, OW, 128, generator=g))
    return c, tensors, xin, w, b, pad, aux


def _act(v, a):
    if a == E.ACT_RELU:
        return torch.relu(v)
    assert a == E.ACT_NONE
    return v


def conv_reference(c, xin, w, b, pad, aux, dtype, tanh=torch.tanh, terms=None):
    """The layer in `dtype` on the CPU: dict of NHWC outputs ("out", and "rh" for the GRU z|r epilogue).
    terms: emulate a split-tf32 GEMM instead, the sum of the named products of hi / lo parts ("hi_hi", "lo_hi", "hi_lo")."""
    if terms is None:
        v = F.conv2d(xin.to(dtype).permute(0, 3, 1, 2), w.to(dtype), b.to(dtype), c["stride"], pad)
    else:
        (xh, xl), (wh, wl) = E.split_tf32(xin), E.split_tf32(w)
        parts = dict(hi_hi=(xh, wh), lo_hi=(xl, wh), hi_lo=(xh, wl))
        v = sum(F.conv2d(parts[t][0].to(dtype).permute(0, 3, 1, 2), parts[t][1].to(dtype), None, c["stride"], pad)
                for t in terms) + b.to(dtype).view(1, -1, 1, 1)
    v = v.permute(0, 2, 3, 1)
    a = {k: t.to(dtype) for k, t in aux.items()}
    if c["epi"] == "zr":
        s = torch.sigmoid(v)
        return dict(out=s[..., :128], rh=s[..., 128:] * a["h"])
    if c["epi"] == "h":
        return dict(out=(1 - a["z"]) * a["h"] + a["z"] * tanh(v))
    v = _act(v, c["act"]) * c["scale"]
    if "res" in aux:
        v = v + a["res"]
    return dict(out=_act(v, c["act2"]))


# ------------------------------------------------------------------------------------------------ GPU fixtures
@pytest.fixture(scope="module")
def eng():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    e = E.Engine(DEV, workspace_gb=1.0)
    yield e
    e.close()
    print("kernel_err / yardstick_err (max, mean):", {k: (round(a, 2), round(b, 2)) for k, (a, b) in RATIOS.items()})


def _filled(shape, g):
    """a split tensor of random values: what an op must leave alone stays recognisable"""
    return split(torch.randn(*shape, generator=g)).to(DEV)


# ------------------------------------------------------------------------------------------------ convolutions
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CONV_CASES))
def test_conv_tf32_matches_float64(eng, name):
    c, tensors, xin, w, b, pad, aux = conv_case(name)
    cin_map = None if "cin" not in c else list(range(c["cin"])) + [-1] * (c["ins"][0][0] - c["cin"])
    eng.register_conv_tf32("t32." + name, w, b, cin_map)
    g = torch.Generator().manual_seed(7)
    N = c["N"]
    ref = conv_reference(c, xin, w, b, pad, aux, torch.float64)
    yard = conv_reference(c, xin, w, b, pad, aux, torch.float32)
    OH, OW = ref["out"].shape[1:3]
    dev_in = [split(t).to(DEV) for t in tensors]
    kw = dict(stride=(c["stride"], c["stride"]), pad=pad, act=c["act"], act2=c["act2"], scale=c["scale"])
    rh = None
    if c["out"] == "fp32":
        out = torch.full((N, OH, OW, c["cout"]), float("nan"), device=DEV)
    else:
        out = _filled((N, OH, OW, c["out"][0]), g)
    if c["epi"] == "h":
        # in place, as in the GRU: hx is the second input (channels 128..383), h (channels 0..127) and the output
        out = dev_in[1]
        kw["gru_h"] = (out, 0, split(aux["z"]).to(DEV), 0)
    if c["epi"] == "zr":
        rh = _filled((N, OH, OW, 128), g)
        kw["gru_zr"] = (dev_in[0], 0, rh, 0)
    if "res" in aux:
        kw["residual"] = (split(aux["res"]).to(DEV), 0)
    before = out.clone()
    inputs = [(t, co, ch) for t, (_, co, ch) in zip(dev_in, c["ins"])]
    eng.profile_enable(True)
    eng.op_conv_tf32("t32." + name, inputs, out, 0 if c["out"] == "fp32" else c["out"][1], out_fp32=c["out"] == "fp32",
                     **kw)
    prof = eng.profile_dump()
    eng.profile_enable(False)
    torch.cuda.synchronize()
    assert any(k.startswith(f"conv:{c['kind']}:") for k in prof), prof       # the kernel this case is meant to cover
    if c["out"] == "fp32":
        got = out.cpu().double()
    else:
        C, co = c["out"]
        cols = torch.zeros(C, dtype=torch.bool)
        cols[co:co + c["cout"]] = True
        o = out.cpu()
        check_split(o, name)
        keep = torch.cat([~cols, ~cols])
        assert torch.equal(o[..., keep], before.cpu()[..., keep]), name + ": channels outside the output were written"
        got = unsplit(o)[..., co:co + c["cout"]]
    bound = fp32_bound if c.get("bias") == "epilogue" else gemm_bound(c["K"])
    assert torch.isfinite(got).all(), name + ": non-finite output"
    assert_within(name, got, ref["out"], yard["out"], bound)
    if rh is not None:
        r = rh.cpu()
        check_split(r, name + " r*h")
        assert torch.isfinite(unsplit(r)).all(), name + ": non-finite r*h"
        assert_within(name + " r*h", unsplit(r), ref["rh"], yard["rh"], bound)


# ------------------------------------------------------------------------------------------------ instance norm
IN_RATIOS = (0.0, 3.0, 30.0)


def instnorm_case(C, HW, seed=0):
    """x [3, HW, C] fp32: channel c has mean / std = IN_RATIOS[c % 3], std exp(randn); residual wide"""
    g = torch.Generator().manual_seed(seed + C + HW)
    ratio = torch.tensor([IN_RATIOS[c % 3] for c in range(C)], dtype=torch.float64)
    std = torch.exp(torch.randn(C, generator=g, dtype=torch.float64))
    x = (std * (ratio + torch.randn(3, HW, C, generator=g, dtype=torch.float64))).float()
    return x, ratio, wide((3, HW, C), g)


def instnorm_reference(x, relu, res, dtype):
    """F.instance_norm (eps 1e-5) [+ relu] [then relu(res + .)] in dtype, NHWC-flat [N, HW, C]"""
    if dtype == torch.float64:
        xd = x.double()
        m = xd.mean(1, keepdim=True)
        v = ((xd - m) ** 2).mean(1, keepdim=True)
        y = (xd - m) / torch.sqrt(v + 1e-5)
    else:
        y = F.instance_norm(x.float().permute(0, 2, 1).unsqueeze(-1)).squeeze(-1).permute(0, 2, 1)
    if relu:
        y = torch.relu(y)
    if res is not None:
        y = torch.relu(res.to(y.dtype) + y)
    return y


IN_MODES = {"plain": (False, False), "relu": (True, False), "residual_relu": (True, True)}


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(IN_MODES))
@pytest.mark.parametrize("HW", [1000, 3 * 1024 + 17, 57600])
@pytest.mark.parametrize("C", [64, 96, 128])
@pytest.mark.parametrize("fp32", [True, False], ids=["fp32", "fp16"])
def test_instnorm_matches_float64(eng, fp32, C, HW, mode):
    relu, use_res = IN_MODES[mode]
    x, ratio, res = instnorm_case(C, HW)
    if not fp32:
        x, res = x.half().float(), res.half().float()
    r = res if use_res else None
    ref = instnorm_reference(x, relu, r, torch.float64)
    yard = instnorm_reference(x, relu, r, torch.float32)
    if fp32:
        out = eng.op_instnorm(split(x).to(DEV), C, relu, None if r is None else split(r).to(DEV), fp32=True).cpu()
        check_split(out, "instnorm")
        got = unsplit(out)
    else:
        out = eng.op_instnorm(x.half().to(DEV), C, relu, None if r is None else r.half().to(DEV), fp32=False)
        got = out.cpu().double()
    for rt in IN_RATIOS:      # each mean / std group on its own: one group's yardstick must not cover another's error
        sel = ratio == rt
        tag = f"instnorm {'fp32' if fp32 else 'fp16'} C={C} HW={HW} {mode} mean/std={rt:g}"
        bound = fp32_bound if fp32 else fp16_bound_for(ref[..., sel])
        assert_within(tag, got[..., sel], ref[..., sel], yard[..., sel], bound)


# ------------------------------------------------------------------------------------------------ correlation
def corr_reference(f1, f2, h8, w8, dtype):
    """[pairs, P, 256] x 2 -> the 4 pyramid levels [pairs*P, h_l*w_l] (corr.py: matmul / 16, 2x2 average pooling)"""
    pairs, P, D = f1.shape
    c = torch.matmul(f1.to(dtype), f2.to(dtype).transpose(1, 2)) / math.sqrt(D)
    c = c.reshape(pairs * P, 1, h8, w8)
    out = [c]
    for _ in range(3):
        c = F.avg_pool2d(c, 2, stride=2)
        out.append(c)
    return [t.reshape(pairs * P, -1) for t in out]


PYR_SIZES = [(22, 40), (18, 30)]      # 18 x 30: odd pooled sizes 9 x 15, 4 x 7, 2 x 3


def pyramid_case(h8, w8, fp32=True):
    """fmap1, fmap2 [3, h8*w8, 256]: wide for fp32; for fp16 O(1), as instance-normed features are (wide ones overflow)"""
    g = torch.Generator().manual_seed(h8 * w8)
    if not fp32:
        return torch.randn(3, h8 * w8, 256, generator=g), torch.randn(3, h8 * w8, 256, generator=g)
    return wide((3, h8 * w8, 256), g), wide((3, h8 * w8, 256), g)


@pytest.mark.gpu
@pytest.mark.parametrize("size", PYR_SIZES, ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("fp32", [True, False], ids=["fp32", "fp16"])
def test_corr_pyramid_matches_float64(eng, fp32, size):
    h8, w8 = size
    f1, f2 = pyramid_case(h8, w8, fp32)
    if not fp32:
        f1, f2 = f1.half().float(), f2.half().float()
    ref = corr_reference(f1, f2, h8, w8, torch.float64)
    yard = corr_reference(f1, f2, h8, w8, torch.float32)
    if fp32:
        lv = eng.op_corr_pyramid(split(f1).to(DEV), split(f2).to(DEV), h8, w8, fp32=True)
    else:
        lv = eng.op_corr_pyramid(f1.half().to(DEV), f2.half().to(DEV), h8, w8, fp32=False)
    for l in range(4):
        tag = f"corr pyramid {'fp32' if fp32 else 'fp16'} {h8}x{w8} level {l}"
        assert lv[l].shape == ref[l].shape, (tag, lv[l].shape, ref[l].shape)
        if fp32:
            assert_within(tag, lv[l].cpu().double(), ref[l], yard[l], gemm_bound(256))
            continue
        if l > 0:   # fp16: each level is stored in fp16, so each pooling is checked on the stored level it reads
            prev = lv[l - 1].cpu().view(-1, 1, h8 >> (l - 1), w8 >> (l - 1))
            ref[l] = F.avg_pool2d(prev.double(), 2, stride=2).reshape(prev.shape[0], -1)
            yard[l] = F.avg_pool2d(prev.float(), 2, stride=2).reshape(prev.shape[0], -1)
        assert_within(tag, lv[l].cpu().double(), ref[l], yard[l], fp16_bound_for(ref[l]))


def lookup_coords(B, h8, w8, g):
    """[B, 2, h8, w8] coordinates: random, exact integers, half-integers, just inside / outside the edges, and far outside
    (beyond radius 4 at every level: all 324 outputs zero).  -> (coords, mask of the far-outside pixels)"""
    P = h8 * w8
    kind = torch.arange(B * P) % 6
    x = torch.rand(B * P, generator=g, dtype=torch.float64) * (w8 + 12) - 6
    y = torch.rand(B * P, generator=g, dtype=torch.float64) * (h8 + 12) - 6
    ix = torch.randint(-5, w8 + 5, (B * P,), generator=g).double()
    iy = torch.randint(-5, h8 + 5, (B * P,), generator=g).double()
    x = torch.where(kind == 1, ix, x)
    y = torch.where(kind == 1, iy, y)
    x = torch.where(kind == 2, ix + 0.5, x)
    y = torch.where(kind == 2, iy + 0.5, y)
    eps = torch.tensor([-1e-3, 1e-3])[torch.randint(0, 2, (B * P,), generator=g)].double()
    edge_x = torch.where(torch.rand(B * P, generator=g) < 0.5, torch.zeros(B * P, dtype=torch.float64),
                         torch.full((B * P,), w8 - 1.0, dtype=torch.float64)) + eps
    x = torch.where(kind == 3, edge_x, x)
    y = torch.where(kind == 4, torch.full((B * P,), h8 - 1.0, dtype=torch.float64) + eps, y)
    far = kind == 5
    x = torch.where(far, torch.where(torch.arange(B * P) % 12 < 6, torch.tensor(-50.0, dtype=torch.float64),
                                     torch.tensor(w8 + 50.0, dtype=torch.float64)), x)
    c = torch.stack([x, y], -1).float()
    return c.view(B, h8, w8, 2).permute(0, 3, 1, 2).contiguous(), far


def lookup_reference(pyr, coords, dtype, r=4):
    """CorrBlock.__call__ (corr.py:29-50) with bilinear_sampler (RAFT/utils/utils.py:66-80) in dtype: pyr [B*P, 1, h_l,
    w_l], coords [B, 2, h, w] -> [B*P, 324]; channel l*81 + i*9 + j samples level l at (x/2^l + i - 4, y/2^l + j - 4)"""
    b, _, h, w = coords.shape
    co = coords.to(dtype).permute(0, 2, 3, 1).reshape(b * h * w, 1, 1, 2)
    d = torch.linspace(-r, r, 2 * r + 1, dtype=dtype)
    delta = torch.stack(torch.meshgrid(d, d, indexing="ij"), dim=-1).view(1, 2 * r + 1, 2 * r + 1, 2)
    out = []
    for lvl, c in enumerate(pyr):
        pts = co / 2 ** lvl + delta
        hh, ww = c.shape[-2:]
        grid = torch.cat([2 * pts[..., 0:1] / (ww - 1) - 1, 2 * pts[..., 1:2] / (hh - 1) - 1], -1)
        out.append(F.grid_sample(c.to(dtype), grid, align_corners=True).reshape(b * h * w, -1))
    return torch.cat(out, -1)


@pytest.mark.gpu
@pytest.mark.parametrize("size", PYR_SIZES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_corr_lookup_f32_matches_float64(eng, size):
    h8, w8 = size
    B, P = 3, h8 * w8
    f1, f2 = pyramid_case(h8, w8)
    lv = eng.op_corr_pyramid(split(f1).to(DEV), split(f2).to(DEV), h8, w8, fp32=True)
    coords, far = lookup_coords(B, h8, w8, torch.Generator().manual_seed(5))
    pyr = [t.cpu().view(B * P, 1, h8 >> l, w8 >> l) for l, t in enumerate(lv)]
    ref = lookup_reference(pyr, coords, torch.float64)
    yard = lookup_reference(pyr, coords, torch.float32)
    out = eng.op_corr_lookup_f32(lv, coords.permute(0, 2, 3, 1).reshape(B * P, 2).contiguous().to(DEV), h8, w8).cpu()
    check_split(out, "corr lookup")
    assert not out[:, 324:352].any() and not out[:, 352 + 324:].any(), "padding channels 324..351 are not zero"
    got = unsplit(out)[:, :324]
    assert not got[far].any(), "points beyond radius 4 outside the map must read zeros"
    assert_within(f"corr lookup fp32 {h8}x{w8}", got, ref, yard)


# ------------------------------------------------------------------------------------------------ convex upsampling
def upsample_reference(coords1, mask, B, h8, w8, dtype):
    """RAFT.upsample_flow (raft.py:81-92) on the flow coords1 - coords0; mask [B*h8*w8, 576] -> [B, 2, 8h8, 8w8]"""
    c0 = torch.stack(torch.meshgrid(torch.arange(w8), torch.arange(h8), indexing="xy"), -1).to(dtype)
    flow = (coords1.to(dtype).view(B, h8, w8, 2) - c0).permute(0, 3, 1, 2)
    m = mask.to(dtype).view(B, h8, w8, 576).permute(0, 3, 1, 2).reshape(B, 1, 9, 8, 8, h8, w8)
    m = torch.softmax(m, dim=2)
    up = F.unfold(8 * flow, [3, 3], padding=1).view(B, 2, 9, 1, 1, h8, w8)
    up = torch.sum(m * up, dim=2).permute(0, 1, 4, 2, 5, 3)
    return up.reshape(B, 2, 8 * h8, 8 * w8)


@pytest.mark.gpu
@pytest.mark.parametrize("fp32", [True, False], ids=["fp32", "fp16"])
def test_convex_upsample_matches_float64(eng, fp32):
    B, h8, w8 = 2, 17, 23
    g = torch.Generator().manual_seed(11)
    c0 = torch.stack(torch.meshgrid(torch.arange(w8), torch.arange(h8), indexing="xy"), -1).float()
    coords1 = (c0 + (torch.rand(B, h8, w8, 2, generator=g) * 2 - 1) * 30 / 8).reshape(B * h8 * w8, 2)
    mask = (torch.rand(B * h8 * w8, 576, generator=g) * 2 - 1) * 40
    if not fp32:
        mask = mask.half().float()
    ref = upsample_reference(coords1, mask, B, h8, w8, torch.float64)
    yard = upsample_reference(coords1, mask, B, h8, w8, torch.float32)
    m_dev = split(mask).to(DEV) if fp32 else mask.half().to(DEV)
    out = eng.op_convex_upsample(coords1.to(DEV), m_dev, B, h8, w8, fp32=fp32).cpu()
    bound = fp32_bound if fp32 else fp16_bound_for(ref)
    assert_within(f"convex upsample {'fp32' if fp32 else 'fp16'}", out, ref, yard, bound)
