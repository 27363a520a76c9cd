"""CPU test: the error bound of tests/test_conv_f16_ops.py does its job.

An fp16 convolution is emulated on the CPU with the kernels' arithmetic: fp16 x fp16 products (exact in fp32), summed
16 at a time (one k16 step of a wgmma) and added to an fp32 accumulator in the kernels' K order (filter tap, 64-channel
chunk, k16 step), then the fp32 epilogue and one fp16 store.  The bound must accept that arithmetic, with the accumulator
rounded to nearest or toward zero, and must reject each defect below by a factor that the test prints.  A second pair of
tests emulates the fast-math forms of sigmoidf_ and gelu_erf (pp_common.cuh) and shows that their error terms cover them
and that a term of one fp32 rounding would not."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from comfyui_propainter_nodes_b200 import engine as E
from tests import test_conv_f16_ops as OPS

F32, F64 = torch.float32, torch.float64


def rz32(s):
    """float64 -> the float32 value next to it toward zero"""
    r = s.to(F32)
    over = r.double().abs() > s.abs()
    r[over] = torch.nextafter(r[over], torch.zeros_like(r[over]))
    return r


def rz16(v):
    """float32 -> fp16 rounded toward zero"""
    a = v.numpy().astype(np.float64)
    r = a.astype(np.float16)
    over = np.abs(r.astype(np.float64)) > np.abs(a)
    r[over] = np.nextafter(r[over], np.float16(0))
    return torch.from_numpy(r)


def make(C=128, cout=16, k=(3, 3), N=2, H=7, W=9, scaling=None, positive=False, act=E.ACT_LRELU, slope=0.2, scale=0.5,
         res=True, act2=E.ACT_NONE, epi="std", seed=0):
    """a small layer: fp16-valued x [N,H,W,C], w [cout,C,kh,kw], fp32 bias, fp16 epilogue operands, the case dict"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, H, W, C, generator=g, dtype=F64)
    if scaling == "cancel":
        x = x * torch.tensor([2.0 ** 8 if i % 2 == 0 else 2.0 ** -8 for i in range(C)], dtype=F64)
    if positive:
        x = x.abs()
    x = x.half().double()
    kh, kw = k
    w = torch.randn(cout, C, kh, kw, generator=g, dtype=F64) / (math.sqrt(C * kh * kw) * float(x.pow(2).mean().sqrt()))
    if positive:
        w = w.abs()
    w = w.half().double()
    b = (torch.randn(cout, generator=g) * 0.5).float()
    c = dict(K=C * kh * kw, epi=epi, act=act, slope=slope, scale=scale, act2=act2, pad=((kh - 1) // 2, (kw - 1) // 2))
    aux = {}
    if epi == "std" and res:
        aux["res"] = torch.randn(N, H, W, cout, generator=g, dtype=F64).half().double()
    if epi == "zr":
        aux["h"] = torch.tanh(torch.randn(N, H, W, cout // 2, generator=g, dtype=F64)).half().double()
    if epi == "h":
        aux["h"] = torch.tanh(torch.randn(N, H, W, cout, generator=g, dtype=F64)).half().double()
        aux["z"] = torch.sigmoid(2 * torch.randn(N, H, W, cout, generator=g, dtype=F64)).half().double()
    return c, x, w, b, aux


def accumulate(c, x, w, mode="rn", fp16_acc=False, drop_edge_tap=None, drop_tap=None, twice_tap=None):
    """The kernels' fp32 accumulation -> float64 tensor of fp32 values [N,OH,OW,cout].
    mode: "rn" / "rz" rounding of each accumulator add; fp16_acc: the accumulator rounded to fp16 after every K chunk;
    drop_edge_tap: a tap left out at the pixels of the last output row and column; drop_tap / twice_tap: a tap left out /
    summed twice everywhere."""
    N, H, W, C = x.shape
    cout, _, kh, kw = w.shape
    ph, pw = c["pad"]
    xp = F.pad(x.permute(0, 3, 1, 2), (pw, pw, ph, ph)).permute(0, 2, 3, 1)
    acc = torch.zeros(N * H * W, cout, dtype=F32)
    oy = torch.arange(H).view(1, H, 1).expand(N, H, W).reshape(-1)
    ox = torch.arange(W).view(1, 1, W).expand(N, H, W).reshape(-1)
    edge = (oy == H - 1) | (ox == W - 1)
    for tap in range(kh * kw):
        ky, kx = divmod(tap, kw)
        xt = xp[:, ky:ky + H, kx:kx + W, :].reshape(-1, C)
        prod = xt[:, None, :] * w[None, :, :, ky, kx]                   # exact: fp16 x fp16 fits fp32
        if tap == drop_tap:
            continue
        for rep in range(2 if tap == twice_tap else 1):
            for c0 in range(0, C, 64):
                for k0 in range(c0, min(c0 + 64, C), 16):
                    part = prod[:, :, k0:k0 + 16].sum(-1).to(F32).double()    # one k16 step, its sum rounded once
                    if tap == drop_edge_tap:
                        part[edge] = 0
                    s = acc.double() + part
                    acc = s.to(F32) if mode == "rn" else rz32(s)
                if fp16_acc:
                    acc = acc.half().float()
    return acc.view(N, H, W, cout).double()


def store(c, acc, b, aux, double_round=False, scale_after_res=False, bias_shift=0, store_rz=False):
    """The fp32 epilogue (conv_epilogue16's order) and the fp16 store -> float64 tensor of fp16 values.
    double_round: the conv result rounded to fp16 before the residual add; scale_after_res: (act1 + residual) * scale;
    bias_shift: each channel gets the bias of channel + bias_shift; store_rz: the store truncates."""
    v = acc.float()
    bb = torch.roll(b, -bias_shift) if bias_shift else b
    v = v + bb
    if c["epi"] == "zr":
        s = torch.sigmoid(v)
        half = v.shape[-1] // 2
        return dict(out=s[..., :half].half().double(), rh=(s[..., half:] * aux["h"].float()).half().double())
    if c["epi"] == "h":
        z, h = aux["z"].float(), aux["h"].float()
        return dict(out=((1 - z) * h + z * torch.tanh(v)).half().double())
    act = lambda t, a: OPS.act_exact(t.double(), a, c["slope"])[0].float()
    v = act(v, c["act"])
    if not scale_after_res:
        v = v * c["scale"]
    if "res" in aux:
        if double_round:
            v = v.half().float()
        v = v + aux["res"].float()
    if scale_after_res:
        v = v * c["scale"]
    v = act(v, c["act2"])
    return dict(out=(rz16(v) if store_rz else v.half()).double())


def ratio(c, x, w, b, aux, outs):
    """max over outputs and elements of |out - ref| / bound"""
    ref = OPS.reference(c | dict(stride=1, dil=1, groups=1, replicate=False), x, w.float(), b, aux)
    return max(float(((outs[k] - val).abs() / OPS.fp16_bound(val, Eb)).max()) for k, (val, Eb) in ref.items())


ACCEPT = {
    "plain 3x3 lrelu scale residual": dict(),
    "cancellation 3x3 C=256": dict(C=256, scaling="cancel", act=E.ACT_NONE, res=False),
    "positive sums 3x3 C=256 (K=2304)": dict(C=256, positive=True, act=E.ACT_NONE, scale=1.0, res=False),
    "1x1 C=1152 relu residual relu": dict(C=1152, k=(1, 1), act=E.ACT_RELU, scale=1.0, act2=E.ACT_RELU),
    "1x5 GRU z|r": dict(C=128, cout=32, k=(1, 5), epi="zr"),
    "5x1 GRU h": dict(C=128, cout=16, k=(5, 1), epi="h"),
}


@pytest.mark.parametrize("name", list(ACCEPT))
@pytest.mark.parametrize("mode", ["rn", "rz"])
def test_bound_accepts_kernel_arithmetic(name, mode):
    c, x, w, b, aux = make(**ACCEPT[name])
    r = ratio(c, x, w, b, aux, store(c, accumulate(c, x, w, mode), b, aux))
    print(f"{name} ({mode} accumulator): max |d| / bound {r:.3f}")
    assert r <= 1.0


# (layer, accumulate() defect, store() defect): 3x3 layers with 128 input channels (two K chunks); at a 16-column N tile
# the halo kernel groups the 9 taps 8 + 1 per weight stage, so tap 8 is the last tap of a ragged stage
DEFECTS = {
    "fp16 accumulator across K chunks": (dict(), dict(fp16_acc=True), dict()),
    "conv result rounded to fp16 before the residual add": (dict(act=E.ACT_NONE, scale=1.0), dict(),
                                                            dict(double_round=True)),
    "top-left tap dropped in the last output row / column": (dict(), dict(drop_edge_tap=0), dict()),
    "last tap of a ragged weight stage dropped": (dict(), dict(drop_tap=8), dict()),
    "a tap taken twice": (dict(), dict(twice_tap=4), dict()),
    "the neighbouring channel's bias": (dict(), dict(), dict(bias_shift=1)),
    "round-toward-zero store": (dict(), dict(), dict(store_rz=True)),
    "scale applied after the residual": (dict(), dict(), dict(scale_after_res=True)),
}


@pytest.mark.parametrize("name", list(DEFECTS))
def test_bound_rejects_defect(name):
    layer, acc_kw, store_kw = DEFECTS[name]
    c, x, w, b, aux = make(**layer)
    r = ratio(c, x, w, b, aux, store(c, accumulate(c, x, w, **acc_kw), b, aux, **store_kw))
    print(f"{name}: exceeds the bound by {r:.1f}x")
    assert r > 1.0


# ---- the activations' error terms
V = torch.linspace(-60, 60, 240001, dtype=F64).float()


def sigmoid_fast(v, d1, d2):
    """sigmoidf_ under --use_fast_math: 1 / (1 + ex2.approx(v * log2(e))) with the division approximate; d1 / d2 the
    relative errors given to ex2.approx and the division (2 ulp each, both signs tried)"""
    t = (-v) * torch.tensor(1.44269504, dtype=F32)
    e = (torch.exp2(t.double()) * (1 + d1)).float()
    d = 1 + e
    return ((1 / d.double()) * (1 + d2)).float()


def gelu_fast(v, d):
    """gelu_erf: 0.5 v (1 + erff(v * 0.70710678f)) with erff `d` ulp off (2 ulp, both signs tried)"""
    y = v * torch.tensor(0.70710678118654752, dtype=F32)
    erf = torch.erf(y.double()).float()
    ulp = torch.from_numpy(np.spacing(np.abs(erf.numpy())))
    return (0.5 * v) * (1 + (erf + d * ulp))


def worst(fn, combos, exact):
    return torch.stack([(fn(*cmb).double() - exact).abs() for cmb in combos]).amax(0)


def test_sigmoid_term_covers_fast_math():
    v = V.double()
    s = torch.sigmoid(v)
    err = worst(lambda a, b: sigmoid_fast(V, a, b), [(a, b) for a in (-2 ** -22, 2 ** -22) for b in (-2 ** -22, 2 ** -22)],
                s)
    r_term = float((err / OPS.sigmoid_err(v, s)).max())
    r_fp32 = float((err / (2.0 ** -24 * s)).max())
    print(f"sigmoidf_: max error / sigmoid_err {r_term:.3f}; / one fp32 rounding {r_fp32:.1e}")
    assert r_term <= 1.0 and r_fp32 > 1.0


def test_gelu_term_covers_fast_math():
    v = V.double()
    g = 0.5 * v * (1 + torch.erf(v / math.sqrt(2)))
    err = worst(lambda d: gelu_fast(V, d), [(-2,), (2,)], g)
    r_term = float((err / OPS.gelu_err(v).clamp_min(1e-300)).max())
    live = v.abs() <= 8          # where GELU is not yet 0 or the identity to fp16 precision
    r_fp32 = float((err / (2.0 ** -24 * g.abs()).clamp_min(1e-300))[live].max())
    print(f"gelu_erf: max error / gelu_err {r_term:.3f}; / one fp32 rounding {r_fp32:.1e}")
    assert r_term <= 1.0 and r_fp32 > 1.0
