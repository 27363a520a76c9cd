"""GPU test: conv_halo_kernel's TMA-store epilogue (fragment epilogue, operands TMA-loaded into the staging tile, TMA
stores) computes bit for bit what its drain epilogue computes.

A launch whose output or operands are not 16-byte aligned (an odd channel offset) keeps the drain epilogue, so the
same layer on the same inputs runs once per path: aligned layouts on the TMA path, the same tensors at a channel offset
of 1 on the drain path.  Each case is also checked loosely against torch's convolution, so two equally wrong paths
cannot pass."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


@pytest.fixture(scope="module")
def eng():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from comfyui_propainter_nodes_b200 import engine as E
    return E.Engine(DEV, workspace_gb=2.0)


def _register(eng, name, cin, cout, kh, kw, groups=1, seed=0):
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(cout, cin // groups, kh, kw, generator=g) / math.sqrt(cin // groups * kh * kw)
    b = torch.randn(cout, generator=g) * 0.1
    eng.register_conv(name, w, b, groups)
    return w, b


def _rand(*shape, seed=1):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g).to(DEV, torch.float16)


def _shift(t):
    """t with one more channel in front: channel c of t is channel c + 1 of the result (the drain path's layout)."""
    return torch.cat([t[..., :1], t], dim=-1).contiguous()


def _bits(t):
    return t.contiguous().view(torch.int16)


def _ref_conv(x, w, b, pad, groups=1):
    """fp32 torch convolution of NHWC fp16 x -> NHWC fp32."""
    y = F.conv2d(x.permute(0, 3, 1, 2).float(), w.to(DEV), b.to(DEV), padding=pad, groups=groups)
    return y.permute(0, 2, 3, 1)


def _both_paths(run, shape, pad_c):
    """run(out, co) on an aligned output (co = 0, TMA epilogue) and at channel offset 1 (drain epilogue)."""
    N, H, W, C = shape
    out_t = torch.full((N, H, W, C + pad_c), float("nan"), device=DEV, dtype=torch.float16)
    out_d = torch.full((N, H, W, C + pad_c + 1), float("nan"), device=DEV, dtype=torch.float16)
    run(out_t, 0)
    run(out_d, 1)
    torch.cuda.synchronize()
    return out_t, out_d


# (N, H, W, Cin, Cout, kh, kw): partial tiles at the right / bottom borders, one- and two-sub-tile CTA tiles
SHAPES = [
    (2, 37, 29, 64, 64, 3, 3),       # small launch: MT = 1, narrowed N tiles
    (8, 45, 83, 128, 128, 3, 3),     # MT = 2, BN = 128
    (6, 45, 80, 256, 192, 3, 3),     # BN = 96: 32-channel panels
    (6, 45, 80, 128, 256, 1, 5),     # 1x5
]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("act", ["none", "relu", "lrelu"])
def test_std_epilogue_matches_drain(eng, shape, act):
    from comfyui_propainter_nodes_b200 import engine as E
    N, H, W, cin, cout, kh, kw = shape
    a = {"none": E.ACT_NONE, "relu": E.ACT_RELU, "lrelu": E.ACT_LRELU}[act]
    name = f"tma_std_{'x'.join(map(str, shape))}"
    w, b = _register(eng, name, cin, cout, kh, kw)
    x = _rand(N, H, W, cin)
    pad = (kh // 2, kw // 2)
    run = lambda out, co: eng.op_conv_ex(name, x, out, out_co=co, pad=pad, act=a, slope=0.2, scale=0.5)
    t, d = _both_paths(run, (N, H, W, cout), 0)
    assert torch.equal(_bits(t[..., :cout]), _bits(d[..., 1:1 + cout]))
    ref = _ref_conv(x, w, b, pad)
    ref = {"none": ref, "relu": ref.clamp_min(0), "lrelu": F.leaky_relu(ref, 0.2)}[act] * 0.5
    assert (t[..., :cout].float() - ref).abs().max().item() < 0.05


@pytest.mark.parametrize("shape", SHAPES[:3], ids=lambda s: "x".join(map(str, s)))
def test_residual_epilogue_matches_drain(eng, shape):
    from comfyui_propainter_nodes_b200 import engine as E
    N, H, W, cin, cout, kh, kw = shape
    name = f"tma_res_{'x'.join(map(str, shape))}"
    w, b = _register(eng, name, cin, cout, kh, kw, seed=2)
    x = _rand(N, H, W, cin, seed=3)
    res = _rand(N, H, W, cout + 8, seed=4)    # residual read at channel 0 (aligned) or 1 (drain)
    ress = {0: res, 1: _shift(res)}
    pad = (kh // 2, kw // 2)

    def run(out, co):
        eng.op_conv_ex(name, x, out, out_co=co, pad=pad, act=E.ACT_LRELU, slope=0.2, residual=(ress[co], co))

    t, d = _both_paths(run, (N, H, W, cout), 0)
    assert torch.equal(_bits(t[..., :cout]), _bits(d[..., 1:1 + cout]))
    ref = F.leaky_relu(_ref_conv(x, w, b, pad), 0.2) + res[..., :cout].float()
    assert (t[..., :cout].float() - ref).abs().max().item() < 0.05


@pytest.mark.parametrize("cout,width,co", [(120, 384, 128), (64, 256, 192), (126, 384, 128)])
def test_channel_slice_output(eng, cout, width, co):
    """A layer writing `cout` channels at channel `co` of a `width`-wide tensor (convf2: 64 at 192 of 256; update.conv:
    126 at 128 of 384, which keeps the drain epilogue: its channel count ends inside a 16-byte unit); nothing else of
    the tensor changes, and cout need not be a multiple of the tile width."""
    N, H, W, cin = 8, 45, 80, 256
    name = f"tma_slice{cout}"
    w, b = _register(eng, name, cin, cout, 3, 3, seed=5)
    x = _rand(N, H, W, cin, seed=6)
    hx_t = _rand(N, H, W, width, seed=7)
    hx_d = _shift(hx_t)                      # width + 1 channels, slice at co + 1
    eng.op_conv_ex(name, x, hx_t, out_co=co, pad=(1, 1))
    eng.op_conv_ex(name, x, hx_d, out_co=co + 1, pad=(1, 1))
    torch.cuda.synchronize()
    assert torch.equal(_bits(hx_t[..., co:co + cout]), _bits(hx_d[..., co + 1:co + 1 + cout]))
    keep = _rand(N, H, W, width, seed=7)
    assert torch.equal(_bits(hx_t[..., :co]), _bits(keep[..., :co]))
    assert torch.equal(_bits(hx_t[..., co + cout:]), _bits(keep[..., co + cout:]))
    assert torch.equal(_bits(hx_d[..., co + 1 + cout:]), _bits(keep[..., co + cout:]))
    ref = _ref_conv(x, w, b, (1, 1))
    assert (hx_t[..., co:co + cout].float() - ref).abs().max().item() < 0.05


def test_grouped_output_matches_drain(eng):
    """gen.encoder.10-like: 2 groups, outputs packed per group (gstep == Cout_g)."""
    N, H, W, cin, cout, groups = 4, 45, 80, 256, 256, 2
    name = "tma_grouped"
    w, b = _register(eng, name, cin, cout, 3, 3, groups=groups, seed=8)
    x = _rand(N, H, W, cin, seed=9)
    run = lambda out, co: eng.op_conv_ex(name, x, out, out_co=co, pad=(1, 1))
    t, d = _both_paths(run, (N, H, W, cout), 0)
    assert torch.equal(_bits(t[..., :cout]), _bits(d[..., 1:1 + cout]))
    ref = _ref_conv(x, w, b, (1, 1), groups=groups)
    assert (t[..., :cout].float() - ref).abs().max().item() < 0.05


@pytest.mark.parametrize("residual", [False, True])
def test_flat_mode_matches_drain(eng, residual):
    """A 1x1 layer too small for conv_gemm_kernel runs on the halo kernel's flat mode; the last tile is partial."""
    N, H, W, cin, cout = 1, 37, 61, 128, 128
    name = "tma_flat"
    w, b = _register(eng, name, cin, cout, 1, 1, seed=10)
    x = _rand(N, H, W, cin, seed=11)
    res = _rand(N, H, W, cout + 8, seed=12)
    ress = {0: res, 1: _shift(res)}
    run = lambda out, co: eng.op_conv_ex(name, x, out, out_co=co, residual=(ress[co], co) if residual else None)
    t, d = _both_paths(run, (N, H, W, cout), 0)
    assert torch.equal(_bits(t[..., :cout]), _bits(d[..., 1:1 + cout]))
    ref = _ref_conv(x, w, b, 0) + (res[..., :cout].float() if residual else 0)
    assert (t[..., :cout].float() - ref).abs().max().item() < 0.05


@pytest.mark.parametrize("N,H,W", [(8, 45, 83), (2, 21, 19)])
def test_gru_zr_matches_drain(eng, N, H, W):
    """z -> out, r * h -> out2, with h a slice of the hidden-state tensor (1x5 taps)."""
    cin, cout = 256, 256
    name = f"tma_gru_zr_{N}"
    w, b = _register(eng, name, cin, cout, 1, 5, seed=13)
    x = _rand(N, H, W, cin, seed=14)
    hx = _rand(N, H, W, 384, seed=15)
    hxs = {0: hx, 1: _shift(hx)}
    outs = {}
    for co in (0, 1):
        z = torch.full((N, H, W, 136), float("nan"), device=DEV, dtype=torch.float16)
        rh = torch.full((N, H, W, 136), float("nan"), device=DEV, dtype=torch.float16)
        eng.op_conv_ex(name, x, z, out_co=co, pad=(0, 2), gru_zr=(hxs[co], co, rh, co))
        outs[co] = (z[..., co:co + 128], rh[..., co:co + 128])
    torch.cuda.synchronize()
    assert torch.equal(_bits(outs[0][0]), _bits(outs[1][0]))
    assert torch.equal(_bits(outs[0][1]), _bits(outs[1][1]))
    s = torch.sigmoid(_ref_conv(x, w, b, (0, 2)))
    assert (outs[0][0].float() - s[..., :128]).abs().max().item() < 0.02
    assert (outs[0][1].float() - s[..., 128:] * hx[..., :128].float()).abs().max().item() < 0.05


@pytest.mark.parametrize("N,H,W", [(8, 45, 83), (2, 21, 19)])
def test_gru_h_in_place_matches_drain(eng, N, H, W):
    """(1 - z) h + z tanh(q) written over h in place (hx[:, 0:128]), 5x1 taps."""
    cin, cout = 384, 128
    name = f"tma_gru_h_{N}"
    w, b = _register(eng, name, cin, cout, 5, 1, seed=16)
    x = _rand(N, H, W, cin, seed=17)
    zt = torch.sigmoid(_rand(N, H, W, 136, seed=18).float()).half()
    h0 = _rand(N, H, W, 384, seed=19)
    zts = {0: zt, 1: _shift(zt)}
    res = {}
    for co in (0, 1):
        hx = h0.clone() if co == 0 else _shift(h0)
        eng.op_conv_ex(name, x, hx, out_co=co, pad=(2, 0), gru_h=(hx, co, zts[co], co))
        res[co] = hx[..., co:co + 128]
    torch.cuda.synchronize()
    assert torch.equal(_bits(res[0]), _bits(res[1]))
    q = torch.tanh(_ref_conv(x, w, b, (2, 0)))
    z, h = zt[..., :128].float(), h0[..., :128].float()
    assert (res[0].float() - ((1 - z) * h + z * q)).abs().max().item() < 0.05
