"""Operator tests of the fp32 flow completion (pp_flow_complete_fp32), -m gpu on an H100.

The new operators of that path, and the convolution geometries of the flow-completion network that the RAFT operator
tests (tests/test_raft_fp32_ops.py) never run, are compared with float64 on the same fp32 inputs.  The yardstick and
the bound are those of tests/test_raft_fp32_ops.py: kernel_err <= 8 x yardstick_err + 2^-24 max|ref| on max and mean
|d| (the CPU fp32 evaluation of the same operation as yardstick), max(8, 1.25 sqrt(K)) in place of 8 for the GEMMs.
tests/test_rfc_fp32_host.py shows on the CPU that the sampler's bound rejects dropped lo columns and a tanh with
2^-11 relative error.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from comfyui_propainter_nodes_b200 import engine as E
from tests import test_raft_fp32_ops as OPS

DEV = "cuda:0"
pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ references
def im2col_reference(x, offs, dtype, max_mag=5.0, tanh=torch.tanh, lo=True, flow=None, sigmoid=torch.sigmoid,
                     pos_delta=0.0):
    """torchvision's modulated deformable im2col (3x3, pad 1, 16 offset groups) in `dtype` on the CPU.
    x [N,H,W,C], offs [N,H,W,432] (offsets (g*9+k)*2 + {0: dy, 1: dx} before max_mag*tanh, modulation 288 + g*9+k
    before the sigmoid) -> columns [N,H,W,9*C] ordered (tap, channel).  lo=False emulates columns without their lo part
    (tf32-rounded).  flow [N,H,W,2] (x, y) is added to every offset (the generator's DeformableAlignment:
    offset + flow.flip(1)).  pos_delta > 0 also returns the largest change of each column when its sample position
    moves by up to pos_delta px in y and x: bilinear interpolation is bilinear inside a cell of the pixel grid, so that
    maximum is attained at a corner of the box, where the box crosses a grid line, or where two grid lines cross."""
    N, H, W, C = x.shape
    x, o = x.to(dtype), offs.to(dtype)
    cpg = C // 16
    ys = torch.arange(H, dtype=dtype).view(1, H, 1, 1)
    xs = torch.arange(W, dtype=dtype).view(1, 1, W, 1)
    flat = x.reshape(N, H * W, C)
    ch = torch.arange(C).view(16, cpg)

    def sample(py, px):                                                # [N,H,W,16] positions -> [N,H,W,16,cpg]
        inside = (py > -1) & (py < H) & (px > -1) & (px < W)
        y0, x0 = torch.floor(py), torch.floor(px)
        lh, lw = py - y0, px - x0
        hh, hw = 1 - lh, 1 - lw
        val = torch.zeros(N, H, W, 16, cpg, dtype=dtype)
        for wgt, yy, xx in ((hh * hw, y0, x0), (hh * lw, y0, x0 + 1), (lh * hw, y0 + 1, x0), (lh * lw, y0 + 1, x0 + 1)):
            ok = inside & (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
            idx = (yy.clamp(0, H - 1) * W + xx.clamp(0, W - 1)).long()   # [N,H,W,16]
            g = flat[torch.arange(N).view(N, 1, 1, 1, 1), idx.unsqueeze(-1), ch.view(1, 1, 1, 16, cpg)]
            val = val + (wgt * ok).unsqueeze(-1) * g
        return val

    def box(p):                                                        # box edges and the grid line inside, if any
        r = torch.round(p)
        return (p - pos_delta, p + pos_delta, torch.where((r - p).abs() < pos_delta, r, p))

    cols = torch.zeros(N, H, W, 9, C, dtype=dtype)
    dev = torch.zeros(N, H, W, 9, C, dtype=dtype)
    for k in range(9):
        gk = torch.arange(16) * 9 + k
        dy = max_mag * tanh(o[..., 2 * gk])
        dx = max_mag * tanh(o[..., 2 * gk + 1])
        if flow is not None:
            dy = dy + flow[..., 1:2].to(dtype)
            dx = dx + flow[..., 0:1].to(dtype)
        mod = sigmoid(o[..., 288 + gk]).unsqueeze(-1)
        py = (ys + (k // 3 - 1)) + dy                                  # [N,H,W,16]
        px = (xs + (k % 3 - 1)) + dx
        val = sample(py, px)
        cols[:, :, :, k] = (mod * val).reshape(N, H, W, C)
        if pos_delta > 0:
            d = torch.zeros_like(val)
            for qy in box(py):
                for qx in box(px):
                    d = torch.maximum(d, (sample(qy, qx) - val).abs())
            dev[:, :, :, k] = (mod * d).reshape(N, H, W, C)
    cols = cols.reshape(N, H, W, 9 * C)
    if not lo:
        cols = E.split_tf32(cols.float())[0].to(dtype)
    return (cols, dev.reshape(N, H, W, 9 * C)) if pos_delta > 0 else cols


def sampler_case(seed, H=23, W=37, N=2):
    """split inputs x0 / x1 (128 channels each) and raw offsets with saturated (+-100) offset and (+-30) mask
    pre-activations, zero offsets (integer-exact sample positions) and samples far beyond the border."""
    g = torch.Generator().manual_seed(seed)
    x = OPS.wide((N, H, W, 256), g)
    o = torch.randn(N, H, W, 432, generator=g) * 0.8
    o[..., 0:288:7] = 0.0                                                       # integer-exact positions
    o[..., 1:288:11] = 100.0 * torch.sign(torch.randn(N, H, W, 27, generator=g))  # saturated tanh: +-5 px
    o[..., 288::5] = 30.0 * torch.sign(torch.randn(N, H, W, 29, generator=g))     # saturated sigmoid
    o[:, :2, :2, :288] = -6.0                                                   # corner: samples beyond the border
    return x, o


@pytest.fixture(scope="module")
def eng():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    e = E.Engine(DEV, workspace_gb=1.0)
    yield e
    e.close()
    print("kernel_err / yardstick_err (max, mean):", {k: (round(a, 2), round(b, 2)) for k, (a, b) in OPS.RATIOS.items()})


def _sample(eng, x, o):
    d = lambda t: OPS.split(t).to(DEV)
    cols = eng.op_dcn_sample_f32(d(x[..., :128]), d(x[..., 128:]), o.float().to(DEV))
    torch.cuda.synchronize()
    return cols.cpu()


# ------------------------------------------------------------------------------------------------ sampler
def test_dcn_sampler_matches_float64(eng):
    x, o = sampler_case(11)
    cols = _sample(eng, x, o)
    OPS.check_split(cols, "dcn columns")
    got = OPS.unsplit(cols)
    assert torch.isfinite(got).all()
    ref, yard = im2col_reference(x, o, torch.float64), im2col_reference(x, o, torch.float32)
    OPS.assert_within("dcn_sample_f32", got, ref, yard)


def test_dcn_sampler_and_gemm_match_deform_conv2d(eng):
    from torchvision.ops import deform_conv2d
    x, o = sampler_case(12)
    g = torch.Generator().manual_seed(13)
    w = torch.randn(128, 256, 3, 3, generator=g) / (math.sqrt(2304) * float(x.pow(2).mean().sqrt()))
    b = torch.randn(128, generator=g) * 0.5
    eng.register_conv_tf32("t32.rfc_dcn", w.permute(0, 2, 3, 1).reshape(128, -1, 1, 1), b)
    cols = eng.op_dcn_sample_f32(OPS.split(x[..., :128]).to(DEV), OPS.split(x[..., 128:]).to(DEV), o.to(DEV))
    N, H, W = x.shape[:3]
    out = torch.full((N, H, W, 128), float("nan"), device=DEV)
    eng.op_conv_tf32("t32.rfc_dcn", [(cols, 0, 2304)], out, out_fp32=True)
    torch.cuda.synchronize()

    def ref(dtype):
        oc = o.to(dtype).permute(0, 3, 1, 2)
        off = 5.0 * torch.tanh(oc[:, :288])
        return deform_conv2d(x.to(dtype).permute(0, 3, 1, 2), off, w.to(dtype), b.to(dtype), 1, 1, 1,
                             torch.sigmoid(oc[:, 288:])).permute(0, 2, 3, 1)
    OPS.assert_within("dcn_sample_f32 + dcn gemm", out.cpu().double(), ref(torch.float64), ref(torch.float32),
                      OPS.gemm_bound(2304))


# ------------------------------------------------------------------------------------------------ upsampling
@pytest.mark.parametrize("C,H,W", [(128, 23, 37), (32, 45, 80), (64, 1, 9)])
def test_split_upsample2x_matches_float64(eng, C, H, W):
    g = torch.Generator().manual_seed(C + H)
    x = OPS.wide((2, H, W, C), g)
    out = eng.op_upsample2x_f32(OPS.split(x).to(DEV))
    torch.cuda.synchronize()
    o = out.cpu()
    OPS.check_split(o, "upsample2x")

    def ref(dtype):
        return F.interpolate(x.to(dtype).permute(0, 3, 1, 2), scale_factor=2, mode="bilinear",
                             align_corners=True).permute(0, 2, 3, 1)
    OPS.assert_within(f"upsample2x_f32 C{C}", OPS.unsplit(o), ref(torch.float64), ref(torch.float32))


# ------------------------------------------------------------------------------------------------ convolutions
# geometries of the flow-completion network the RAFT cases do not run: (N, H, W, cin (tensor channels), cout, kh, kw,
# stride, dilation, replicate, fp32 out, kernel)
GEOMS = {
    "temporal_3x1_dil2": (1, 9, 2 * 12 * 20, 64, 64, 3, 1, 1, 2, False, False, "halo"),
    "mid_3x3_dil3": (2, 23, 41, 128, 128, 3, 3, 1, 3, False, False, "halo"),
    "mid_3x3_dil2": (2, 23, 41, 128, 128, 3, 3, 1, 2, False, False, "halo"),
    "downsample_5x5_s2_replicate": (2, 40, 56, (3, 4), 32, 5, 5, 2, 1, True, False, "igemm"),
    "encoder_3x3_s2": (2, 37, 53, 32, 64, 3, 3, 2, 1, False, False, "igemm"),
    "tail_3x3_32_2_fp32out": (2, 40, 56, 32, 2, 3, 3, 1, 1, False, True, "halo"),
}


@pytest.mark.parametrize("name", list(GEOMS))
def test_rfc_conv_geometry_matches_float64(eng, name):
    N, H, W, cin, cout, kh, kw, s, dil, rep, f32out, kind = GEOMS[name]
    cin, ctensor = (cin, cin) if isinstance(cin, int) else cin
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    x = OPS.wide((N, H, W, ctensor), g)
    x[..., cin:] = 0
    w = torch.randn(cout, cin, kh, kw, generator=g) / (math.sqrt(cin * kh * kw) * float(x.pow(2).mean().sqrt()))
    b = torch.randn(cout, generator=g) * 0.5
    eng.register_conv_tf32("t32." + name, w, b, None if cin == ctensor else list(range(cin)) + [-1] * (ctensor - cin))
    pad = ((kh - 1) // 2 * dil, (kw - 1) // 2 * dil)

    def ref(dtype):
        xt = x[..., :cin].to(dtype).permute(0, 3, 1, 2)
        if rep:
            xt, p = F.pad(xt, (pad[1], pad[1], pad[0], pad[0]), mode="replicate"), 0
        else:
            p = pad
        v = F.conv2d(xt, w.to(dtype), b.to(dtype), s, p, dil)
        return F.leaky_relu(v, 0.2).permute(0, 2, 3, 1) if not f32out else v.permute(0, 2, 3, 1)
    r64, r32 = ref(torch.float64), ref(torch.float32)
    OH, OW = r64.shape[1:3]
    out = torch.full((N, OH, OW, cout if f32out else 2 * cout), float("nan"), device=DEV)
    act = dict() if f32out else dict(act=E.ACT_LRELU, slope=0.2)
    eng.profile_enable(True)
    eng.op_conv_tf32("t32." + name, [(OPS.split(x).to(DEV), 0, ctensor)], out, stride=(s, s), pad=pad,
                     dilation=(dil, dil), replicate=rep, out_fp32=f32out, **act)
    prof = eng.profile_dump()
    eng.profile_enable(False)
    torch.cuda.synchronize()
    assert any(k.startswith(f"conv:{kind}:") for k in prof), prof
    o = out.cpu()
    if not f32out:
        OPS.check_split(o, name)
        o = OPS.unsplit(o)
    assert torch.isfinite(o).all(), name
    OPS.assert_within(name, o.double(), r64, r32, OPS.gemm_bound(cin * kh * kw))
