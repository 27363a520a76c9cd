"""Operator and stage tests of the generator (pp_gen_run), -m gpu on an H100.

Every generator kernel computes in fp32 and rounds its result once to fp16, so each one is compared with a float64
evaluation of the same operation on the same fp16 inputs, element by element, against

    |out - ref64| <= 1 fp16 ulp of |ref64| + 2^-20 max|ref64|                                  (fp16_bound)

The bilinear samplers add a position term, what the reference's bilinear interpolation changes by when its sample
position moves by delta px: delta (|d ref / dy| + |d ref / dx|) with one-sided slopes on both sides for the feature
warp, delta = 2^-14 px (exact fp16 flows, only the normalise round trip of grid_sample is rounded), and the exact
largest change over the delta box, which also covers positions next to a grid line, for the fp16 deformable sampler,
delta = max_mag 2^-10 (tanh.approx of --use_fast_math has ~2^-11 relative error).  The window attention is bounded per query row and head by 2^-10 max |v| over the row's
keys + 1 fp16 ulp of |ref|, which covers the fp16 rounding of the softmax weights P and of the output.
tests/test_gen_ops_host.py shows on the CPU that these bounds reject the defects they are there to catch.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from comfyui_propainter_nodes_b200 import engine as E
from comfyui_propainter_nodes_b200 import weights as Wt
from oracle import propainter_oracle as O
from tests import test_raft_fp32_ops as OPS
from tests import test_rfc_fp32_ops as RFC

DEV = "cuda:0"
RATIOS = {}      # op / case -> max over elements of |out - ref64| / bound, printed at the end of the module


# ------------------------------------------------------------------------------------------------ bounds
def fp16_bound(ref, extra=None):
    ref = ref.double()
    b = OPS.fp16_ulp(ref) + 2.0 ** -20 * float(ref.abs().max())
    return b if extra is None else b + extra


def excess(out, ref, bound):
    """max over elements of |out - ref| / bound: <= 1 passes"""
    return float(((out.double() - ref.double()).abs() / bound).max())


def assert_within(op, out, ref, bound):
    out = out.double()
    assert torch.isfinite(out).all(), op
    r = excess(out, ref, bound)
    RATIOS[op] = r
    print(f"{op}: max |d| / bound {r:.3f}  max |d| {float((out - ref.double()).abs().max()):.3e}")
    assert r <= 1.0, (op, r)


# ------------------------------------------------------------------------------------------------ references
def layernorm_reference(x, gamma, beta):
    return F.layer_norm(x.double(), (x.shape[-1],), gamma.double(), beta.double(), eps=1e-5)


def layernorm_case(t, gh, gw, ratio, seed):
    """fp16 token rows whose mean / std is +-ratio (sign per row)"""
    g = torch.Generator().manual_seed(seed)
    R = t * gh * gw
    mu = ratio * torch.sign(torch.randn(R, 1, generator=g))
    x = (mu + torch.randn(R, 512, generator=g)).half()
    gamma = 0.8 + 0.4 * torch.rand(512, generator=g)
    beta = 0.05 * torch.randn(512, generator=g)
    return x, gamma, beta


def pool_reference(x, w, b):
    """x [t, nh, nw, C], w [C, 1, 4, 4], b [C] -> [t, ph, pw, C] (depthwise 4x4 stride 4, the reference's pool_layer)"""
    C = x.shape[-1]
    return F.conv2d(x.double().permute(0, 3, 1, 2), w.double(), b.double(), stride=4, groups=C).permute(0, 2, 3, 1)


def fold_reference(x, t, H, W, C, normalise, gelu, count_size=None):
    """x [t*gh*gw, 49*C] with column (ky*7 + kx)*C + c -> F.fold(7, 3, 3) [t, H, W, C] in float64, divided by
    F.fold(ones) and passed through erf-GELU on request.  count_size: output size of the overlap count (a larger
    size emulates a count that is wrong at the bottom / right border)."""
    L = x.shape[0] // t
    cols = x.double().view(t, L, 49, C).permute(0, 3, 2, 1).reshape(t, C * 49, L)
    y = F.fold(cols, (H, W), **O.T2T)
    if normalise:
        ch, cw = count_size or (H, W)
        gh, gw = (ch - 1) // 3 + 1, (cw - 1) // 3 + 1
        cnt = F.fold(torch.ones(1, 49, gh * gw, dtype=torch.float64), (ch, cw), **O.T2T)[..., :H, :W]
        y = y / cnt
    if gelu:
        y = F.gelu(y)
    return y.permute(0, 2, 3, 1)


def window_flags_reference(mask4, win_f0, win_lt):
    """mask4 [T, h4, w4] -> bool [windows, nwh*nww]: max_pool2d(7, 3, 3) (propainter.py:417-428), then the 5x9 max-pool
    over the zero-padded token grid and the sum over local frames (sparse_transformer.py:322-326)"""
    h4, w4 = mask4.shape[1:]
    gh, gw = (h4 - 1) // 3 + 1, (w4 - 1) // 3 + 1
    nh, nw = -(-gh // 5) * 5, -(-gw // 9) * 9
    out = []
    for f0, lt in zip(win_f0, win_lt):
        mp = F.max_pool2d(mask4[f0:f0 + lt, None].double(), 7, 3, 3)
        mp = F.pad(mp, (0, nw - gw, 0, nh - gh))
        out.append(F.max_pool2d(mp, (5, 9), (5, 9)).sum(0).flatten() > 0)
    return torch.stack(out)


def upsample2x_reference(x):
    """F.interpolate(x2, bilinear, align_corners=True) of x [N, H, W, C] in float64 -> (out, position term).  The kernel
    computes source coordinates as ATen does, scale * index in fp32 with scale = (H - 1) / (2H - 1) rounded: up to
    2^-23 (H - 1) px off, times the largest neighbour difference around the source pixel (either side of it)."""
    N, H, W, C = x.shape
    xd = x.double()
    ref = F.interpolate(xd.permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=True).permute(0, 2, 3, 1)
    pad = F.pad(xd.permute(0, 3, 1, 2), (1, 1, 1, 1), mode="replicate")
    dy = (pad[:, :, 1:] - pad[:, :, :-1]).abs()
    dy = torch.maximum(dy[:, :, :-1], dy[:, :, 1:])[..., 1:-1]              # [N, C, H, W]: rows y-1..y+1
    dx = (pad[..., 1:] - pad[..., :-1]).abs()
    dx = torch.maximum(dx[..., :-1], dx[..., 1:])[:, :, 1:-1]
    oy = torch.tensor([(o * (H - 1)) // max(2 * H - 1, 1) for o in range(2 * H)])
    ox = torch.tensor([(o * (W - 1)) // max(2 * W - 1, 1) for o in range(2 * W)])
    oy1, ox1 = torch.clamp(oy + 1, max=H - 1), torch.clamp(ox + 1, max=W - 1)
    near = lambda d: torch.stack([d[:, :, a][..., b] for a in (oy, oy1) for b in (ox, ox1)]).amax(0)
    pos = 2.0 ** -23 * ((H - 1) * near(dy) + (W - 1) * near(dx))
    return ref, pos.permute(0, 2, 3, 1)


def warp_reference(x, flow, h=2.0 ** -10):
    """O.warp_by_flow in float64 of x [N, H, W, C] by flow [N, H, W, 2] -> (warped, |d/dy| + |d/dx|) with one-sided
    slopes over h px (the larger side)"""
    xd, fd = x.double().permute(0, 3, 1, 2), flow.double()
    w = lambda f: O.warp_by_flow(xd, f).permute(0, 2, 3, 1)
    ref = w(fd)
    slope = 0
    for c in range(2):
        e = torch.zeros(2, dtype=torch.float64)
        e[c] = h
        slope = slope + torch.maximum((w(fd + e) - ref).abs(), (ref - w(fd - e)).abs()) / h
    return ref, slope


def fb_sides64(flow_prop, flow_check):
    """both sides of fbConsistencyCheck's test in float64: (|f_p + warp(f_c)|^2, 0.01 (|f_p|^2 + |warp|^2) + 0.5)"""
    fp, fc = flow_prop.double().permute(0, 3, 1, 2), flow_check.double().permute(0, 3, 1, 2)
    bw = O.warp_by_flow(fc, fp.permute(0, 2, 3, 1))
    lhs = ((fp + bw) ** 2).sum(1)
    rhs = 0.01 * ((fp ** 2).sum(1) + (bw ** 2).sum(1)) + 0.5
    return lhs, rhs


def dcn_case(seed, C, N=2, H=23, W=37, flow_px=0.0):
    """fp16 features, offsets and flow with saturated (+-100) offset and (+-30) modulation pre-activations, zero offsets
    (integer-exact positions without flow) and samples beyond the border in a corner (RFC.sampler_case)"""
    x, o = RFC.sampler_case(seed, H, W, N)
    g = torch.Generator().manual_seed(seed + 1)
    x = (x[..., :C] / x[..., :C].abs().amax()).half()
    flow = (flow_px * torch.randn(N, H, W, 2, generator=g)).half()
    return x, o.half(), flow


def dcn_reference(x, o, max_mag, flow=None):
    """float64 columns and their bound: fp16_bound plus the largest change of the column over sample positions within
    max_mag 2^-10 px"""
    ref, dev = RFC.im2col_reference(x.double(), o.double(), torch.float64, max_mag=max_mag,
                                    flow=None if flow is None else flow.double(), pos_delta=max_mag * 2.0 ** -10)
    return ref, fp16_bound(ref, dev)


# ---- window attention ----------------------------------------------------------------------------------------------
ATT_GRID = (8, 12)                  # token grid gh x gw, padded to 10 x 18: 2 x 2 windows, 2 x 4 pooled tokens
ATT_T = (10, 7, 4)                  # frames of the three sliding windows of one launch
ATT_FLAGS = ((1, 0, 0, 1), (1, 1, 1, 1), (0, 0, 0, 0))   # mixed, all masked, none masked


def ring_tokens(nh, nw):
    """[windows, 193]: token indices of each 5x9 window's own 45 keys and its 148 ring keys, taken from torch.roll of
    the token grid with the reference's shifts and valid_ind_rolled (sparse_transformer.py:182-197, 232-283)"""
    idx = torch.arange(nh * nw).view(nh, nw)
    valid = torch.from_numpy(Wt.rolled_valid_indices())
    rolled = [torch.roll(idx, s, (0, 1)) for s in ((-3, -5), (-3, 5), (3, -5), (3, 5))]
    out = []
    for wy in range(nh // 5):
        for wx in range(nw // 9):
            win = lambda a: a[wy * 5:wy * 5 + 5, wx * 9:wx * 9 + 9].reshape(-1)
            out.append(torch.cat([win(idx), torch.cat([win(r) for r in rolled])[valid]]))
    return torch.stack(out)


def attention_case(seed):
    """q, k, v [frames, nh*nw, 4, 128], pooled pk, pv [frames, n_pool, 4, 128] (fp16 values) of the three sliding windows
    ATT_T.  Logits are sharp: even query tokens align with u_a, odd ones with u_b (per head, orthogonal); the first ring
    key of every 5x9 window (a token of the grid wrap-around for the right-hand windows) is 20 u_a in the first two
    frames of a sliding window -- the first key tile in both parities -- and the last pooled token of the last two
    frames is 20 u_b -- the last key tile.  A masked row's dominant logit is then ~50 (log2 units) above the others'."""
    g = torch.Generator().manual_seed(seed)
    gh, gw = ATT_GRID
    nh, nw = -(-gh // 5) * 5, -(-gw // 9) * 9
    n_pool = ((nh - 4) // 4 + 1) * ((nw - 4) // 4 + 1)
    TT, ntok = sum(ATT_T), nh * nw
    basis = torch.linalg.qr(torch.randn(4, 128, 2, generator=g, dtype=torch.float64))[0]     # [4, 128, 2] orthonormal
    ua, ub = basis[..., 0].float(), basis[..., 1].float()
    q = 0.5 * torch.randn(TT, ntok, 4, 128, generator=g)
    q[:, 0::2] += 20 * ua
    q[:, 1::2] += 20 * ub
    k = torch.randn(TT, ntok, 4, 128, generator=g)
    v = torch.randn(TT, ntok, 4, 128, generator=g)
    pk = torch.randn(TT, n_pool, 4, 128, generator=g)
    pv = torch.randn(TT, n_pool, 4, 128, generator=g)
    ring = ring_tokens(nh, nw)
    f0 = 0
    for t in ATT_T:
        for f in (f0, f0 + 1):
            k[f, ring[:, 45]] = 20 * ua
        for f in (f0 + t - 2, f0 + t - 1):
            pk[f, n_pool - 1] = 20 * ub
        f0 += t
    h = lambda a: a.half()
    return dict(q=h(q), k=h(k), v=h(v), pk=h(pk), pv=h(pv), nh=nh, nw=nw, gh=gh, gw=gw, n_pool=n_pool,
                flags=torch.tensor(ATT_FLAGS, dtype=torch.int32), ring=ring, win_t=ATT_T)


def softmax_pv64(s, v):
    """float64 softmax(s) v; s in log2 units [heads, rows, keys], v [heads, keys, 128]"""
    p = torch.exp2(s - s.amax(-1, keepdim=True))
    return (p @ v) / p.sum(-1, keepdim=True)


def attention_reference(c, parity, attend=softmax_pv64, ring=None, pooled_frame=lambda f: f):
    """float64 sparse window attention of the case's sliding windows (c["win_t"] frames each, concatenated) (SparseWindowAttention, sparse_transformer.py:
    327-357) -> (out [frames, gh, gw, 512], per-element bound [frames, gh, gw, 512], log2 logit spread and position of
    the dominant key (first / last tile) of every masked query row).  Masked 5x9 windows: all t*45 queries attend, for
    the key frames parity, parity + 2, ..., to the window's own 45 tokens, its 148 ring tokens and the pooled tokens;
    unmasked windows: per frame, 45 queries to the 45 own tokens.  ring / pooled_frame / attend substitute defects."""
    ring = c["ring"] if ring is None else ring
    gh, gw, nw = c["gh"], c["gw"], c["nw"]
    hd = lambda a: a.double().permute(1, 0, 2)           # [rows, 4, 128] -> [4, rows, 128]
    scale = 1.4426950408889634 / math.sqrt(128)
    TT = sum(c["win_t"])
    out = torch.zeros(TT, gh, gw, 512, dtype=torch.float64)
    bnd = torch.zeros_like(out)
    spreads, first_tile = [], []

    def store(frames, toks, o, vmax):
        for i, (f, tok) in enumerate(zip(frames, toks)):
            y, x = divmod(int(tok), nw)
            if y < gh and x < gw:
                out[f, y, x] = o[:, i].reshape(512)
                bnd[f, y, x] = (2.0 ** -10 * vmax[:, i]).repeat_interleave(128)

    f0 = 0
    for sw, t in enumerate(c["win_t"]):
        for win in range(ring.shape[0]):
            own = ring[win, :45]
            if c["flags"][sw, win]:
                frames = [f0 + i // 45 for i in range(t * 45)]
                toks = own.repeat(t)
                qr = hd(c["q"][frames, toks])
                kf = range(f0 + parity, f0 + t, 2)
                ks = torch.cat([torch.cat([c["k"][f, ring[win]], c["pk"][pooled_frame(f)]]) for f in kf])
                vs = torch.cat([torch.cat([c["v"][f, ring[win]], c["pv"][pooled_frame(f)]]) for f in kf])
                kr, vr = hd(ks), hd(vs)
                s = (qr @ kr.transpose(1, 2)) * scale
                spreads.append(s.amax(-1) - s.amin(-1))
                first_tile.append(s.argmax(-1) < 64)
                vmax = vr.abs().amax(-1).amax(-1, keepdim=True).expand(4, len(frames))
                store(frames, toks, attend(s, vr), vmax)
            else:
                for f in range(f0, f0 + t):
                    qr, kr, vr = hd(c["q"][f, own]), hd(c["k"][f, own]), hd(c["v"][f, own])
                    s = (qr @ kr.transpose(1, 2)) * scale
                    vmax = vr.abs().amax(-1).amax(-1, keepdim=True).expand(4, 45)
                    store([f] * 45, own, attend(s, vr), vmax)
        f0 += t
    bnd = bnd + OPS.fp16_ulp(out)
    return out, bnd, torch.cat(spreads, 1), torch.cat(first_tile, 1)


def attention_pack(c):
    """the case as the kernel's operands: qkv [frames, nh*nw, 1536], pkv [frames, n_pool, 1024]"""
    TT = sum(c["win_t"])
    qkv = torch.cat([c["q"], c["k"], c["v"]], -2).reshape(TT, -1, 1536)
    pkv = torch.cat([c["pk"], c["pv"]], -2).reshape(TT, -1, 1024)
    return qkv, pkv


# ------------------------------------------------------------------------------------------------ GPU tests
@pytest.fixture(scope="module")
def eng():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    e = E.Engine(DEV, workspace_gb=1.0)
    yield e
    e.close()
    print("max |d| / bound:", {k: round(v, 3) for k, v in RATIOS.items()})


def _d(t):
    return t.contiguous().to(DEV)


LN_GRIDS = {"padded_8x12": (4, 8, 12, 10, 18), "outpaint_11x16": (4, 11, 16, 15, 18), "unpadded_10x18": (4, 10, 18, 10, 18),
            "many_rows_per_warp": (240, 10, 18, 10, 18)}


@pytest.mark.gpu
@pytest.mark.parametrize("ratio", [0, 3, 30, 100])
@pytest.mark.parametrize("grid", list(LN_GRIDS))
def test_layernorm_matches_float64(eng, grid, ratio):
    t, gh, gw, nh, nw = LN_GRIDS[grid]
    if grid == "many_rows_per_warp":
        assert t * gh * gw > 148 * 32 * 8
    x, gamma, beta = layernorm_case(t, gh, gw, ratio, seed=ratio + nh * nw + t)
    sentinel = 7.0
    out = eng.op_layernorm(_d(x), _d(gamma), _d(beta), gh, gw, nh, nw, fill=sentinel).cpu()
    pad = torch.ones(t, nh, nw, dtype=torch.bool)
    pad[:, :gh, :gw] = False
    assert bool((out[pad] == sentinel).all()), "layernorm wrote into the padding"
    ref = layernorm_reference(x, gamma, beta).view(t, gh, gw, 512)
    assert_within(f"layernorm {grid} mean/std {ratio}", out[:, :gh, :gw], ref, fp16_bound(ref))


@pytest.mark.gpu
def test_pool_tokens_matches_float64(eng):
    g = torch.Generator().manual_seed(41)
    t, nh, nw, C = 5, 10, 18, 512                         # 10 x 18 -> 2 x 4: rows / columns beyond 8 / 16 are not pooled
    x = torch.randn(t, nh, nw, C, generator=g).half()
    w = torch.full((C, 1, 4, 4), 1 / 16.0) + 0.02 * torch.randn(C, 1, 4, 4, generator=g)
    b = 0.1 * torch.randn(C, generator=g)
    out = eng.op_pool_tokens(_d(x), _d(w.view(C, 16).t()), _d(b)).cpu()
    ref = pool_reference(x, w, b)
    assert out.shape == ref.shape == (t, 2, 4, C)
    assert_within("pool_tokens", out, ref, fp16_bound(ref))


FOLD_CASES = {"ffn_8x13": (40, 8, 13, True), "ffn_10x14": (40, 10, 14, True), "ffn_12x9": (40, 12, 9, True),
              "softcomp_8x13": (128, 8, 13, False), "softcomp_10x14": (128, 10, 14, False),
              "softcomp_12x9": (128, 12, 9, False)}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(FOLD_CASES))
def test_fold_matches_float64(eng, name):
    C, H, W, ffn = FOLD_CASES[name]
    t = 3
    gh, gw = (H - 1) // 3 + 1, (W - 1) // 3 + 1
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    x = torch.randn(t * gh * gw, 49 * C, generator=g).half()
    out = eng.op_fold(_d(x), t, H, W, C, ffn, ffn).cpu()
    ref = fold_reference(x, t, H, W, C, ffn, ffn)
    assert_within("fold " + name, out, ref, fp16_bound(ref))


def window_flags_case():
    """mask4 [T, 32, 56, 8] (gh x gw = 11 x 19 tokens, padded to 15 x 27: 3 x 3 windows) with single pixels on
    receptive-field edges (y = 3 ty +- 3, x = 3 tx +- 3), on the image border and in the last (mostly padding) window;
    channel 1 holds a different mask that must not be read"""
    g = torch.Generator().manual_seed(8)
    T, h4, w4 = 12, 32, 56
    m = torch.zeros(T, h4, w4)
    for f in range(T):
        for _ in range(int(torch.randint(0, 3, (1,), generator=g))):
            ty, tx = int(torch.randint(0, 11, (1,), generator=g)), int(torch.randint(0, 19, (1,), generator=g))
            sy, sx = [int(v) for v in torch.randint(0, 2, (2,), generator=g) * 6 - 3]
            y, x = min(max(3 * ty + sy, 0), h4 - 1), min(max(3 * tx + sx, 0), w4 - 1)
            m[f, y, x] = 1.0
    m[3, h4 - 1, w4 - 1] = 1.0          # bottom-right image corner: only the last window
    m[5, 0, 30] = 1.0                    # top border
    m[7, 20, 0] = 1.0                    # left border
    m4 = torch.zeros(T, h4, w4, 8)
    m4[..., 0] = m
    m4[..., 1] = (torch.rand(T, h4, w4, generator=g) > 0.7).float()
    return m4.half()


@pytest.mark.gpu
@pytest.mark.parametrize("wins", [((0,), (1,)), ((3,), (1,)), ((0, 4, 9), (4, 1, 3)), ((2, 5, 7), (3, 2, 5))])
def test_window_flags_match_reference_exactly(eng, wins):
    m4 = window_flags_case()
    f0, lt = wins
    out = eng.op_window_flags(_d(m4), 0, f0, lt).cpu()
    ref = window_flags_reference(m4[..., 0].float(), f0, lt)
    assert torch.equal(out != 0, ref) and bool(((out == 0) | (out == 1)).all()), (out, ref)


@pytest.mark.gpu
def test_featprop_cond_matches_float64(eng):
    g = torch.Generator().manual_seed(17)
    N, H, W = 2, 24, 40
    cur = torch.randn(N, H, W, 128, generator=g).half()
    prop = torch.randn(N, H, W, 128, generator=g).half()
    # a smooth +-20 px motion per image: samples beyond the border, and a check flow that is consistent up to noise,
    # so that both outcomes of the validity test occur
    base = torch.tensor([[12.0, -7.0], [-20.0, 15.0]]).view(N, 1, 1, 2)
    fp = (base + 0.3 * torch.randn(N, H, W, 2, generator=g)).half()
    fc = (-base + 0.6 * torch.randn(N, H, W, 2, generator=g)).half()
    m2 = torch.randn(N, H, W, 8, generator=g).half()
    m2[..., :2] = (torch.rand(N, H, W, 2, generator=g) > 0.5).half()
    cond = eng.op_featprop_cond(_d(cur), _d(prop), _d(fp), _d(fc), _d(m2)).cpu()
    # copies and the zero padding: bit exact
    assert torch.equal(cond[..., :128], cur)
    assert torch.equal(cond[..., 256:258], fp)
    assert torch.equal(cond[..., 259:261], m2[..., :2])
    assert bool((cond[..., 261:] == 0).all())
    # warped features: fp16 bound + 2^-14 px of position
    ref, slope = warp_reference(prop, fp.float())
    assert_within("featprop_cond warp", cond[..., 128:256], ref, fp16_bound(ref, 2.0 ** -14 * slope))
    # validity: the reference's fp32 evaluation on the CPU, except where float64 says it is a tie to 2^-20
    valid32 = O.fb_consistency(fp.float().permute(0, 3, 1, 2), fc.float().permute(0, 3, 1, 2))[:, 0]
    lhs, rhs = fb_sides64(fp, fc)
    tie = (lhs - rhs).abs() < 2.0 ** -20 * torch.maximum(lhs, rhs)
    diff = cond[..., 258].float() != valid32
    print(f"featprop_cond validity: {int(diff.sum())} differences, {int(tie.sum())} ties to 2^-20, "
          f"{float(valid32.mean()):.2f} valid")
    assert 0.05 < float(valid32.mean()) < 0.95
    assert not bool((diff & ~tie).any())


DCN_CASES = {"generator_cpg8_flow": dict(C=128, max_mag=3.0, flow=True),
             "flow_completion_cpg16_x0_x1": dict(C=256, max_mag=5.0, flow=False)}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(DCN_CASES))
def test_fp16_dcn_sample_matches_float64(eng, name):
    cfg = DCN_CASES[name]
    x, o, flow = dcn_case(31 + cfg["C"], cfg["C"], flow_px=4.0 if cfg["flow"] else 0.0)
    if cfg["flow"]:    # the flow sits in channels 256, 257 of the 264-channel DCN condition, as in pp_gen_run
        cond = torch.randn(*x.shape[:3], 264).half()
        cond[..., 256:258] = flow
        cols = eng.op_dcn_sample(_d(x), _d(o), cfg["max_mag"], flow=(_d(cond), 256)).cpu()
        ref, bnd = dcn_reference(x, o, cfg["max_mag"], flow=flow)
    else:
        cols = eng.op_dcn_sample(_d(x[..., :128]), _d(o), cfg["max_mag"], x1=_d(x[..., 128:])).cpu()
        ref, bnd = dcn_reference(x, o, cfg["max_mag"])
    assert_within("dcn_sample " + name, cols, ref, bnd)


@pytest.mark.gpu
def test_downsample4_matches_float64(eng):
    g = torch.Generator().manual_seed(23)
    n, H, W = 3, 44, 72
    flows = 20 * torch.randn(n, 2, H, W, generator=g)
    masks = (torch.rand(n + 1, 1, H, W, generator=g) > 0.5).float()
    f4, m4 = eng.op_downsample4(_d(flows), _d(masks), mask_co=1)
    ref = F.interpolate(flows.double(), scale_factor=0.25, mode="bilinear", align_corners=False).permute(0, 2, 3, 1) / 4
    assert_within("downsample_flow4", f4.cpu(), ref, fp16_bound(ref))
    mref = F.interpolate(masks, scale_factor=0.25, mode="nearest")[:, 0]
    m4 = m4.cpu()
    assert torch.equal(m4[..., 1].float(), mref)
    assert bool((m4[..., [0, 2, 3, 4, 5, 6, 7]] == 0).all())


@pytest.mark.gpu
@pytest.mark.parametrize("C,H,W", [(128, 23, 37), (64, 12, 20), (64, 1, 9)])
def test_fp16_upsample2x_matches_float64(eng, C, H, W):
    g = torch.Generator().manual_seed(C + H + W)
    x = torch.randn(2, H, W, C, generator=g).half()
    out = eng.op_upsample2x(_d(x)).cpu()
    ref, pos = upsample2x_reference(x)
    assert_within(f"upsample2x C{C} {H}x{W}", out, ref, fp16_bound(ref, pos))


@pytest.mark.gpu
@pytest.mark.parametrize("parity", [0, 1])
def test_batched_window_attention_matches_float64(eng, parity):
    c = attention_case(3)
    qkv, pkv = attention_pack(c)
    out = eng.op_attention(_d(qkv), _d(pkv), _d(c["flags"]), list(ATT_T), c["gh"], c["gw"], c["n_pool"], parity).cpu()
    ref, bnd, spread, first = attention_reference(c, parity)
    # the case is what it claims: every masked row is sharp, both tile positions of the dominant key occur
    assert float(spread.min()) >= 30.0 and bool(first.any()) and bool((~first).any())
    assert_within(f"attention parity {parity}", out, ref, bnd)


# ------------------------------------------------------------------------------------------------ stage checks
GEN_T, GEN_H, GEN_W = 40, 96, 160             # 24 x 40 features: token grid 8 x 14, padded to 10 x 18
GEN_WINDOWS = [([0, 1, 2, 3, 4], [6, 9]), ([5, 6, 7], [0, 2]), ([8, 9], [1, 5]), ([36], [3, 8]), ([33, 34, 35], [36, 4])]
GEN_NEEDED = sorted(set(range(GEN_T)) - {10, 20, 21, 30})     # 36 frames: two encoder chunks of at most 32


def gen_clip(T=GEN_T, H=GEN_H, W=GEN_W, seed=5):
    from comfyui_propainter_nodes_b200.synthetic import synthetic_clip, synthetic_mask
    g = torch.Generator().manual_seed(seed)
    frames = (synthetic_clip(T, H, W, seed).permute(0, 3, 1, 2) * 2 - 1).contiguous()
    m = synthetic_mask(T, H, W)[:, None].contiguous()
    upd = m * (torch.rand(T, 1, H, W, generator=g) > 0.3).float()
    ff, fb = 2 * torch.randn(T - 1, 2, H, W, generator=g), 2 * torch.randn(T - 1, 2, H, W, generator=g)
    return frames, m, upd, ff, fb


def _gen_engine(workspace_gb, **kw):
    return E.Engine(DEV, workspace_gb=workspace_gb).load_weights(Wt.synthetic_raft_state_dict(),
                                                                 Wt.synthetic_rfc_state_dict(),
                                                                 Wt.synthetic_generator_state_dict(**kw))


@pytest.fixture(scope="module")
def gen_eng():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    e = _gen_engine(4.0)
    yield e
    e.close()


def _rgb(p):
    return p[..., :3].cpu()


@pytest.mark.gpu
def test_batched_gen_run_equals_single_windows(gen_eng):
    clip = [_d(a) for a in gen_clip()]
    gen_eng.gen_begin(*clip)
    batched = _rgb(gen_eng.gen_run(GEN_WINDOWS))
    single = torch.cat([_rgb(gen_eng.gen_window(nb + refs, len(nb))) for nb, refs in GEN_WINDOWS])
    gen_eng.gen_end()
    assert torch.isfinite(batched.float()).all()
    assert torch.equal(batched, single)
    # a session that encodes only the frames its windows need, packed into several encoder chunks
    gen_eng.gen_begin(*clip, frames_needed=GEN_NEEDED)
    subset = _rgb(gen_eng.gen_run(GEN_WINDOWS))
    gen_eng.gen_end()
    assert torch.equal(subset, batched)
    # an arena that holds ~ 1/2 of the windows' slots: gen_run splits the batch
    slots = sum(len(nb) + len(refs) for nb, refs in GEN_WINDOWS) * E.Engine.gen_slot_bytes(GEN_H, GEN_W)
    fixed = GEN_T * (GEN_H // 4) * (GEN_W // 4) * 288 + (64 << 20) + 24 * GEN_H * GEN_W * 2 * 200
    small = _gen_engine((fixed + slots // 2) / (1 << 30))
    try:
        small.gen_begin(*clip)
        split = _rgb(small.gen_run(GEN_WINDOWS))
        small.gen_end()
        assert small.gen_run_calls >= 2, small.gen_run_calls
    finally:
        small.close()
    assert torch.equal(split, batched)


@pytest.mark.gpu
def test_gen_run_rejects_a_window_of_one_frame(gen_eng):
    clip = [_d(a) for a in gen_clip(T=4)]
    gen_eng.gen_begin(*clip)
    try:
        with pytest.raises(RuntimeError, match="at least 2"):
            gen_eng.gen_window([2], 1)
        with pytest.raises(RuntimeError, match="at least 2"):
            gen_eng.gen_run([([0, 1], [3]), ([2], [])])
        assert torch.isfinite(gen_eng.gen_window([2, 0], 1).float()).all()     # l_t = 1 with a reference frame runs
    finally:
        gen_eng.gen_end()


@pytest.mark.gpu
def test_sharp_attention_window_matches_float64_oracle():
    """gen_window with attention logits 9x the default variance (attn_logit_gain 3), at a padded token grid, against
    InpaintGenerator.forward in float64 on the CPU"""
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    T, H, W, l_t = 7, 96, 160, 5
    frames, m, upd, ff, fb = gen_clip(T, H, W, seed=9)
    sd = Wt.synthetic_generator_state_dict(attn_logit_gain=3.0)
    e = _gen_engine(2.0, attn_logit_gain=3.0)
    try:
        e.gen_begin(*[_d(a) for a in (frames, m, upd, ff, fb)])
        pred = e.gen_window(list(range(T)), l_t)[..., :3].permute(0, 3, 1, 2).float().cpu()
        e.gen_end()
    finally:
        e.close()
    sd64 = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
    d = lambda a: a.double()[None]
    ref = O.inpaint_window(sd64, d(frames), (d(ff[:l_t - 1]), d(fb[:l_t - 1])), d(m), d(upd), l_t)[0]
    err = (pred.double() - ref).abs()
    print(f"sharp attention window: max |d| {float(err.max()):.4f}  mean |d| {float(err.mean()):.5f}")
    # measured on an H100 80GB HBM3 (700 W): 0.096 / 0.0104, 3x the default-weights window (check_window, < 0.03),
    # while every operator of the window stays within half of its fp16 bound above
    assert float(err.max()) < 0.15 and float(err.mean()) < 0.015
