"""CPU tests of the generator's operator tests (tests/test_gen_ops.py): the new C-ABI entry points exist, the float64
attention reference is the reference's SparseWindowAttention, and every operator bound rejects the defect it is there
to catch while it accepts an emulation of the kernel's own arithmetic."""
import math
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from comfyui_propainter_nodes_b200 import engine as E
from comfyui_propainter_nodes_b200 import weights as Wt
from oracle import propainter_oracle as O
from tests import test_gen_ops as GEN

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ("pp_op_layernorm", "pp_op_pool_tokens", "pp_op_window_flags", "pp_op_fold", "pp_op_featprop_cond",
               "pp_op_dcn_sample", "pp_op_downsample4", "pp_op_upsample2x", "pp_op_attention")


def test_generator_operator_entry_points_are_declared_and_exported():
    import ctypes
    hdr = open(os.path.join(ROOT, "include", "propainter_b200.h")).read()
    lib = ctypes.CDLL(E.LIB_PATH)
    for name in NEW_SYMBOLS:
        decl = re.search(r"PP_API int " + name + r"\(([^;]*)\);", hdr)
        assert decl, name
        assert len(decl.group(1).split(",")) == len(E._SIGNATURES[name][1]), name
        assert name in E.exported_symbols()
        getattr(lib, name)
    # one attention entry point, taking one t per sliding window
    assert len(re.findall(r"PP_API int pp_op_attention", hdr)) == 1
    assert re.search(r"const int\* win_t,\s*int n_windows", hdr)


# ---- layernorm: the one-pass variance --------------------------------------------------------------------------------
def _ln_emulate(x16, gamma, beta, two_pass):
    """layernorm512's arithmetic in numpy float32: lane l sums channels 16l..16l+15 in pairs, xor-butterfly over the 32
    lanes; variance E[x^2] - mean^2 (one pass) or the mean of (x - mean)^2 (two pass)"""
    x = x16.numpy().astype(np.float32)
    R = x.shape[0]
    v = x.reshape(R, 32, 16)
    f32 = np.float32

    def butterfly(s):
        for o in (16, 8, 4, 2, 1):
            s = (s + s[:, np.arange(32) ^ o]).astype(f32)
        return s[:, :1]
    s = np.zeros((R, 32), f32)
    q = np.zeros((R, 32), f32)
    for i in range(8):
        a, c = v[:, :, 2 * i], v[:, :, 2 * i + 1]
        s = (s + (a + c)).astype(f32)
        q = (q + (a * a + c * c)).astype(f32)
    mean = (butterfly(s) * f32(1 / 512)).astype(f32)
    if two_pass:
        q = np.zeros((R, 32), f32)
        for i in range(8):
            a, c = (v[:, :, 2 * i] - mean).astype(f32), (v[:, :, 2 * i + 1] - mean).astype(f32)
            q = (q + (a * a + c * c)).astype(f32)
        var = (butterfly(q) * f32(1 / 512)).astype(f32)
    else:
        var = np.maximum((butterfly(q) * f32(1 / 512) - mean * mean).astype(f32), 0)
    rstd = (1 / np.sqrt(var + f32(1e-5))).astype(f32)
    g, b = gamma.numpy().astype(f32), beta.numpy().astype(f32)
    return torch.from_numpy((((x - mean) * rstd) * g + b).astype(f32).astype(np.float16))


def _ln_excess(ratio, two_pass):
    x, gamma, beta = GEN.layernorm_case(2, 8, 12, ratio, seed=ratio)
    ref = GEN.layernorm_reference(x, gamma, beta)
    return GEN.excess(_ln_emulate(x, gamma, beta, two_pass), ref, GEN.fp16_bound(ref))


@pytest.mark.parametrize("ratio", [0, 3, 30, 100])
def test_layernorm_bound_accepts_the_two_pass_variance(ratio):
    assert _ln_excess(ratio, two_pass=True) <= 1.0


def test_layernorm_bound_rejects_the_one_pass_variance():
    assert _ln_excess(3, two_pass=False) <= 1.0          # harmless at small mean / std
    assert _ln_excess(100, two_pass=False) > 4.0


# ---- fold -----------------------------------------------------------------------------------------------------------
def _fold_case(C, H, W, t=2):
    gh, gw = (H - 1) // 3 + 1, (W - 1) // 3 + 1
    g = torch.Generator().manual_seed(C + H + W)
    return torch.randn(t * gh * gw, 49 * C, generator=g).half()


@pytest.mark.parametrize("H,W", [(8, 13), (10, 14), (12, 9)])
def test_fold_bound_accepts_fp32_and_rejects_a_wrong_border_count(H, W):
    x, t, C = _fold_case(40, H, W), 2, 40
    ref = GEN.fold_reference(x, t, H, W, C, True, True)
    bnd = GEN.fp16_bound(ref)
    # fp32 overlap-add, count, erf-GELU, one rounding to fp16
    L = x.shape[0] // t
    y = F.fold(x.float().view(t, L, 49, C).permute(0, 3, 2, 1).reshape(t, C * 49, L), (H, W), **O.T2T)
    cnt = F.fold(torch.ones(1, 49, L), (H, W), **O.T2T)
    emu = F.gelu(y / cnt).half().permute(0, 2, 3, 1)
    assert GEN.excess(emu, ref, bnd) <= 1.0
    wrong = GEN.fold_reference(x, t, H, W, C, True, True, count_size=(H + 3, W + 3)).half()
    assert GEN.excess(wrong, ref, bnd) > 10.0


# ---- fp16 deformable sampler ----------------------------------------------------------------------------------------
def _dcn(**mutation):
    x, o, flow = GEN.dcn_case(159, 128, N=1, flow_px=4.0)
    ref, bnd = GEN.dcn_reference(x, o, 3.0, flow=flow)
    flow_used = mutation.pop("flow", flow)
    got = GEN.RFC.im2col_reference(x.float(), o.float(), torch.float32, max_mag=3.0, flow=flow_used.float(),
                                   **mutation).half()
    return GEN.excess(got, ref, bnd)


def test_dcn_bound_accepts_fp32_sampling_with_an_approximate_tanh():
    assert _dcn() <= 1.0
    for sign in (1, -1):
        assert _dcn(tanh=lambda v: torch.tanh(v) * (1 + sign * 2.0 ** -11)) <= 1.0


def test_dcn_bound_rejects_swapped_flow_components():
    x, o, flow = GEN.dcn_case(159, 128, N=1, flow_px=4.0)
    assert _dcn(flow=flow.flip(-1)) > 10.0


def test_dcn_bound_rejects_a_missing_modulation():
    assert _dcn(sigmoid=torch.ones_like) > 10.0


# ---- window attention -----------------------------------------------------------------------------------------------
def tiled_attend(rescale=True):
    """window_attention_tc's softmax: key tiles of 64, a reference max kept in fp16 and raised only when the running max
    grew by more than 8 (log2 units) -- then the row is rescaled (rescale=False drops that) -- and P rounded to fp16
    for P.V; the row sum adds the unrounded P"""
    def attend(s, v):
        o = torch.zeros(*s.shape[:2], v.shape[-1], dtype=torch.float64)
        row_sum = torch.zeros(*s.shape[:2], 1, dtype=torch.float64)
        m_used = m_run = None
        for j0 in range(0, s.shape[-1], 64):
            st = s[..., j0:j0 + 64]
            m_tile = st.amax(-1, keepdim=True).half().double()
            m_new = m_tile if m_run is None else torch.maximum(m_run, m_tile)
            if m_used is None:
                m_used = m_new
            else:
                up = m_new > m_used + 8
                f = torch.where(up, torch.exp2(m_used - m_new), torch.ones_like(m_new))
                if rescale:
                    o, row_sum = o * f, row_sum * f
                m_used = torch.where(up, m_new, m_used)
            m_run = m_new
            p = torch.exp2(st - m_used)
            row_sum = row_sum + p.sum(-1, keepdim=True)
            o = o + p.half().double() @ v[:, j0:j0 + 64]
        return o / row_sum
    return attend


@pytest.fixture(scope="module")
def att():
    c = GEN.attention_case(3)
    return c, {p: GEN.attention_reference(c, p) for p in (0, 1)}


@pytest.mark.parametrize("parity", [0, 1])
def test_attention_case_is_sharp_in_both_tile_positions(att, parity):
    _, refs = att
    _, _, spread, first = refs[parity]
    assert float(spread.min()) >= 30.0
    assert bool(first.any()) and bool((~first).any())


@pytest.mark.parametrize("parity", [0, 1])
def test_attention_bound_accepts_the_tiled_fp16_softmax(att, parity):
    c, refs = att
    ref, bnd = refs[parity][:2]
    emu = GEN.attention_reference(c, parity, attend=tiled_attend())[0].half()
    assert GEN.excess(emu, ref, bnd) <= 1.0


@pytest.mark.parametrize("parity", [0, 1])
def test_attention_bound_rejects_a_missing_rescale(att, parity):
    c, refs = att
    ref, bnd = refs[parity][:2]
    emu = GEN.attention_reference(c, parity, attend=tiled_attend(rescale=False))[0].half()
    assert GEN.excess(emu, ref, bnd) > 10.0


@pytest.mark.parametrize("parity", [0, 1])
def test_attention_bound_rejects_a_ring_index_off_by_one(att, parity):
    c, refs = att
    ref, bnd = refs[parity][:2]
    ring = c["ring"].clone()
    ring[:, 45:] = (ring[:, 45:] + 1) % (c["nh"] * c["nw"])
    assert GEN.excess(GEN.attention_reference(c, parity, ring=ring)[0], ref, bnd) > 10.0


@pytest.mark.parametrize("parity", [0, 1])
def test_attention_bound_rejects_pooled_tokens_of_the_wrong_parity(att, parity):
    c, refs = att
    ref, bnd = refs[parity][:2]
    wrong = GEN.attention_reference(c, parity, pooled_frame=lambda f: f - 1 if f % 2 else f + 1)[0]
    assert GEN.excess(wrong, ref, bnd) > 10.0


@pytest.mark.parametrize("parity", [0, 1])
def test_attention_reference_is_the_sparse_window_attention(parity):
    """with identity query / proj projections, random key / value projections and zero biases, the kernel-operand
    reference equals O.sparse_window_attention (the reference's module restated) on the same tokens"""
    g = torch.Generator().manual_seed(7)
    t, (gh, gw), C = 5, GEN.ATT_GRID, 512
    nh, nw = 10, 18
    x = torch.randn(1, t, gh, gw, C, generator=g, dtype=torch.float64)
    p = "a."
    sd = {p + n + ".bias": torch.zeros(C, dtype=torch.float64) for n in ("query", "key", "value", "proj")}
    sd[p + "query.weight"] = sd[p + "proj.weight"] = torch.eye(C, dtype=torch.float64)
    sd[p + "key.weight"] = torch.randn(C, C, generator=g, dtype=torch.float64) / math.sqrt(C)
    sd[p + "value.weight"] = torch.randn(C, C, generator=g, dtype=torch.float64) / math.sqrt(C)
    sd[p + "pool_layer.weight"] = 1 / 16.0 + 0.02 * torch.randn(C, 1, 4, 4, generator=g, dtype=torch.float64)
    sd[p + "pool_layer.bias"] = torch.zeros(C, dtype=torch.float64)
    sd[p + "valid_ind_rolled"] = torch.from_numpy(Wt.rolled_valid_indices())
    mask = torch.zeros(1, 3, gh, gw, 1, dtype=torch.float64)
    mask[0, 1, 1:3, 2:5] = 1                  # window (0, 0)
    mask[0, 2, 7, 11] = 1                     # window (1, 1)
    ref = O.sparse_window_attention(sd, p, x, mask, torch.arange(parity, t, 2))[0]

    xp = F.pad(x[0], (0, 0, 0, nw - gw, 0, nh - gh))                       # [t, nh, nw, C]
    pooled = F.conv2d(xp.permute(0, 3, 1, 2), sd[p + "pool_layer.weight"], stride=4, groups=C)
    pooled = pooled.permute(0, 2, 3, 1).reshape(t, -1, C)
    heads = lambda a: a.reshape(t, -1, 4, 128)
    wm = F.max_pool2d(F.pad(mask[0, ..., 0], (0, nw - gw, 0, nh - gh)), (5, 9), (5, 9)).sum(0).flatten()
    c = dict(q=heads(xp), k=heads(xp @ sd[p + "key.weight"].T), v=heads(xp @ sd[p + "value.weight"].T),
             pk=heads(pooled @ sd[p + "key.weight"].T), pv=heads(pooled @ sd[p + "value.weight"].T), nh=nh, nw=nw,
             gh=gh, gw=gw, n_pool=pooled.shape[1], flags=(wm > 0).int()[None], ring=GEN.ring_tokens(nh, nw),
             win_t=(t,))
    assert c["flags"].tolist() == [[1, 0, 0, 1]]
    out = GEN.attention_reference(c, parity)[0]
    assert float((out - ref).abs().max()) < 1e-12
