"""GPU tests of the flat-layer GEMM kernel (conv_gemm.cu) against torch fp32 on the fp16-rounded operands.

The cases are launches of at least one wave of 128 x 256 (or, for Cout <= 128, 256 x 128) tiles, so they reach the
GEMM kernel rather than the halo kernel that takes smaller flat launches: M and N tails, a ragged last K chunk, both
tile shapes with a residual, and M < 128 (which keeps the implicit-GEMM kernel).  The bound is the one of the other
conv cases (tests/test_gpu_parity.py)."""
import pytest
import torch

from comfyui_propainter_nodes_b200 import engine as E

pytestmark = pytest.mark.gpu

GEMM_CASES = {
    # name: (N, H, W, Cin_ref, Cout, kh, kw, stride, pad, dil, groups, replicate, act, slope, residual, cin_pad_to)
    # M tail (20000 = 156 x 128 + 32), N tail (1960 = 7 x 256 + 168), GELU + residual
    "gemm_m_tail_1960_gelu_res": (1, 1, 20000, 512, 1960, 1, 1, 1, 0, 1, 1, 0, E.ACT_GELU, 0.0, True, None),
    # N tail of a 3-tile layer (576 = 2 x 256 + 64), images x rows x columns flattened
    "gemm_n576_relu": (6, 50, 100, 256, 576, 1, 1, 1, 0, 1, 1, 0, E.ACT_RELU, 0.0, False, None),
    # 256 x 128 tiles: Cout 126 in one 128-column tile, M tail (40000 = 156 x 256 + 64)
    "gemm_n126_mb2": (1, 1, 40000, 256, 126, 1, 1, 1, 0, 1, 1, 0, E.ACT_RELU, 0.0, False, None),
    # ragged last K chunk: 324 input channels in a 328-channel tensor, 6 chunks (328 of 384)
    "gemm_ragged_k_324": (1, 1, 20000, 324, 256, 1, 1, 1, 0, 1, 1, 0, E.ACT_RELU, 0.0, False, 328),
    # 256 x 128 tiles with a residual and K = 1152 (the flow-propagation DCN shape)
    "gemm_k1152_mb2_res": (1, 1, 34000, 1152, 128, 1, 1, 1, 0, 1, 1, 0, E.ACT_LRELU, 0.1, True, None),
    # M < 128: not a GEMM-kernel launch, still a flat layer
    "gemm_m_lt_128": (1, 1, 100, 512, 256, 1, 1, 1, 0, 1, 1, 0, E.ACT_NONE, 0.0, False, None),
}


@pytest.fixture(scope="module")
def C():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from tests import gpu_checks
    return gpu_checks


@pytest.mark.parametrize("name", list(GEMM_CASES))
def test_gemm_conv_matches_torch_fp32(C, monkeypatch, name):
    monkeypatch.setitem(C.CONV_CASES, name, GEMM_CASES[name])
    s = C.check_conv(name)
    assert not s["nan"] and s["rel"] < 2e-3, s


@pytest.mark.parametrize("name,kind", [("gemm_n576_relu", "gemm"), ("gemm_m_lt_128", "igemm")])
def test_flat_layer_profile_label(C, monkeypatch, name, kind):
    """The profile names the kernel a flat layer ran on: conv:gemm: for launches of at least one wave of tiles."""
    monkeypatch.setitem(C.CONV_CASES, name, GEMM_CASES[name])
    eng = C.bare_engine()
    eng.profile_enable(True)
    try:
        C.check_conv(name)
        prof = eng.profile_dump()
    finally:
        eng.profile_enable(False)
    assert f"conv:{kind}:t.{name}" in prof, sorted(prof)
