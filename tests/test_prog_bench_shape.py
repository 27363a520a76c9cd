"""GPU test (-m gpu, H100): flow completion at the benchmark's size (80 frames, 640x360, both directions batched) gives
bit-identical completed flows as multi-layer programs (PP_PROG=1, one launch per propagation step) and as one launch per
layer (PP_PROG=0).

The tile plans of the program layers depend on the pixel count of a step; at this size the 432-channel offset head runs
as two 224-column N tiles, a plan the small cases of the other GPU tests never reach.  Changing the N or M tiling keeps
the order in which each output's K terms are summed, so the two variants must agree bit for bit."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


def _inputs(T, H, W, dev):
    # the inputs of tools/rfc_bench.py
    from comfyui_propainter_nodes_b200.synthetic import synthetic_mask
    g = torch.Generator().manual_seed(0)
    ff = (torch.randn(T - 1, 2, H // 8, W // 8, generator=g) * 2).to(dev)
    ff = torch.nn.functional.interpolate(ff, size=(H, W), mode="bilinear") + 1.5
    masks = synthetic_mask(T, H, W)[:, None].contiguous().to(dev)
    return ff, -ff, masks


def test_flow_completion_program_equals_per_layer_at_bench_size():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from comfyui_propainter_nodes_b200 import weights as Wt
    from comfyui_propainter_nodes_b200.engine import Engine
    dev = torch.device("cuda:0")
    eng = Engine(dev, workspace_gb=24.0).load_weights(Wt.synthetic_raft_state_dict(), Wt.synthetic_rfc_state_dict(),
                                                      Wt.synthetic_generator_state_dict())
    ff, fb, masks = _inputs(80, 360, 640, dev)
    outs = {}
    keep = os.environ.get("PP_PROG")
    try:
        for prog in ("1", "0"):
            os.environ["PP_PROG"] = prog
            of, ob = eng.flow_complete(ff, fb, masks)
            torch.cuda.synchronize()
            outs[prog] = (of.clone(), ob.clone())
    finally:
        if keep is None:
            os.environ.pop("PP_PROG", None)
        else:
            os.environ["PP_PROG"] = keep
    del eng
    torch.cuda.empty_cache()
    for a, b in zip(outs["1"], outs["0"]):
        assert torch.isfinite(a).all()
        assert int((a != b).sum()) == 0
