"""GPU tests of the fp32 RAFT path (pp_raft_bidir_fp32, the node's fp16="disable"), -m gpu on an H100.

The reference always runs RAFT in fp32.  With fp32 activations and 3xTF32 GEMMs the engine's remaining error against
it comes from the accumulation order, so the bounds here are far below those of the fp16 path
(tests/test_gpu_parity_r2.py), on the same round-2 fixtures:

  un-damped 20-iteration case   mean |d| < 1 x raft20_undamped_sens at every stored iteration (fp16 path: 10 x)
  damped case, iteration 20     max and mean |d| at least 10 x below the fp16 path's in the same run
  config[0] through the node    RAFT flow max |d| < 0.01 px, mean < 1e-3 px (fp16 path: 0.1 / 0.01)
  pair batches                  bit-identical whatever the workspace forces the batch size to be
"""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def C():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from tests import gpu_checks
    return gpu_checks


def _raft20(C, golden2):
    from comfyui_propainter_nodes_b200 import engine as E
    from comfyui_propainter_nodes_b200 import weights as Wt
    from tests.golden import cases
    fr = cases.raft20_case()[0].to(C.DEV)
    out = {}
    for tag, gain in cases.RAFT20_GAINS.items():
        eng = E.Engine(C.DEV, workspace_gb=6.0).load_weights(Wt.synthetic_raft_state_dict(flow_head_gain=gain),
                                                           Wt.synthetic_rfc_state_dict(), Wt.synthetic_generator_state_dict())
        for it in cases.RAFT20_ITERS:
            ref = torch.from_numpy(golden2[f"raft20_{tag}_it{it}_s4"])
            for fp32 in (True, False):
                ff, _ = eng.raft_bidir(fr, it, fp32=fp32)
                torch.cuda.synchronize()
                out[(tag, it, fp32)] = C.stats(ff[:, :, ::4, ::4], ref)
        eng.close()
    return out


@pytest.fixture(scope="module")
def raft20(C, golden2):
    return _raft20(C, golden2)


def test_fp32_raft_20_iterations_undamped_within_fp32_yardstick(raft20, golden2):
    from tests.golden import cases
    sens = golden2["raft20_undamped_sens"]
    for i, it in enumerate(cases.RAFT20_ITERS):
        s = raft20[("undamped", it, True)]
        print("undamped it", it, "fp32", s["max_abs"], s["mean_abs"], "fp16", raft20[("undamped", it, False)]["mean_abs"],
              "sens", float(sens[i, 0]))
        assert not s["nan"]
        assert s["mean_abs"] < 1.0 * float(sens[i, 0]), (it, s, sens[i])


def test_fp32_raft_20_iterations_damped_10x_below_fp16(raft20):
    s32, s16 = raft20[("damped", 20, True)], raft20[("damped", 20, False)]
    print("damped it20 fp32", s32["max_abs"], s32["mean_abs"], "fp16", s16["max_abs"], s16["mean_abs"])
    assert s32["max_abs"] * 10 <= s16["max_abs"] and s32["mean_abs"] * 10 <= s16["mean_abs"], (s32, s16)


def test_config1_inpaint_node_fp32_raft_matches_reference(C, golden2):
    s = C.check_c1_node(golden2)          # fp16="disable": compute_flow runs the fp32 path
    print("c1 raft flow", s["raft_flow"], "pred flow", s["pred_flow"], "psnr", s["psnr"], s.get("psnr_hole"))
    assert s["flow_masks_equal"] and s["masks_dilated_equal"], s
    assert s["raft_flow"]["max_abs"] < 0.01 and s["raft_flow"]["mean_abs"] < 1e-3, s
    assert s["pred_flow"]["max_abs"] < 0.1, s
    assert s["updated_masks_mismatch"] < 1e-3, s
    assert s["psnr"] > 45.0 and s.get("psnr_hole", 99.0) > 38.0 and s["frac_gt1"] < 2e-3, s


def test_fp32_raft_is_independent_of_pair_batching(C):
    """8 frames at 320x176: 14 pair slots fit one batch in 4 GB, 0.3 GB splits them into two (10 + 4, one batch across
    both directions); the flows must be bit-identical, and so must a repeated run."""
    from comfyui_propainter_nodes_b200 import engine as E
    from comfyui_propainter_nodes_b200 import weights as Wt
    from comfyui_propainter_nodes_b200.synthetic import synthetic_clip
    sd = Wt.synthetic_raft_state_dict()
    fr = (synthetic_clip(8, 176, 320, 5).permute(0, 3, 1, 2) * 2 - 1).contiguous().to(C.DEV)
    res = {}
    for tag, gb in (("big", 4.0), ("small", 0.3)):
        eng = E.Engine(C.DEV, workspace_gb=gb)
        eng.load_weights(sd, Wt.synthetic_rfc_state_dict(), Wt.synthetic_generator_state_dict())
        a = eng.raft_bidir(fr, 3, fp32=True)
        b = eng.raft_bidir(fr, 3, fp32=True)
        torch.cuda.synchronize()
        res[tag] = (a, b, eng.workspace_peak)
        eng.close()
    (fb_, bb_, peak_big), (fs_, bs_, peak_small) = res["big"], res["small"]
    print("workspace peak big", peak_big, "small", peak_small)
    assert peak_small < peak_big, (peak_small, peak_big)      # the small arena really ran smaller pair batches
    for x, y in ((fb_, bb_), (fs_, bs_), (fb_, fs_)):
        assert torch.equal(x[0], y[0]) and torch.equal(x[1], y[1])
    assert float(fb_[0].abs().mean()) > 0.0
