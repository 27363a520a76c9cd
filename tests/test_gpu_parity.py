"""GPU parity tests (run on an H100: python -m pytest tests -m gpu).

CUDA path (through the C ABI) vs. the golden outputs of the REAL reference / the CPU oracle on identical
seeded inputs.  Tolerances: the engine stores activations in fp16 and accumulates in fp32, the oracle and the
golden fixtures are fp32 end to end, so the stated bounds are the fp16 tolerance of this port:

  flows (RAFT, 4 GRU iterations)    max |d| < 0.05 px, mean < 0.01 px
  completed flows                   max |d| < 0.02 px
  image propagation                 < 0.1 % of pixels differ (nearest-neighbour ties), masks identical
  generator window (tanh output)    max |d| < 0.03
  end-to-end uint8 frames           PSNR > 45 dB vs the reference's frames, <= 0.1 % of values off by more than 1
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def C():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from tests import gpu_checks
    return gpu_checks


@pytest.mark.parametrize("name", ["linear_512_1536", "conv3x3_128_128_lrelu_res", "conv7x7_s2_3_64", "conv3x3_dil3",
                                  "conv5x5_s2_replicate", "grouped_g4", "cout2", "cout126", "cout432", "cin261",
                                  "conv7x7_s3_40_512", "conv1x5", "conv5x1_tanh", "k2304", "halo_mt2_64_64",
                                  "halo_odd_size", "halo_mt2_256_192", "halo_5x5_dil2", "halo_flat_328_256",
                                  "halo_flat_ragged_rows"])
def test_tcgen05_conv_matches_torch_fp32(C, name):
    s = C.check_conv(name)
    assert not s["nan"] and s["rel"] < 2e-3, s


def test_corr_lookup_matches_oracle(C):
    s = C.check_corr_lookup()
    assert s["max_abs"] < 5e-3 and s["pad_zero"] == 0.0, s


def test_image_propagation_step_matches_oracle(C):
    s = C.check_imgprop_step()
    assert s["frame_mismatch_frac"] < 1e-3 and s["mask_mismatch_frac"] < 1e-3, s


def test_window_attention_matches_oracle(C):
    for k, s in C.check_attention().items():
        assert not s["nan"] and s["rel"] < 3e-3, (k, s)


def test_raft_matches_reference(C, golden):
    for k, s in C.check_raft(golden).items():
        assert not s["nan"] and s["max_abs"] < 0.05 and s["mean_abs"] < 0.01, (k, s)


def test_flow_completion_matches_reference(C, golden):
    for k, s in C.check_rfc(golden).items():
        assert not s["nan"] and s["max_abs"] < 0.02, (k, s)


def test_image_propagation_matches_reference(C, golden):
    s = C.check_imgprop(golden)
    assert s["frame_mismatch_frac"] < 1e-3 and s["mask_mismatch_frac"] < 1e-3, s


def test_generator_window_matches_reference(C, golden):
    s = C.check_window(golden)
    assert not s["nan"] and s["max_abs"] < 0.03, s


def test_end_to_end_matches_reference(C, golden):
    s = C.check_e2e(golden)
    assert s["psnr"] > 45.0 and s["psnr_hole"] > 40.0 and s["frac_gt1"] < 1e-3, s
    assert s["flow"]["max_abs"] < 0.05, s


# ---- full-size (640x360) properties that do not need the oracle -----------------------------------------

def _full(C, T=4, H=360, W=640):
    from comfyui_propainter_nodes_b200.synthetic import synthetic_clip, synthetic_mask
    m = C.full_models()
    img = synthetic_clip(T, H, W, 99)
    frames = (img.permute(0, 3, 1, 2) * 2 - 1).contiguous().to(C.DEV)
    masks = synthetic_mask(T, H, W)[:, None].contiguous().to(C.DEV)
    return m, img, frames, masks


def test_fullsize_flow_completion_keeps_known_flow(C):
    """combine_flow: outside the mask the completed flow IS the input flow (bit exact)."""
    m, img, frames, masks = _full(C)
    eng = m.raft_model.engine
    ff, fb = eng.raft_bidir(frames, 2)
    of, ob = eng.flow_complete(ff, fb, masks)
    keep = (masks[:-1] == 0).expand_as(ff)
    assert torch.equal(of[keep], ff[keep])
    keep_b = (masks[1:] == 0).expand_as(fb)
    assert torch.equal(ob[keep_b], fb[keep_b])
    assert torch.isfinite(of).all() and torch.isfinite(ob).all()
    # determinism: same inputs -> bit-identical outputs (RAFT included: instance-norm statistics use no float atomics)
    of2, _ = eng.flow_complete(ff, fb, masks)
    assert torch.equal(of, of2)
    ff2, fb2 = eng.raft_bidir(frames, 2)
    assert torch.equal(ff, ff2) and torch.equal(fb, fb2)
    # and independent of how the pairs are batched (a shard of the pairs gives the same flows)
    ff3, fb3 = eng.raft_bidir(frames[1:3], 2)
    assert torch.equal(ff3[0], ff[1]) and torch.equal(fb3[0], fb[1])


def test_fullsize_image_propagation_identities(C):
    m, img, frames, masks = _full(C)
    eng = m.inpaint_model.engine
    T, _, H, W = frames.shape
    zero = torch.zeros(T - 1, 2, H, W, device=C.DEV)
    # no hole: nothing to propagate, frames unchanged (up to the fp16 store) and masks stay empty
    uf, um = eng.image_propagate(frames, torch.zeros_like(masks), zero, zero)
    assert float((uf - frames).abs().max()) == 0.0 and float(um.abs().max()) == 0.0
    # zero flow and a static hole: nothing valid can be pulled in, the hole stays masked and known pixels stay
    uf, um = eng.image_propagate(frames, masks, zero, zero)
    assert torch.equal(um, masks)
    known = (masks == 0).expand_as(frames)
    assert torch.equal(uf[known], frames[known])


def test_fullsize_composite_keeps_known_pixels(C):
    """Outside the dilated mask the composited uint8 frame is the original frame, bit exact."""
    from comfyui_propainter_nodes_b200 import propainter_inference as PI
    from comfyui_propainter_nodes_b200.utils import image_utils as IU
    m, img, _, _ = _full(C, T=6)
    T, H, W = 6, 360, 640
    from comfyui_propainter_nodes_b200.synthetic import synthetic_mask
    icfg = IU.ImageConfig(W, H, 5, 8, (W, H), T)
    ft, fm, md, orig = IU.prepare_frames_and_masks(IU.convert_image_to_frames(img), synthetic_mask(T, H, W), icfg,
                                                   torch.device(C.DEV))
    cfg = PI.ProPainterConfig(3, 4, 80, 3, "enable", T, torch.device(C.DEV), icfg.process_size)
    uf, um, flows = PI.process_inpainting(m, ft, fm, md, cfg)
    comp = np.stack(PI.feature_propagation(m.inpaint_model, uf, um, md, flows, orig, cfg))
    o = np.stack(orig)
    keep = md[0, :, 0].cpu().numpy() == 0
    assert (comp[keep] == o[keep]).all()
    assert (comp[~keep] != o[~keep]).any()
    # window sharding (multi-GPU path): every window computed separately gives the same frames
    sched = PI.window_schedule(cfg)
    orig_t = torch.from_numpy(o)
    parts = [PI.feature_propagation_device(m.inpaint_model, uf, um, md, flows, orig_t, cfg, windows=[i])
             for i in range(len(sched))]
    full = PI.feature_propagation_device(m.inpaint_model, uf, um, md, flows, orig_t, cfg)
    assert torch.equal(full.cpu(), torch.from_numpy(comp))
    # frames covered by exactly one window must agree bit for bit with the full run
    cover = np.zeros(T, dtype=int)
    for nb, _ in sched:
        for i in nb:
            cover[i] += 1
    for wi, (nb, _) in enumerate(sched):
        for i in nb:
            if cover[i] == 1:
                assert torch.equal(parts[wi][i], full[i])


def test_device_preprocessing_is_bit_exact(C):
    """pp_preprocess == the host path (uint8 truncation, scipy cross dilation x N) on the same inputs."""
    from comfyui_propainter_nodes_b200.utils import image_utils as IU
    from comfyui_propainter_nodes_b200.synthetic import synthetic_clip
    T, H, W = 5, 72, 104
    img = synthetic_clip(T, H, W, 3)
    g = torch.Generator().manual_seed(1)
    mask = (torch.rand(T, H, W, generator=g) > 0.995).float() * torch.rand(T, H, W, generator=g)
    mask[:, 10:20, 30:50] = 0.7
    mask[:, 0:3, 0:3] = 1.0              # touches the border
    eng = C.full_models().raft_model.engine
    for fd, mdil, msk in ((8, 5, mask), (0, 3, mask), (4, 0, mask[:1])):
        cfg = IU.ImageConfig(W, H, mdil, fd, (W, H), T)
        ft, fm, md, orig = IU.prepare_frames_and_masks(IU.convert_image_to_frames(img), msk.clone(), cfg, torch.device("cpu"))
        ft2, fm2, md2, orig2 = eng.preprocess(img, msk, fd, mdil)
        assert torch.equal(ft2.cpu(), ft) and torch.equal(fm2.cpu(), fm) and torch.equal(md2.cpu(), md)
        assert np.array_equal(orig2.cpu().numpy(), np.stack(orig))
    u8 = torch.randint(0, 256, (2, 8, 8, 3), dtype=torch.uint8)
    assert torch.equal(eng.postprocess(u8.to(C.DEV)).cpu(), u8.float() / 255.0)
