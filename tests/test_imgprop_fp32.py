"""GPU tests of the fp32 image propagation (pp_image_propagate_fp32, the node's fp16="disable"), -m gpu on an H100.

The propagation's decisions are discrete: the forward-backward validity test, the > 0.1 threshold of the warped mask and
the nearest-pixel pick.  The fp32 path keeps frames, masks and flows in fp32 and rounds the bilinear sums and the fb
test as torch does in fp32 on the CPU (where the reference's fixtures are made), so it takes the same decisions:

  one step, against torch fp32 on the CPU     zero mask mismatches, frames equal (copied pixels)
  golden fixture imgprop_frames / _masks      zero mask mismatches, frames within 1e-6 (fp16 path: < 1e-3 mismatches)
  chunked branch (T > subvideo_length)        the same bounds against the CPU oracle
  config[0] stage tensors                     updated-mask mismatches not above the fp16 path's in the same run
"""
import types

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def C():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from tests import gpu_checks
    return gpu_checks


def _step_ref(cur, mc, prop, mp, fp_, fc_, dtype):
    """One propagation step (model/propainter.py:186-196) by the CPU oracle in `dtype`."""
    from oracle import propainter_oracle as O
    cur, mc, prop, mp, fp_, fc_ = (t.to(dtype) for t in (cur, mc, prop, mp, fp_, fc_))
    valid = O.fb_consistency(fp_[None], fc_[None])
    warped = O.warp_by_flow(prop[None], fp_[None].permute(0, 2, 3, 1), "nearest")
    mv = O._bin(O.warp_by_flow(mp[None], fp_[None].permute(0, 2, 3, 1)))
    u = O._bin(mc[None] * valid * (1 - mv))
    return (u * warped + (1 - u) * cur[None])[0], O._bin(mc[None] * (1 - valid * (1 - mv)))[0, 0]


def _step_inputs(kind):
    from tests.golden import cases
    frames, m, (ff, fb) = cases.imgprop_case()
    cur, prop = frames[0, 1] * (1 - m[0, 1]), frames[0, 2] * (1 - m[0, 2])
    mc, mp = m[0, 1], m[0, 2]                                       # [1,H,W]
    fp_, fc_ = ff[0, 1], fb[0, 1]
    if kind == "border":
        # up to 24.5 px: samples land on and beyond the border; half-pixel flows put the nearest picks on rounding ties,
        # where the float32 and float64 oracles pick different pixels (frames differ by ~0.05)
        fp_ = torch.round(fp_ * 16) / 2
        fp_[1] = -fp_[1]
        fc_ = -fp_
    return cur, mc, prop, mp, fp_, fc_


@pytest.mark.parametrize("kind", ["fixture", "border"])
def test_fp32_imgprop_step_takes_the_reference_decisions(C, kind):
    cur, mc, prop, mp, fp_, fc_ = _step_inputs(kind)
    eng = C.bare_engine()
    pack = lambda f, k: torch.cat([f, k], 0).permute(1, 2, 0).contiguous().to(C.DEV)
    n2 = lambda f: f.permute(1, 2, 0).contiguous().to(C.DEV)
    out = eng.op_imgprop_step_f32(pack(cur, mc), pack(prop, mp), n2(fp_), n2(fc_)).cpu()
    out16 = eng.op_imgprop_step(pack(cur, mc).half(), pack(prop, mp).half(), n2(fp_).half(), n2(fc_).half()).float().cpu()
    f32, m32 = _step_ref(cur, mc, prop, mp, fp_, fc_, torch.float32)
    f64, m64 = _step_ref(cur, mc, prop, mp, fp_, fc_, torch.float64)
    mism = lambda o, m: int((o[..., 3] != m.float()).sum())
    print(kind, "mask mismatches vs fp32 oracle", mism(out, m32), "vs float64", mism(out, m64), "fp16 path vs fp32 oracle",
          mism(out16, m32), "fp32 oracle vs float64", int((m32.double() != m64).sum()))
    assert torch.isfinite(out).all()
    assert mism(out, m32) == 0
    assert torch.equal(out[..., :3].permute(2, 0, 1), f32)
    assert mism(out, m64) <= int((m32.double() != m64).sum())
    if kind == "border":
        assert float((m32 != mc[0]).float().sum()) > 0                  # the step did fill part of the hole
        assert float((f32.double() - f64).abs().max()) > 1e-3          # and hit ties that fp32 and float64 round apart


def test_fp32_image_propagation_matches_reference_fixture(C, golden):
    from tests.golden import cases
    frames, mk, (ff, fb) = cases.imgprop_case()
    eng = C.bare_engine()
    args = [t[0].to(C.DEV) for t in (frames, mk, ff, fb)]
    res = {}
    for fp32 in (True, False):
        uf, um = eng.image_propagate(*args, fp32=fp32)
        torch.cuda.synchronize()
        d = (uf.cpu() - torch.from_numpy(golden["imgprop_frames"])[0]).abs()
        res[fp32] = (float(d.max()), float((um.cpu() != torch.from_numpy(golden["imgprop_masks"])[0]).float().mean()))
    print("fp32 frame max |d|, mask mismatch", res[True], "fp16", res[False])
    assert res[True][1] == 0.0, res
    assert res[True][0] <= 1e-6, res
    assert res[False][1] < 1e-3, res


def test_fp32_image_propagation_is_deterministic_and_leaves_unmasked_clips_alone(C):
    from tests.golden import cases
    frames, mk, (ff, fb) = cases.imgprop_case()
    eng = C.bare_engine()
    fr, m, f, b = (t[0].to(C.DEV) for t in (frames, mk, ff, fb))
    a, b1 = eng.image_propagate(fr, m, f, b, fp32=True)
    c, d = eng.image_propagate(fr, m, f, b, fp32=True)
    assert torch.equal(a, c) and torch.equal(b1, d)
    uf, um = eng.image_propagate(fr, torch.zeros_like(m), f, b, fp32=True)
    assert torch.equal(uf, fr) and not um.any()


def test_fp32_chunked_image_propagation_matches_oracle(C):
    """T = 16 > subvideo_length = 4: the 10-frame halo branch of image_propagation, against the CPU oracle in fp32."""
    from comfyui_propainter_nodes_b200 import propainter_inference as PI
    from oracle import propainter_oracle as O
    from tests.golden import cases
    T, H, W = 16, 48, 64
    ff, fb = cases._flows(T - 1, H, W, 33, amp=2.0)
    frames, m = cases._clip(T, H, W, 34), cases._mask(T, H, W)
    cfg = PI.ProPainterConfig(3, 4, 4, 2, "disable", T, torch.device(C.DEV), (W, H))
    model = types.SimpleNamespace(engine=C.bare_engine())
    uf, um = PI.image_propagation(model, frames.to(C.DEV), m.to(C.DEV), (ff.to(C.DEV), fb.to(C.DEV)), cfg)
    torch.cuda.synchronize()
    rf, rm = O.image_propagation(frames, m, (ff, fb), cfg.subvideo_length)
    assert uf.dtype == torch.float32
    d, mm = float((uf.cpu() - rf).abs().max()), int((um.cpu() != rm).sum())
    print("chunked fp32 frame max |d|", d, "mask mismatches", mm)
    assert mm == 0 and d <= 1e-6


def test_config0_fp32_propagation_mask_mismatches_not_above_fp16(C, golden2):
    """BASELINE config[0] (16 frames, 320x176, fp16="disable"): the stage tensors process_inpainting hands to the
    generator, with the fp32 propagation it now runs, against the fp16 propagation on the same completed flows."""
    from comfyui_propainter_nodes_b200 import propainter_inference as PI
    from comfyui_propainter_nodes_b200.utils import image_utils as IU
    from tests.golden import cases
    m = C.full_models()
    c = cases.c1_case()
    kw = c["kwargs"]
    T, H, W = c["image"].shape[:3]
    icfg = IU.ImageConfig(kw["width"], kw["height"], kw["mask_dilates"], kw["flow_mask_dilates"], (W, H), T)
    ft, fm, md, _ = IU.prepare_frames_and_masks(IU.convert_image_to_frames(c["image"]), c["mask"], icfg, torch.device(C.DEV))
    cfg = PI.ProPainterConfig(kw["ref_stride"], kw["neighbor_length"], kw["subvideo_length"], kw["raft_iter"], kw["fp16"],
                              T, torch.device(C.DEV), icfg.process_size)
    assert not cfg.use_half
    uf32, um32, pf = PI.process_inpainting(m, ft, fm, md, cfg)
    uf16, um16 = m.inpaint_model.engine.image_propagate(ft[0], md[0], pf[0][0], pf[1][0], fp32=False)
    torch.cuda.synchronize()
    ref = golden2["c1_updated_masks_u8"]
    mis32 = float((C._img_u8(um32) != ref).mean())
    mis16 = float((C._img_u8(um16[None]) != ref).mean())
    print("config[0] updated-mask mismatch fp32", mis32, "fp16", mis16)
    assert mis32 <= mis16, (mis32, mis16)
    assert torch.isfinite(uf32).all()
