"""GPU tests of the fp32 flow completion (pp_flow_complete_fp32, the node's fp16="disable"), -m gpu on an H100.

The float64 truth is the oracle (oracle/propainter_oracle.py, pinned to the reference by tests/test_oracle_golden.py)
run on a float64 copy of the weights and inputs.  Required:

  golden rfc_f / rfc_b (the reference in fp32)   max |d| < 2e-3 px (fp16 path: 2e-2)
  three cases against float64                    max |d| at least 10x and mean |d| at least 5x below the fp16 path's
                                                 in the same run, mean |d| <= 250 x the CPU fp32 oracle's own mean |d|
  outside the mask                               the input flow, bit for bit
  repeated run / small arena                     bit-identical (the small arena runs the decoder in frame batches)

Measured on an H100 80GB HBM3 (700 W), both directions: fp32 max |d| is 15.8-22.1 x below the fp16 path's, mean |d|
6.2-36 x below it and 149-202 x the CPU fp32 oracle's.  The mean criteria are looser than a single operator's: on this
data one 3xTF32 convolution is only ~2^-17 relative (tests/test_rfc_fp32_ops.py), 1/30 of a layer with tf32 inputs, and
~40 such layers leave a floor of the order of one tf32 layer.  What the criteria must catch, and do
(test_stage_criteria_reject_one_layer_without_its_lo_term): one decoder layer with tf32 inputs (max |d| 4.3-4.8 x below
fp16, mean 270-298 x CPU) or tf32 weights (3.8-3.9 x, 433-504 x).  A tf32 offset head is not visible at this level
(its error moves the output by 0.1 %); the operator tests cover those layers.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
MAX_FP16_FACTOR = 10.0      # fp32 max |d| at least this far below the fp16 path's
MEAN_FP16_FACTOR = 5.0      # fp32 mean |d| at least this far below the fp16 path's
MEAN_RATIO = 250.0          # fp32 mean |d| at most this multiple of the CPU fp32 oracle's
RATIOS = {}


@pytest.fixture(scope="module")
def eng():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from comfyui_propainter_nodes_b200 import engine as E
    from comfyui_propainter_nodes_b200 import weights as Wt
    e = E.Engine(DEV, workspace_gb=12.0).load_weights(Wt.synthetic_raft_state_dict(), Wt.synthetic_rfc_state_dict(),
                                                      Wt.synthetic_generator_state_dict())
    yield e
    e.close()
    print("fp32 mean |d| / CPU fp32 oracle mean |d|:", RATIOS)


def _d(a, b):
    d = (a.detach().double().cpu() - b.detach().double().cpu()).abs()
    return float(d.max()), float(d.mean())


def _run(eng, ff, fb, fm, fp32):
    of, ob = eng.flow_complete(ff.to(DEV), fb.to(DEV), fm.to(DEV), fp32=fp32)
    torch.cuda.synchronize()
    return of.cpu(), ob.cpu()


def test_fp32_flow_completion_matches_golden(eng, golden):
    from tests.golden import cases
    (ff, fb), masks = cases.rfc_case()
    of, ob = _run(eng, ff[0], fb[0], masks[0], True)
    for got, key in ((of, "rfc_f"), (ob, "rfc_b")):
        mx, mean = _d(got[None], torch.from_numpy(golden[key]))
        print(key, "fp32 max", mx, "mean", mean)
        assert mx < 2e-3, (key, mx, mean)


def _errors(name, eng, flows_bi, masks, complete, fp16=True):
    """-> per direction (fp32 max, fp32 mean, fp16 max, fp16 mean, CPU fp32 max, CPU fp32 mean) |d| against float64.
    complete(sd, flows_bi, masks, fp32 or None = the CPU oracle in the dtype of its inputs) -> (of, ob) [1,T-1,2,H,W]"""
    from comfyui_propainter_nodes_b200 import weights as Wt
    sd = Wt.synthetic_rfc_state_dict()
    with torch.no_grad():
        truth = complete({k: v.double() for k, v in sd.items()}, tuple(f.double() for f in flows_bi), masks.double(), None)
        cpu32 = complete({k: v.float() for k, v in sd.items()}, tuple(f.float() for f in flows_bi), masks.float(), None)
    e32 = complete(None, flows_bi, masks, True)
    e16 = complete(None, flows_bi, masks, False)
    out = []
    for k in range(2):
        assert torch.isfinite(e32[k]).all()
        (m32, a32), (m16, a16), (mc, ac) = _d(e32[k], truth[k]), _d(e16[k], truth[k]), _d(cpu32[k], truth[k])
        print(f"{name} dir {k}: fp32 {m32:.3e}/{a32:.3e}  fp16 {m16:.3e}/{a16:.3e}  cpu fp32 {mc:.3e}/{ac:.3e}  "
              f"fp16/fp32 {m16 / m32:.1f}/{a16 / a32:.1f}  fp32/cpu mean {a32 / ac:.0f}")
        out.append((m32, a32, m16, a16, mc, ac))
    return out


def _violations(errs):
    """the stage criteria a result breaks (empty: it passes)"""
    bad = []
    for k, (m32, a32, m16, a16, mc, ac) in enumerate(errs):
        if m32 * MAX_FP16_FACTOR > m16:
            bad.append(f"dir {k}: max |d| {m32:.3e} not {MAX_FP16_FACTOR}x below fp16's {m16:.3e}")
        if a32 * MEAN_FP16_FACTOR > a16:
            bad.append(f"dir {k}: mean |d| {a32:.3e} not {MEAN_FP16_FACTOR}x below fp16's {a16:.3e}")
        if a32 > MEAN_RATIO * ac:
            bad.append(f"dir {k}: mean |d| {a32:.3e} above {MEAN_RATIO} x CPU fp32's {ac:.3e}")
    return bad


def _against_float64(name, eng, flows_bi, masks, complete):
    errs = _errors(name, eng, flows_bi, masks, complete)
    for k, e in enumerate(errs):
        RATIOS[f"{name}[{k}]"] = round(e[1] / max(e[5], 1e-300), 1)
    bad = _violations(errs)
    assert not bad, (name, bad)


def _clip(T, H, W, seed):
    from comfyui_propainter_nodes_b200.synthetic import synthetic_mask
    from tests.golden import cases
    ff, fb = cases._flows(T - 1, H, W, seed)
    return (ff, fb), synthetic_mask(T, H, W)[None, :, None].contiguous()


def _bidir(eng):
    from oracle import propainter_oracle as O

    def complete(sd, flows_bi, masks, fp32):
        if fp32 is None:
            return O.rfc_bidirectional(sd, flows_bi, masks)
        of, ob = _run(eng, flows_bi[0][0].float(), flows_bi[1][0].float(), masks[0].float(), fp32)
        return of[None], ob[None]
    return complete


def test_fp32_flow_completion_fixture_against_float64(eng):
    from tests.golden import cases
    flows, masks = cases.rfc_case()
    _against_float64("fixture", eng, flows, masks, _bidir(eng))


def test_fp32_flow_completion_640x360_against_float64(eng):
    flows, masks = _clip(8, 360, 640, 41)
    _against_float64("640x360x8", eng, flows, masks, _bidir(eng))


def test_fp32_flow_completion_chunked_against_float64(eng):
    """T = 26 > subvideo_length 12: propainter_inference.complete_flow's chunks with the 5-flow halo"""
    from comfyui_propainter_nodes_b200 import propainter_inference as PI
    from comfyui_propainter_nodes_b200.utils.model_utils import StageHandle
    from oracle import propainter_oracle as O
    flows, masks = _clip(26, 64, 96, 43)

    def complete(sd, flows_bi, m, fp32):
        if fp32 is None:
            return O.complete_flow(sd, flows_bi, m, 12)
        dt = torch.float32 if fp32 else torch.float16
        of, ob = PI.complete_flow(StageHandle(eng, "flow"), tuple(f.to(DEV, dt) for f in flows_bi), m.to(DEV, dt), 12)
        torch.cuda.synchronize()
        return of.cpu(), ob.cpu()
    _against_float64("chunked", eng, flows, masks, complete)


def test_fp32_combine_keeps_the_input_flow_outside_the_mask(eng):
    flows, masks = _clip(6, 64, 96, 45)
    ff, fb = flows[0][0], flows[1][0]
    of, ob = _run(eng, ff, fb, masks[0], True)
    m = masks[0]
    for got, src, mk in ((of, ff, m[:-1]), (ob, fb, m[1:])):
        out = (mk == 0).expand_as(src)
        assert torch.equal(got[out], src[out])
        assert not torch.equal(got[~out], src[~out])          # inside the hole it is the network's prediction


def test_fp32_flow_completion_is_deterministic_and_independent_of_arena_size():
    """16 frames at 320x176: a 3 GB arena runs the decoder over all 15 frames at once, 1 GB forces frame batches;
    the completed flows must be bit-identical, and so must a repeated run."""
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from comfyui_propainter_nodes_b200 import engine as E
    from comfyui_propainter_nodes_b200 import weights as Wt
    flows, masks = _clip(16, 176, 320, 47)
    res = {}
    for tag, gb in (("big", 3.0), ("small", 1.0)):
        e = E.Engine(DEV, workspace_gb=gb).load_weights(Wt.synthetic_raft_state_dict(), Wt.synthetic_rfc_state_dict(),
                                                        Wt.synthetic_generator_state_dict())
        a = _run(e, flows[0][0], flows[1][0], masks[0], True)
        b = _run(e, flows[0][0], flows[1][0], masks[0], True)
        res[tag] = (a, b, e.workspace_peak)
        e.close()
    (ab, bb, peak_big), (as_, bs, peak_small) = res["big"], res["small"]
    print("workspace peak big", peak_big, "small", peak_small)
    assert peak_small < peak_big, (peak_small, peak_big)         # the small arena really ran smaller frame batches
    for x, y in ((ab, bb), (as_, bs), (ab, as_)):
        assert torch.equal(x[0], y[0]) and torch.equal(x[1], y[1])


# ---- the stage criteria reject a single layer that loses the split's precision -------------------------------------
def _image_without(w, term):
    """pack_conv_weight_tf32's image with one of the three products of its split GEMM removed: "lo_hi" reads the layer's
    inputs without their lo parts (tf32 inputs), "hi_lo" uses only the hi part of the weights."""
    from comfyui_propainter_nodes_b200 import engine as E
    packed, meta = E.pack_conv_weight_tf32(w)
    cout, cin, kh, kw = w.shape
    hi, lo = E.split_tf32(w)
    parts = dict(hi_hi=hi, lo_hi=hi, hi_lo=lo)
    parts[term] = torch.zeros_like(hi)
    wk = torch.cat([parts["hi_hi"], parts["lo_hi"], parts["hi_lo"]], 1).permute(0, 2, 3, 1).reshape(cout, -1)
    rows, num_kc = meta["cout_g_pad"], packed.shape[0]
    buf = torch.zeros(rows, num_kc * 32)
    buf[:cout, :wk.shape[1]] = wk
    buf = buf.view(rows, num_kc, 8, 4).permute(1, 0, 2, 3).contiguous()
    pos = torch.arange(8).view(1, 8) ^ (torch.arange(rows).view(-1, 1) & 7)
    return torch.gather(buf, 2, pos.view(1, rows, 8, 1).expand(num_kc, rows, 8, 4)).contiguous(), meta


# (layer, product removed): one decoder layer with tf32 inputs or tf32 weights
FAULTS = {"decoder1_deconv_tf32_inputs": ("rfc.decoder1.deconv", "lo_hi"),
          "decoder1_deconv_tf32_weights": ("rfc.decoder1.deconv", "hi_lo")}


@pytest.mark.parametrize("fault", list(FAULTS))
def test_stage_criteria_reject_one_layer_without_its_lo_term(fault):
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from comfyui_propainter_nodes_b200 import engine as E
    from comfyui_propainter_nodes_b200 import weights as Wt
    from tests.golden import cases
    layer, term = FAULTS[fault]
    sds = Wt.synthetic_raft_state_dict(), Wt.synthetic_rfc_state_dict(), Wt.synthetic_generator_state_dict()
    e = E.Engine(DEV, workspace_gb=4.0).load_weights(*sds)
    w, b = E.build_layers(*sds)[0][layer][:2]
    packed, meta = _image_without(w, term)
    e._register_packed(layer + ".tf32", packed, meta, w, b, None)
    flows, masks = cases.rfc_case()
    bad = _violations(_errors(fault, e, flows, masks, _bidir(e)))
    e.close()
    print(fault, "rejected by:", bad)
    assert bad, fault + " passes the stage criteria"


# ---- config[0] through the node's stages: what image propagation receives --------------------------------------------
def test_config0_completed_flow_in_the_hole_not_above_fp16(golden2):
    """BASELINE config[0] (16 frames, 320x176, fp16="disable"): on the same fp32 RAFT flows, the fp32 flow completion's
    mean |d| inside the hole against the reference's completed flow is not above the fp16 flow completion's."""
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from comfyui_propainter_nodes_b200 import propainter_inference as PI
    from comfyui_propainter_nodes_b200.utils import image_utils as IU
    from tests import gpu_checks as C
    from tests.golden import cases
    m = C.full_models()
    c = cases.c1_case()
    kw = c["kwargs"]
    T, H, W = c["image"].shape[:3]
    icfg = IU.ImageConfig(kw["width"], kw["height"], kw["mask_dilates"], kw["flow_mask_dilates"], (W, H), T)
    ft, fm, md, _ = IU.prepare_frames_and_masks(IU.convert_image_to_frames(c["image"]), c["mask"], icfg, torch.device(DEV))
    cfg = PI.ProPainterConfig(kw["ref_stride"], kw["neighbor_length"], kw["subvideo_length"], kw["raft_iter"], kw["fp16"],
                              T, torch.device(DEV), icfg.process_size)
    assert not cfg.use_half
    gt = PI.compute_flow(m.raft_model, ft, cfg)
    eng = m.flow_model.engine
    ref = torch.from_numpy(golden2["c1_pred_flow_f"]).float()[0]
    hole = (fm[0, :-1] > 0).expand(-1, 2, -1, -1).cpu()
    d = {}
    for fp32 in (True, False):
        of, _ = eng.flow_complete(gt[0][0], gt[1][0], fm[0], fp32=fp32)
        torch.cuda.synchronize()
        d[fp32] = float((of.cpu() - ref).abs()[hole].mean())
    print("config[0] completed flow, mean |d| in the hole: fp32", d[True], "fp16", d[False])
    assert hole.any() and d[True] <= d[False], d


# ---- several GPUs: the sharded fp32 flow completion equals the 1-GPU one ---------------------------------------------
def test_fp32_flow_completion_on_several_gpus_equals_one_gpu(tmp_path):
    """pp_flow_complete_dist_fp32 through parallel.complete_flow_distributed (teams, direction halves, frame shards with
    the encoder halo, NCCL all-gathers) on every GPU of the machine, against the 1-GPU fp32 result: bit-identical."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 or more GPUs")
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    n = min(torch.cuda.device_count(), 4)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}",
           "--master-addr=127.0.0.1", "--master-port=29517", os.path.join(root, "tools", "dist_check.py"),
           "20", "128", "160", "8", "disable"]
    res = subprocess.run(cmd, cwd=str(tmp_path), capture_output=True, text=True, timeout=1200)
    print(res.stdout[-2000:])
    assert res.returncode == 0, (res.stdout[-2000:], res.stderr[-4000:])
