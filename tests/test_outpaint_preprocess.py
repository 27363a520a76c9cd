"""The Outpaint node's device pre-processing (Engine.preprocess_outpaint -> pp_preprocess_outpaint_u8) against the host
path it replaces (convert_image_to_frames -> extrapolation -> prepare_frames_and_masks_for_outpaint): bit-identical
frames, band masks and uint8 canvas for every input size, the same node outputs, and the same rejections.

The GPU cases are marked ``gpu``; the node wiring and the input checks run on the CPU with a stub engine."""
import numpy as np
import pytest
import torch

from comfyui_propainter_nodes_b200 import propainter_nodes as PN
from comfyui_propainter_nodes_b200.utils import image_utils as IU

# id -> (T, H, W, width, height, width_scale, height_scale, (process_size, outpaint_size) set directly or None)
CASES = {
    "down_1280x720_horizontal_bands_inset": (3, 720, 1280, 640, 360, 1.2, 1.0, None),
    "odd_333x201_vertical_bands": (3, 201, 333, 320, 200, 1.0, 1.5, None),
    "up_96x72_both_bands_inset": (3, 72, 96, 160, 128, 1.2, 1.2, None),
    "bands_up_to_10px_no_inset_one_axis_resize": (3, 180, 320, 320, 176, 1.05, 1.1, None),
    "scale_1_empty_band": (3, 120, 200, 160, 96, 1.0, 1.0, None),
    "scaled_size_not_multiple_of_8": (3, 150, 250, 200, 120, 1.33, 1.17, None),
    # sizes the widgets cannot produce: odd frames, odd pw - rw and ph - rh (the floor in x0 / y0), x0 = 11 (inset)
    "odd_offsets": (3, 110, 190, 160, 96, 1.0, 1.0, ((157, 93), (180, 100))),
    "no_resize": (3, 96, 160, 160, 96, 1.5, 1.25, None),
}


def _config(case):
    T, H, W, w, h, ws, hs, sizes = case
    icfg = IU.ImageOutpaintConfig(w, h, 5, 8, (W, H), T, ws, hs)
    if sizes is not None:
        icfg.process_size, icfg.outpaint_size = sizes
    return icfg


def _clip(T, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(T, H, W, 3, generator=g) * 1.1 - 0.05        # values outside [0, 1] exercise the clip


def _host_path(image, icfg):
    canvas, flow_masks, masks_dilated = IU.extrapolation(IU.convert_image_to_frames(image), icfg)
    ft, fm, md, originals = IU.prepare_frames_and_masks_for_outpaint(canvas, flow_masks, masks_dilated,
                                                                     torch.device("cpu"))
    return ft, fm, md, torch.from_numpy(np.stack(originals))


@pytest.fixture(scope="module")
def C():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from tests import gpu_checks
    return gpu_checks


def _assert_equal(dev, ref):
    for name, a, b in zip(("frames", "flow_masks", "masks_dilated", "orig"), dev, ref):
        assert a.is_cuda and a.dtype == b.dtype and a.shape == b.shape, (name, a.dtype, a.shape, b.dtype, b.shape)
        assert torch.equal(a.cpu(), b), name


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_device_outpaint_preprocessing_is_bit_exact(C, case):
    icfg = _config(CASES[case])
    T, H, W = CASES[case][:3]
    image = _clip(T, H, W, seed=len(case))
    eng = C.full_models().raft_model.engine
    out = eng.preprocess_outpaint(image, icfg)
    ref = _host_path(image, icfg)
    pw, ph = icfg.outpaint_size
    assert tuple(out[0].shape) == (1, T, 3, ph, pw) and tuple(out[3].shape) == (T, ph, pw, 3)
    _assert_equal(out, ref)


@pytest.mark.gpu
def test_device_outpaint_preprocessing_of_a_device_image_is_bit_exact(C):
    icfg = IU.ImageOutpaintConfig(256, 144, 5, 8, (320, 180), 3, 1.25, 1.25)
    image = _clip(3, 180, 320, seed=7)
    eng = C.full_models().raft_model.engine
    _assert_equal(eng.preprocess_outpaint(image.cuda(), icfg), _host_path(image, icfg))


@pytest.mark.gpu
def test_outpaint_node_matches_the_host_path(C):
    """The node end to end: the same IMAGE and OUTPAINT_MASK, bit for bit, as the pipeline fed with the host path's
    tensors (160x136 -> 128x128, a 160x128 canvas: RAFT needs 128 px on each side)."""
    from comfyui_propainter_nodes_b200.propainter_inference import ProPainterConfig
    from comfyui_propainter_nodes_b200.synthetic import synthetic_clip
    models = C._node_models()
    image = synthetic_clip(8, 136, 160, 21)
    widgets = dict(width=128, height=128, width_scale=1.25, height_scale=1.0, mask_dilates=5, flow_mask_dilates=8,
                   ref_stride=10, neighbor_length=10, subvideo_length=80, raft_iter=4, fp16="enable")
    img, omask, ow, oh = PN.ProPainterOutpaint().propainter_outpainting(image, **widgets)
    icfg = IU.ImageOutpaintConfig(128, 128, 5, 8, (160, 136), 8, 1.25, 1.0)
    cfg = ProPainterConfig(10, 10, 80, 4, "enable", 8, torch.device(C.DEV), icfg.outpaint_size)
    ft, fm, md, orig = _host_path(image, icfg)
    dev = torch.device(C.DEV)
    ref_img, ref_mask, _ = PN._run(models, ft.to(dev), fm.to(dev), md.to(dev), orig, cfg)
    torch.cuda.synchronize()
    assert (ow, oh) == (160, 128) and tuple(img.shape) == (8, 128, 160, 3)
    assert torch.equal(img.cpu(), ref_img.cpu())
    assert torch.equal(omask.cpu(), ref_mask.cpu())


@pytest.mark.gpu
def test_pp_preprocess_outpaint_u8_rejects_sizes_that_do_not_fit(C):
    eng = C.full_models().raft_model.engine
    image = _clip(2, 40, 64, seed=3)
    for process_size, outpaint_size, match in (((64, 40), (56, 40), "do not fit"), ((64, 40), (64, 32), "do not fit"),
                                               ((48, 0), (48, 8), "bad size"), ((0, 32), (8, 32), "bad size")):
        icfg = IU.ImageOutpaintConfig(64, 40, 5, 8, (64, 40), 2)
        icfg.process_size, icfg.outpaint_size = process_size, outpaint_size
        with pytest.raises(RuntimeError, match=match):
            eng.preprocess_outpaint(image, icfg)


# ---- CPU: node wiring with a stub engine, and the input checks --------------------------------------------------------


class _StubEngine:
    def __init__(self):
        self.calls, self.reserved = [], []

    def reserve_for_clip(self, T, H, W):
        self.reserved.append((T, H, W))

    def preprocess_outpaint(self, image, icfg):
        self.calls.append((image, icfg))
        (pw, ph), T = icfg.outpaint_size, image.shape[0]
        return (torch.zeros(1, T, 3, ph, pw), torch.zeros(1, T, 1, ph, pw), torch.zeros(1, T, 1, ph, pw),
                torch.zeros(T, ph, pw, 3, dtype=torch.uint8))


def _host_path_must_not_run(*args, **kwargs):
    raise AssertionError("the host pre-processing ran")


@pytest.fixture
def stub_node(monkeypatch):
    """The Outpaint node with a stub engine: records what it is asked for and what reaches the pipeline."""
    from types import SimpleNamespace
    eng = _StubEngine()
    seen = {}

    def run(models, ft, fm, md, orig, cfg):
        seen["run"] = (ft, fm, md, orig, cfg)
        return torch.zeros(cfg.video_length, *cfg.process_size[::-1], 3), fm[0, :, 0], md[0, :, 0]

    def init(device, use_half):
        seen["models"] = SimpleNamespace(raft_model=SimpleNamespace(engine=eng))
        return seen["models"]

    monkeypatch.setattr(PN, "_compute_device", lambda: torch.device("cpu"))
    monkeypatch.setattr(PN, "initialize_models", init)
    monkeypatch.setattr(PN, "_run", run)
    return eng, seen


def _widgets(width, height, width_scale, height_scale):
    return dict(width=width, height=height, width_scale=width_scale, height_scale=height_scale, mask_dilates=5,
                flow_mask_dilates=8, ref_stride=10, neighbor_length=10, subvideo_length=80, raft_iter=20, fp16="enable")


@pytest.mark.parametrize("H,W,width,height", [(72, 128, 64, 40), (40, 64, 64, 40)], ids=["resize", "no_resize"])
def test_outpaint_node_preprocesses_on_the_engine(stub_node, monkeypatch, H, W, width, height):
    eng, seen = stub_node
    for name in ("convert_image_to_frames", "extrapolation", "prepare_frames_and_masks_for_outpaint",
                 "outpaint_tensors"):
        monkeypatch.setattr(IU, name, _host_path_must_not_run)
    image = torch.rand(3, H, W, 3)
    img, omask, ow, oh = PN.ProPainterOutpaint().propainter_outpainting(image, **_widgets(width, height, 1.25, 1.2))
    assert len(eng.calls) == 1 and eng.calls[0][0] is image
    icfg = eng.calls[0][1]
    assert tuple(icfg.input_size) == (W, H) and tuple(icfg.process_size) == (64, 40)
    assert tuple(icfg.outpaint_size) == (80, 48) == (ow, oh)
    assert eng.reserved == [(3, 48, 80)]
    ft, fm, md, orig, cfg = seen["run"]
    assert tuple(ft.shape) == (1, 3, 3, 48, 80) and tuple(orig.shape) == (3, 48, 80, 3)
    assert tuple(cfg.process_size) == (80, 48) and cfg.video_length == 3
    assert tuple(omask.shape) == (3, 48, 80)


def _host_error(image, icfg):
    """The exception the host pre-processing raises on these inputs (None when it accepts them)."""
    try:
        if tuple(icfg.process_size) == tuple(icfg.input_size):
            IU.outpaint_tensors(image, icfg, torch.device("cpu"))
        else:
            _host_path(image, icfg)
    except Exception as e:  # noqa: BLE001 -- the type is what is compared
        return type(e)
    return None


# (T, H, W, width, height, width_scale, height_scale)
REJECTED = {
    "resize_width_scale_below_1": (2, 72, 128, 64, 40, 0.9, 1.0),
    "resize_height_scale_below_1": (2, 72, 128, 64, 40, 1.0, 0.5),
    "resize_width_scale_0": (2, 72, 128, 64, 40, 0.0, 1.0),
    "resize_both_scales_below_1": (2, 72, 128, 64, 40, 0.5, 0.5),
    "resize_width_below_8": (2, 72, 128, 5, 40, 1.2, 1.0),
    "resize_height_below_8": (2, 72, 128, 64, 7, 1.2, 1.0),
    "resize_no_frames": (0, 72, 128, 64, 40, 1.2, 1.0),
    "no_resize_width_scale_below_1": (2, 40, 64, 64, 40, 0.99, 1.0),
    "no_resize_height_scale_0": (2, 40, 64, 64, 40, 1.0, 0.0),
}


@pytest.mark.parametrize("case", list(REJECTED))
def test_outpaint_node_rejects_what_the_host_path_rejected(stub_node, case):
    T, H, W, w, h, ws, hs = REJECTED[case]
    image = torch.rand(T, H, W, 3)
    expected = _host_error(image, IU.ImageOutpaintConfig(w, h, 5, 8, (W, H), T, ws, hs))
    assert expected is not None, case
    with pytest.raises(expected):
        PN.ProPainterOutpaint().propainter_outpainting(image, **_widgets(w, h, ws, hs))
    assert "models" not in stub_node[1]             # rejected before any model is loaded


def test_outpaint_node_rejects_an_empty_clip_without_resize(stub_node):
    """Without a resize the host path accepted an empty clip and the pipeline failed on it with RuntimeError (RAFT's
    flow buffers of T - 1 frames)."""
    with pytest.raises(RuntimeError):
        PN.ProPainterOutpaint().propainter_outpainting(torch.rand(0, 40, 64, 3), **_widgets(64, 40, 1.2, 1.0))
    assert "models" not in stub_node[1]
