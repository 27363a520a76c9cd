"""ComfyUI nodes "ProPainter Inpainting" / "ProPainter Outpainting" backed by the sm_90a engine.

Drop-in for the reference's propainter_nodes.py: same node keys, display names, INPUT_TYPES (names, order,
defaults, ranges), RETURN_TYPES / RETURN_NAMES, FUNCTION and CATEGORY (reference propainter_nodes.py:38-321).
Outputs: IMAGE float32 [T,h,w,3] on the CPU at the processing size (width/height rounded down to a multiple
of 8, not resized back), masks squeezed to [T,h,w] and left on the compute device, as the reference does.
"""
from __future__ import annotations

import os

import numpy as np
import torch

from .propainter_inference import ProPainterConfig, feature_propagation_device, process_inpainting
from .utils import image_utils as iu
from .utils.model_utils import initialize_models


def _compute_device() -> torch.device:
    try:  # inside ComfyUI
        from comfy import model_management
        return model_management.get_torch_device()
    except ImportError:
        return torch.device("cuda", torch.cuda.current_device())


def check_inputs(frames: torch.Tensor, masks: torch.Tensor) -> None:
    """Same three conditions and bare ``Exception`` type as the reference (propainter_nodes.py:21-35)."""
    n_img, n_msk = frames.size(dim=0), masks.size(dim=0)
    if n_img <= 1:
        raise Exception(f"Image length must be greater than 1, but got:\n Image length: ({n_img})")
    if n_msk not in (1, n_img):
        raise Exception("Image and Mask must have the same length or Mask have length 1, but got:\n"
                        f" Image length: {n_img}\n Mask length: {n_msk}")
    if tuple(frames.shape[1:3]) != tuple(masks.shape[1:3]):
        raise Exception("Image and Mask must have the same dimensions, but got:\n"
                        f" Image: ({frames.size(dim=1)}, {frames.size(dim=2)})\n"
                        f" Mask: ({masks.size(dim=1)}, {masks.size(dim=2)})")


def check_outpaint_sizes(icfg: iu.ImageOutpaintConfig, n: int) -> None:
    """The Outpaint node's input checks.  The reference performs none, and its pre-processing fails in PIL, numpy or
    torch instead; these raise the same exception types, before any model is loaded.  With a resize: an empty clip
    IndexError, a processing size of zero or a canvas smaller than the frames ValueError.  Without one: RuntimeError."""
    (rw, rh), (pw, ph) = icfg.process_size, icfg.outpaint_size
    resize = tuple(icfg.process_size) != tuple(icfg.input_size)
    if n == 0:
        raise (IndexError if resize else RuntimeError)("Outpainting needs at least one frame")
    if resize and (rw <= 0 or rh <= 0):
        raise ValueError(f"height and width must be > 0, but the processing size is {rw}x{rh}")
    if pw < rw or ph < rh:
        raise (ValueError if resize else RuntimeError)(
            f"The {rw}x{rh} frames do not fit the {pw}x{ph} outpainting canvas: width_scale and height_scale must not "
            "shrink it below the processing size")


def _int(default, lo, hi):
    return ("INT", {"default": default, "min": lo, "max": hi})


def _scale(default):
    return ("FLOAT", {"default": default, "min": 0.0, "max": 10.0, "step": 0.01})


_SIZE_WIDGETS = (("width", _int(640, 0, 2560)), ("height", _int(360, 0, 2560)))
_TUNING_WIDGETS = (
    ("mask_dilates", _int(5, 0, 100)),
    ("flow_mask_dilates", _int(8, 0, 100)),
    ("ref_stride", _int(10, 1, 100)),
    ("neighbor_length", _int(10, 2, 300)),
    ("subvideo_length", _int(80, 1, 300)),
    ("raft_iter", _int(20, 1, 100)),
    ("fp16", (["enable", "disable"],)),
)


def _run(models, frames_t, flow_masks_t, masks_dilated_t, originals_u8, cfg: ProPainterConfig):
    """originals_u8: uint8 [T,H,W,3] tensor (host or device)."""
    print(f"\nProcessing  {cfg.video_length} frames...")
    w, h = cfg.process_size
    models.raft_model.engine.reserve_for_clip(cfg.video_length, h, w)    # arena sized from the clip (no-op when fixed)
    updated_frames, updated_masks, flows = process_inpainting(models, frames_t, flow_masks_t, masks_dilated_t, cfg)
    comp = feature_propagation_device(models.inpaint_model, updated_frames, updated_masks, masks_dilated_t, flows,
                                      originals_u8, cfg)
    images = models.inpaint_model.engine.postprocess(comp)
    if os.environ.get("PP_IMAGE_ON_DEVICE", "0") in ("", "0"):
        images = _to_host(images)          # default: the IMAGE is a CPU tensor like the reference's (handle_output)
    # PP_IMAGE_ON_DEVICE=1: zero-copy hand-over -- the float32 IMAGE stays in HBM for downstream nodes that take CUDA
    # tensors (saves the 221 MB device->host copy of an 80-frame 640x360 result, ~9 ms)
    return images, flow_masks_t.squeeze(), masks_dilated_t.squeeze()


def _to_host(dev: torch.Tensor) -> torch.Tensor:
    """Device -> host copy of the IMAGE result into page-locked memory from torch's caching host allocator.

    A fresh pageable 221 MB tensor (80 frames 640x360 float32) costs 60-90 ms of page faults per call on the GPU
    host (measured, tools/e2e_breakdown.py); a pinned block is recycled by the allocator once the previous result
    has been released, never while a caller still holds it, and the copy runs at PCIe rate."""
    try:
        host = torch.empty(dev.shape, dtype=dev.dtype, device="cpu", pin_memory=True)
    except RuntimeError:        # locked-memory limit reached (results held by a caller stay pinned): pageable copy
        return dev.cpu()
    host.copy_(dev, non_blocking=True)
    torch.cuda.current_stream(dev.device).synchronize()
    return host


class ProPainterInpaint:
    """Video inpainting of the masked region."""

    RETURN_TYPES = ("IMAGE", "MASK", "MASK")
    RETURN_NAMES = ("IMAGE", "FLOW_MASK", "MASK_DILATE")
    FUNCTION = "propainter_inpainting"
    CATEGORY = "ProPainter"

    @classmethod
    def INPUT_TYPES(cls):
        req = {"image": ("IMAGE",), "mask": ("MASK",)}
        req.update(_SIZE_WIDGETS)
        req.update(_TUNING_WIDGETS)
        return {"required": req}

    def propainter_inpainting(self, image, mask, width, height, mask_dilates, flow_mask_dilates, ref_stride,
                              neighbor_length, subvideo_length, raft_iter, fp16):
        check_inputs(image, mask)
        device = _compute_device()
        n = image.size(dim=0)
        input_size = (image.size(dim=2), image.size(dim=1))       # (width, height) like PIL's Image.size
        icfg = iu.ImageConfig(width, height, mask_dilates, flow_mask_dilates, input_size, n)
        cfg = ProPainterConfig(ref_stride, neighbor_length, subvideo_length, raft_iter, fp16, n, device,
                               icfg.process_size)
        models = initialize_models(cfg.device, cfg.fp16)
        if mask.dtype == torch.float32:
            # quantisation, PIL's 8-bit bicubic resize and the mask dilations run on the device with the reference's
            # integer semantics, bit for bit (float32 masks only: the reference scales only those by 255, other dtypes
            # go to PIL unscaled -- host path below)
            eng = models.raft_model.engine
            eng.reserve_for_clip(n, icfg.process_size[1], icfg.process_size[0])
            ft, fm, md, orig = eng.preprocess(image, mask, flow_mask_dilates, mask_dilates, icfg.process_size)
        else:
            ft, fm, md, originals = iu.prepare_frames_and_masks(iu.convert_image_to_frames(image), mask, icfg, device)
            orig = torch.from_numpy(np.stack(originals))
        return _run(models, ft, fm, md, orig, cfg)


class ProPainterOutpaint:
    """Video outpainting: the clip is centred on a larger canvas and the border band is synthesised."""

    RETURN_TYPES = ("IMAGE", "MASK", "INT", "INT")
    RETURN_NAMES = ("IMAGE", "OUTPAINT_MASK", "output_width", "output_height")
    FUNCTION = "propainter_outpainting"
    CATEGORY = "ProPainter"

    @classmethod
    def INPUT_TYPES(cls):
        req = {"image": ("IMAGE",)}
        req.update(_SIZE_WIDGETS)
        req.update((("width_scale", _scale(1.2)), ("height_scale", _scale(1.0))))
        req.update(_TUNING_WIDGETS)
        return {"required": req}

    def propainter_outpainting(self, image, width, height, width_scale, height_scale, mask_dilates,
                               flow_mask_dilates, ref_stride, neighbor_length, subvideo_length, raft_iter, fp16):
        device = _compute_device()
        n = image.size(dim=0)
        input_size = (image.size(dim=2), image.size(dim=1))
        icfg = iu.ImageOutpaintConfig(width, height, mask_dilates, flow_mask_dilates, input_size, n,
                                      width_scale, height_scale)
        cfg = ProPainterConfig(ref_stride, neighbor_length, subvideo_length, raft_iter, fp16, n, device,
                               icfg.outpaint_size)
        check_outpaint_sizes(icfg, n)
        models = initialize_models(cfg.device, cfg.fp16)
        # quantisation, PIL's 8-bit bicubic resize, the canvas and its band masks run on the device with the reference's
        # integer semantics, bit for bit
        eng = models.raft_model.engine
        pw, ph = icfg.outpaint_size
        eng.reserve_for_clip(n, ph, pw)
        ft, fm, md, orig = eng.preprocess_outpaint(image, icfg)
        images, out_masks, _ = _run(models, ft, fm, md, orig, cfg)
        out_w, out_h = cfg.process_size
        return images, out_masks, out_w, out_h


NODE_CLASS_MAPPINGS = {"ProPainterInpaint": ProPainterInpaint, "ProPainterOutpaint": ProPainterOutpaint}
NODE_DISPLAY_NAME_MAPPINGS = {"ProPainterInpaint": "ProPainter Inpainting",
                              "ProPainterOutpaint": "ProPainter Outpainting"}
