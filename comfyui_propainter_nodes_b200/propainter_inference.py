"""Inference orchestration with the reference's entry points, executed by the sm_90a engine.

Same public names and argument meaning as the reference's ``propainter_inference.py``
(ProPainterConfig, get_ref_index, compute_flow, complete_flow, image_propagation, feature_propagation,
process_inpainting), so ``propainter_nodes`` and external callers read the same.  Each function calls the C ABI
exactly where the reference calls its PyTorch modules:

* compute_flow        -> Engine.raft_bidir        (reference propainter_inference.py:61-99)
* complete_flow       -> Engine.flow_complete     (:102-156, chunks of subvideo_length with a 5-flow halo)
* image_propagation   -> Engine.image_propagate   (:159-225, chunks of min(100, subvideo_length) with a 10-frame halo)
* feature_propagation -> Engine.gen_begin/gen_window/composite (:228-311)

Tensors keep the reference layouts ([1,T,C,H,W]).  RAFT follows the ``fp16`` switch: "enable" runs it with fp16
activations and fp32 accumulation, "disable" at fp32 accuracy (fp32 activations, 3xTF32 GEMMs), like the reference,
which always runs RAFT in fp32.  Image propagation follows it too: "disable" keeps frames, masks and flows in fp32
(pp_image_propagate_fp32), "enable" stores them in fp16.  So does flow completion: "disable" runs it at fp32 accuracy
(pp_flow_complete_fp32: fp32 activations, 3xTF32 GEMMs, fp32 deformable sampling), "enable" with fp16 activations and
fp32 accumulation.  The generator computes in fp16 with fp32 accumulation in both modes (there the switch only selects
the dtype of the tensors handed back).
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np
import torch

from .utils.model_utils import Models


@dataclass
class ProPainterConfig:
    ref_stride: int
    neighbor_length: int
    subvideo_length: int
    raft_iter: int
    fp16: str
    video_length: int
    device: torch.device
    process_size: tuple
    use_half: bool = field(init=False)

    def __post_init__(self) -> None:
        self.use_half = self.fp16 == "enable" and torch.device(self.device).type != "cpu"


def get_ref_index(mid_neighbor_id: int, neighbor_ids: list, config: ProPainterConfig, ref_num: int = -1) -> list:
    """Global reference frames of a window (reference propainter_inference.py:36-58)."""
    if ref_num == -1:
        return [i for i in range(0, config.video_length, config.ref_stride) if i not in neighbor_ids]
    half = config.ref_stride * (ref_num // 2)
    lo, hi = max(0, mid_neighbor_id - half), min(config.video_length, mid_neighbor_id + half)
    picked = []
    for i in range(lo, hi, config.ref_stride):
        if i in neighbor_ids:
            continue
        if len(picked) > ref_num:  # the reference stops one past ref_num
            break
        picked.append(i)
    return picked


def _out_dtype(config):
    return torch.float16 if config.use_half else torch.float32


def compute_flow(raft_model, frames: torch.Tensor, config: ProPainterConfig):
    """Bidirectional RAFT flow of the whole clip, fp32 -> 2 x [1,T-1,2,H,W].

    The reference splits the clip into <=12/8/4/2-frame pieces only to bound memory; pairs are independent,
    so the engine batches all of them (it chunks internally against its workspace)."""
    eng = raft_model.engine
    ff, fb = eng.raft_bidir(frames[0], config.raft_iter, fp32=not config.use_half)
    return ff.unsqueeze(0), fb.unsqueeze(0)


def complete_flow(recurrent_flow_model, flows_tuple, flow_masks: torch.Tensor, subvideo_length: int):
    """Recurrent flow completion, chunked exactly like the reference (temporal convs see the 5-flow halo).

    The precision follows the dtype of the flows process_inpainting hands over, as the reference's network follows
    ``fp16``: float32 (fp16="disable") runs at fp32 accuracy, float16 with fp16 activations."""
    eng = recurrent_flow_model.engine
    ff, fb, fm = flows_tuple[0][0], flows_tuple[1][0], flow_masks[0]
    dt = flows_tuple[0].dtype
    fp32 = dt == torch.float32
    L = ff.shape[0]
    if L <= subvideo_length:
        of, ob = eng.flow_complete(ff, fb, fm, fp32=fp32)
    else:
        pad = 5
        pf, pb = [], []
        for f in range(0, L, subvideo_length):
            s, e = max(0, f - pad), min(L, f + subvideo_length + pad)
            ps, pe = f - s, e - min(L, f + subvideo_length)
            a, b = eng.flow_complete(ff[s:e], fb[s:e], fm[s:e + 1], fp32=fp32)
            pf.append(a[ps:e - s - pe])
            pb.append(b[ps:e - s - pe])
        of, ob = torch.cat(pf, 0), torch.cat(pb, 0)
    return of.unsqueeze(0).to(dt), ob.unsqueeze(0).to(dt)


def image_propagation(inpaint_model, frames: torch.Tensor, masks_dilated: torch.Tensor, prediction_flows,
                      config: ProPainterConfig):
    """Non-learnable pixel propagation -> (updated_frames [1,T,3,H,W], updated_masks [1,T,1,H,W]).

    fp16="disable" keeps frames and flows in fp32 through the propagation (its decisions are discrete: an fp16 flow
    moves whole pixels); "enable" stores them in fp16."""
    eng = inpaint_model.engine
    fr, md = frames[0], masks_dilated[0]
    ff, fb = prediction_flows[0][0], prediction_flows[1][0]
    dt = frames.dtype
    T = config.video_length
    fp32 = not config.use_half
    sub = min(100, config.subvideo_length)
    if T <= sub:
        uf, um = eng.image_propagate(fr, md, ff, fb, fp32=fp32)
    else:
        pad = 10
        lf, lm = [], []
        for f in range(0, T, sub):
            s, e = max(0, f - pad), min(T, f + sub + pad)
            ps, pe = f - s, e - min(T, f + sub)
            a, b = eng.image_propagate(fr[s:e], md[s:e], ff[s:e - 1], fb[s:e - 1], fp32=fp32)
            lf.append(a[ps:e - s - pe])
            lm.append(b[ps:e - s - pe])
        uf, um = torch.cat(lf, 0), torch.cat(lm, 0)
    return uf.unsqueeze(0).to(dt), um.unsqueeze(0).to(dt)


def window_schedule(config: ProPainterConfig):
    """[(neighbor_ids, ref_ids)] walked by feature_propagation (reference :245-262)."""
    stride = config.neighbor_length // 2
    ref_num = config.subvideo_length // config.ref_stride if config.video_length > config.subvideo_length else -1
    out = []
    for f in range(0, config.video_length, stride):
        nb = list(range(max(0, f - stride), min(config.video_length, f + stride + 1)))
        out.append((nb, get_ref_index(f, nb, config, ref_num)))
    return out


def feature_propagation_device(inpaint_model, updated_frames, updated_masks, masks_dilated, prediction_flows,
                               original_frames_u8: torch.Tensor, config: ProPainterConfig, windows=None) -> torch.Tensor:
    """Sliding-window generator + device composite.  Returns uint8 [T,H,W,3] on the device.

    ``windows`` restricts the schedule to a subset (multi-GPU sharding); frames not touched stay zero."""
    eng = inpaint_model.engine
    dev = eng.device
    T = config.video_length
    sched = window_schedule(config)
    if windows is not None:
        sched = [sched[i] for i in windows]
    md = masks_dilated[0].to(device=dev, dtype=torch.float32).contiguous()
    orig = original_frames_u8.to(dev).contiguous()
    comp = torch.zeros_like(orig)
    eng.gen_begin(updated_frames[0], md, updated_masks[0], prediction_flows[0][0], prediction_flows[1][0])
    try:
        # every window of the schedule in one batched engine pass (sub-batches when the workspace is small)
        preds = eng.gen_run(sched)
    finally:
        eng.gen_end()           # the session's arena share is returned on every exit
    # the order-dependent uint8 composite
    flat_ids, first = [], []
    visited = [False] * T
    for nb, _ in sched:
        for i in nb:
            flat_ids.append(i)
            first.append(0 if visited[i] else 1)
            visited[i] = True
    ids_dev = torch.tensor(flat_ids, dtype=torch.int32, device=dev)
    first_dev = torch.tensor(first, dtype=torch.int32, device=dev)
    o = 0
    for nb, _ in sched:   # windows in order: frames shared by consecutive windows are blended 0.5/0.5 in this order
        n = len(nb)
        eng.composite(preds[o:o + n], md, orig, comp, ids_dev[o:o + n], first_dev[o:o + n], config.use_half)
        o += n
    return comp


def feature_propagation(inpaint_model, updated_frames, updated_masks, masks_dilated, prediction_flows,
                        original_frames, config: ProPainterConfig) -> list:
    """Reference-compatible signature: original_frames is a list of HxWx3 uint8 arrays; returns such a list."""
    orig = torch.from_numpy(np.stack(original_frames).astype(np.uint8))
    comp = feature_propagation_device(inpaint_model, updated_frames, updated_masks, masks_dilated, prediction_flows,
                                      orig, config)
    out = comp.cpu().numpy()
    return [out[i] for i in range(out.shape[0])]


def process_inpainting(models: Models, frames: torch.Tensor, flow_masks: torch.Tensor, masks_dilated: torch.Tensor,
                       config: ProPainterConfig):
    """RAFT -> flow completion -> image propagation (reference :314-341)."""
    with torch.no_grad():
        gt_flows_bi = compute_flow(models.raft_model, frames, config)
        dt = _out_dtype(config)
        frames, flow_masks, masks_dilated = frames.to(dt), flow_masks.to(dt), masks_dilated.to(dt)
        gt_flows_bi = (gt_flows_bi[0].to(dt), gt_flows_bi[1].to(dt))
        pred_flows_bi = complete_flow(models.flow_model, gt_flows_bi, flow_masks, config.subvideo_length)
        updated_frames, updated_masks = image_propagation(models.inpaint_model, frames, masks_dilated, pred_flows_bi,
                                                          config)
    return updated_frames, updated_masks, pred_flows_bi
