"""Model residency: three checkpoints -> one packed sm_90a engine (reference: utils/model_utils.py:13-59).

``Models`` keeps the reference's three fields; each is a thin stage handle sharing one ``Engine``.
Checkpoints are the reference's ``.pth`` state_dict files under ``<package>/weights/``
(raft-things.pth, recurrent_flow_completion.pth, ProPainter.pth).  Unlike the reference, which reloads the
three files on every node execution, the packed engine stays resident: the cache is keyed by the device AND the
SHA-256 of the checkpoint files (re-hashed only when a file's size / mtime changes), so swapping a file in
``weights/`` rebuilds the engine instead of silently keeping the old weights.  There is no download step here
(no network); place the files, or pass state dicts to ``build_models``.
"""
from __future__ import annotations

import hashlib
import os
from dataclasses import dataclass

import torch

WEIGHTS_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "weights")
CHECKPOINTS = ("raft-things.pth", "recurrent_flow_completion.pth", "ProPainter.pth")


class StageHandle:
    """What the orchestration functions receive where the reference passes an nn.Module."""

    def __init__(self, engine, stage: str):
        self.engine = engine
        self.stage = stage

    def __repr__(self):
        return f"<propainter_b200 stage '{self.stage}' on {self.engine.device}>"


@dataclass
class Models:
    raft_model: StageHandle
    flow_model: StageHandle
    inpaint_model: StageHandle


_CACHE = {}        # (device string, checkpoint key) -> Models
_RESIDENT = {}     # device string -> Models installed by set_resident_models (tests, bench: synthetic weights)
_FILE_HASH = {}    # path -> ((size, mtime_ns), sha256 hex)


def file_sha256(path: str) -> str:
    """SHA-256 of a checkpoint file, recomputed only when its size or mtime changed."""
    st = os.stat(path)
    sig = (st.st_size, st.st_mtime_ns)
    hit = _FILE_HASH.get(path)
    if hit is not None and hit[0] == sig:
        return hit[1]
    h = hashlib.sha256()
    with open(path, "rb") as fh:
        for block in iter(lambda: fh.read(1 << 22), b""):
            h.update(block)
    _FILE_HASH[path] = (sig, h.hexdigest())
    return _FILE_HASH[path][1]


def checkpoint_key(paths) -> tuple:
    return tuple(file_sha256(p) for p in paths)


def build_models(device, raft_sd, rfc_sd, gen_sd, workspace_gb: float | None = None) -> Models:
    """``workspace_gb=None``: the scratch arena starts small and is sized per clip (``Engine.reserve_for_clip``)."""
    from ..engine import Engine
    eng = Engine(device, workspace_gb=workspace_gb).load_weights(raft_sd, rfc_sd, gen_sd)
    return Models(StageHandle(eng, "raft"), StageHandle(eng, "flow_completion"), StageHandle(eng, "inpaint"))


def set_resident_models(device, models: Models | None) -> None:
    """Install (or, with None, remove) models that ``initialize_models`` returns for `device` without touching
    ``weights/`` -- how tests and the bench run the node classes on synthetic checkpoints."""
    key = str(torch.device(device))
    if models is None:
        _RESIDENT.pop(key, None)
    else:
        _RESIDENT[key] = models


def release_models(device=None) -> None:
    """Drop cached engines (all devices, or one) and give their HBM back to the allocator -- the hook for ComfyUI's
    model-unload / soft_empty_cache path; the next node execution rebuilds from the checkpoint files."""
    keys = [k for k in _CACHE if device is None or k[0] == str(torch.device(device))]
    for k in keys:
        _CACHE.pop(k).raft_model.engine.close()
    if torch.cuda.is_available():
        torch.cuda.empty_cache()


def initialize_models(device: torch.device, use_half: str = "enable") -> Models:
    """Load the three checkpoints from ``weights/`` (same files as the reference) into a cached engine."""
    dkey = str(torch.device(device))
    if dkey in _RESIDENT:
        return _RESIDENT[dkey]
    paths = [os.path.join(WEIGHTS_DIR, n) for n in CHECKPOINTS]
    missing = [p for p in paths if not os.path.exists(p)]
    if missing:
        raise FileNotFoundError(
            "ProPainter checkpoints not found: " + ", ".join(missing) +
            " (download raft-things.pth, recurrent_flow_completion.pth and ProPainter.pth from the "
            "sczhou/ProPainter v0.1.0 release into the weights/ directory)")
    key = (dkey, checkpoint_key(paths))
    if key not in _CACHE:
        for stale in [k for k in _CACHE if k[0] == dkey]:      # a checkpoint changed: free the old engine first
            _CACHE.pop(stale).raft_model.engine.close()
        sds = [torch.load(p, map_location="cpu") for p in paths]
        _CACHE[key] = build_models(device, *sds)
    return _CACHE[key]
