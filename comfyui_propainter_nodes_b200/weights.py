"""Checkpoint contract of the three ProPainter networks + a seeded synthetic generator.

The reference loads three PyTorch ``state_dict`` files with ``strict=True``
(reference: model/modules/flow_comp_raft.py:17-19, model/recurrent_flow_completion.py:310-313,
model/propainter.py:342-345).  This module restates that contract as a table of
``key -> shape`` built by loops (``raft_spec`` / ``rfc_spec`` / ``generator_spec``), so that

* real checkpoints can be validated before they are packed for the CUDA engine, and
* parity tests and the bench can build *seeded synthetic* checkpoints on a box that has
  no network (there are no pretrained files in this environment).

The synthetic initialisation is not the reference's training init: it is tuned so that every
stage stays numerically well-conditioned with random weights (recurrent residual branches are
damped, the DCN offset heads are non-zero so the deformable sampler is exercised, the RAFT flow
head is small so 20 GRU iterations do not diverge).
"""
from __future__ import annotations

import math
from collections import OrderedDict

import numpy as np
import torch

# ----------------------------------------------------------------------------------------------
# key/shape tables
# ----------------------------------------------------------------------------------------------


def _conv(spec, name, cout, cin, kh, kw=None, bias=True):
    kw = kh if kw is None else kw
    spec[name + ".weight"] = (cout, cin, kh, kw)
    if bias:
        spec[name + ".bias"] = (cout,)


def _bn(spec, name, c):
    spec[name + ".weight"] = (c,)
    spec[name + ".bias"] = (c,)
    spec[name + ".running_mean"] = (c,)
    spec[name + ".running_var"] = (c,)
    spec[name + ".num_batches_tracked"] = ()


def _raft_encoder(spec, p, out_dim, batchnorm):
    """BasicEncoder (reference: model/modules/RAFT/extractor.py:121-193)."""
    if batchnorm:
        _bn(spec, p + "norm1", 64)
    _conv(spec, p + "conv1", 64, 3, 7)
    cin = 64
    for li, (dim, stride) in enumerate([(64, 1), (96, 2), (128, 2)], start=1):
        for bi in range(2):
            q = f"{p}layer{li}.{bi}."
            s = stride if bi == 0 else 1
            _conv(spec, q + "conv1", dim, cin, 3)
            _conv(spec, q + "conv2", dim, dim, 3)
            if batchnorm:
                _bn(spec, q + "norm1", dim)
                _bn(spec, q + "norm2", dim)
                if s != 1:
                    _bn(spec, q + "norm3", dim)
            if s != 1:
                _conv(spec, q + "downsample.0", dim, cin, 1)
                if batchnorm:
                    _bn(spec, q + "downsample.1", dim)  # same module object as norm3
            cin = dim
    _conv(spec, p + "conv2", out_dim, 128, 1)


def raft_spec() -> "OrderedDict[str, tuple]":
    """RAFT-things (full model) keys, without the ``module.`` DataParallel prefix."""
    s: OrderedDict = OrderedDict()
    _raft_encoder(s, "fnet.", 256, batchnorm=False)
    _raft_encoder(s, "cnet.", 256, batchnorm=True)
    u = "update_block."
    _conv(s, u + "encoder.convc1", 256, 324, 1)
    _conv(s, u + "encoder.convc2", 192, 256, 3)
    _conv(s, u + "encoder.convf1", 128, 2, 7)
    _conv(s, u + "encoder.convf2", 64, 128, 3)
    _conv(s, u + "encoder.conv", 126, 256, 3)
    for n in ("z", "r", "q"):
        _conv(s, u + f"gru.conv{n}1", 128, 384, 1, 5)
    for n in ("z", "r", "q"):
        _conv(s, u + f"gru.conv{n}2", 128, 384, 5, 1)
    _conv(s, u + "flow_head.conv1", 256, 128, 3)
    _conv(s, u + "flow_head.conv2", 2, 256, 3)
    _conv(s, u + "mask.0", 256, 128, 3)
    _conv(s, u + "mask.2", 576, 256, 1)
    return s


def rfc_spec() -> "OrderedDict[str, tuple]":
    """RecurrentFlowCompleteNet keys (reference: model/recurrent_flow_completion.py:236-308)."""
    s: OrderedDict = OrderedDict()
    s["downsample.0.weight"] = (32, 3, 1, 5, 5)
    s["downsample.0.bias"] = (32,)
    for enc, chans in (("encoder1", [(32, 32), (64, 32)]), ("encoder2", [(64, 64), (128, 64)])):
        for idx, (co, ci) in zip((0, 2), chans):
            s[f"{enc}.{idx}.conv1.0.weight"] = (co, ci, 1, 3, 3)
            s[f"{enc}.{idx}.conv1.0.bias"] = (co,)
            s[f"{enc}.{idx}.conv2.0.weight"] = (co, co, 3, 1, 1)
            s[f"{enc}.{idx}.conv2.0.bias"] = (co,)
    for i in (0, 2, 4):
        s[f"mid_dilation.{i}.weight"] = (128, 128, 1, 3, 3)
        s[f"mid_dilation.{i}.bias"] = (128,)
    fp = "feat_prop_module."
    for d in ("backward_", "forward_"):
        a = fp + "deform_align." + d
        s[a + ".weight"] = (128, 256, 3, 3)
        s[a + ".bias"] = (128,)
        _conv(s, a + ".conv_offset.0", 128, 384, 3)
        _conv(s, a + ".conv_offset.2", 128, 128, 3)
        _conv(s, a + ".conv_offset.4", 128, 128, 3)
        _conv(s, a + ".conv_offset.6", 432, 128, 3)
    for i, d in enumerate(("backward_", "forward_")):
        _conv(s, fp + f"backbone.{d}.0", 128, (2 + i) * 128, 3)
        _conv(s, fp + f"backbone.{d}.2", 128, 128, 3)
    _conv(s, fp + "fusion", 128, 256, 1)
    _conv(s, "decoder2.0", 128, 128, 3)
    _conv(s, "decoder2.2.conv", 64, 128, 3)
    _conv(s, "decoder1.0", 64, 64, 3)
    _conv(s, "decoder1.2.conv", 32, 64, 3)
    _conv(s, "upsample.0", 32, 32, 3)
    _conv(s, "upsample.2.conv", 2, 32, 3)
    # training-only edge head: present in the checkpoint (strict load), never executed in eval
    _conv(s, "edgeDetector.projection.0", 16, 2, 3)
    _conv(s, "edgeDetector.mid_layer_1.0", 16, 16, 3)
    _conv(s, "edgeDetector.mid_layer_2.0", 16, 16, 3)
    _conv(s, "edgeDetector.out_layer", 1, 16, 1)
    # the reference orders deform_align(backward_, forward_) fully before backbone; dict order
    # is irrelevant for loading, only the key set matters.
    return s


N_TRANSFORMER_BLOCKS = 8
FFN_HIDDEN = 1960  # 40 channels x 7x7 (reference: model/modules/sparse_transformer.py:79-90)


def generator_spec() -> "OrderedDict[str, tuple]":
    """InpaintGenerator keys (reference: model/propainter.py:294-348)."""
    s: OrderedDict = OrderedDict()
    enc = [(0, 64, 5), (2, 64, 64), (4, 128, 64), (6, 256, 128), (8, 384, 256),
           (10, 512, 320), (12, 384, 192), (14, 256, 80), (16, 128, 512)]
    for idx, co, ci in enc:
        _conv(s, f"encoder.layers.{idx}", co, ci, 3)
    _conv(s, "decoder.0.conv", 128, 128, 3)
    _conv(s, "decoder.2", 64, 128, 3)
    _conv(s, "decoder.4.conv", 64, 64, 3)
    _conv(s, "decoder.6", 3, 64, 3)
    s["ss.embedding.weight"] = (512, 6272)
    s["ss.embedding.bias"] = (512,)
    s["sc.embedding.weight"] = (6272, 512)
    s["sc.embedding.bias"] = (6272,)
    _conv(s, "sc.bias_conv", 128, 128, 3)
    fp = "feat_prop_module."
    for d in ("backward_1", "forward_1"):
        a = fp + "deform_align." + d
        s[a + ".weight"] = (128, 128, 3, 3)
        s[a + ".bias"] = (128,)
        _conv(s, a + ".conv_offset.0", 128, 261, 3)
        _conv(s, a + ".conv_offset.2", 128, 128, 3)
        _conv(s, a + ".conv_offset.4", 128, 128, 3)
        _conv(s, a + ".conv_offset.6", 432, 128, 3)
    for d in ("backward_1", "forward_1"):
        _conv(s, fp + f"backbone.{d}.0", 128, 258, 3)
        _conv(s, fp + f"backbone.{d}.2", 128, 128, 3)
    _conv(s, fp + "fuse.0", 128, 258, 3)
    _conv(s, fp + "fuse.2", 128, 128, 3)
    for b in range(N_TRANSFORMER_BLOCKS):
        t = f"transformers.transformer.{b}."
        s[t + "attention.valid_ind_rolled"] = (148,)
        for n in ("key", "query", "value", "proj"):
            s[t + f"attention.{n}.weight"] = (512, 512)
            s[t + f"attention.{n}.bias"] = (512,)
        s[t + "attention.pool_layer.weight"] = (512, 1, 4, 4)
        s[t + "attention.pool_layer.bias"] = (512,)
        for n in ("norm1", "norm2"):
            s[t + n + ".weight"] = (512,)
            s[t + n + ".bias"] = (512,)
        s[t + "mlp.fc1.0.weight"] = (FFN_HIDDEN, 512)
        s[t + "mlp.fc1.0.bias"] = (FFN_HIDDEN,)
        s[t + "mlp.fc2.1.weight"] = (512, FFN_HIDDEN)
        s[t + "mlp.fc2.1.bias"] = (512,)
    return s


def rolled_valid_indices(window=(5, 9)) -> np.ndarray:
    """The 148 ring positions kept from the four rolled copies of a 5x9 window.

    Restates the buffer built at reference model/modules/sparse_transformer.py:182-197:
    four 5x9 corner masks (tl, tr, bl, br) flattened and concatenated; indices of the ones.
    """
    wh, ww = window
    eh, ew = (wh + 1) // 2, (ww + 1) // 2
    masks = []
    for top, left in ((True, True), (True, False), (False, True), (False, False)):
        m = np.ones((wh, ww), dtype=np.int64)
        rs = slice(0, wh - eh) if top else slice(eh, wh)
        cs = slice(0, ww - ew) if left else slice(ew, ww)
        m[rs, cs] = 0
        masks.append(m.reshape(-1))
    return np.nonzero(np.concatenate(masks))[0].astype(np.int64)


# ----------------------------------------------------------------------------------------------
# synthetic checkpoints
# ----------------------------------------------------------------------------------------------


def _fan_in(shape):
    return int(np.prod(shape[1:])) if len(shape) > 1 else 1


def _fill(spec, seed, gain_of, bias_std=0.05):
    rng = np.random.RandomState(seed)
    out: OrderedDict = OrderedDict()
    for key, shape in spec.items():
        if key.endswith("num_batches_tracked"):
            out[key] = torch.tensor(100, dtype=torch.int64)
        elif key.endswith("valid_ind_rolled"):
            out[key] = torch.from_numpy(rolled_valid_indices())
        elif key.endswith("running_var"):
            out[key] = torch.from_numpy(rng.uniform(0.7, 1.3, shape).astype(np.float32))
        elif key.endswith("running_mean"):
            out[key] = torch.from_numpy((0.1 * rng.randn(*shape)).astype(np.float32))
        elif key.endswith(".bias"):
            out[key] = torch.from_numpy((bias_std * rng.randn(*shape)).astype(np.float32))
        else:
            g = gain_of(key, shape)
            if len(shape) == 1:  # norm scale
                out[key] = torch.from_numpy(rng.uniform(0.8, 1.2, shape).astype(np.float32))
            else:
                std = g / math.sqrt(_fan_in(shape))
                out[key] = torch.from_numpy((std * rng.randn(*shape)).astype(np.float32))
    return out


def synthetic_raft_state_dict(seed: int = 0, module_prefix: bool = True, flow_head_gain: float = 0.15):
    """Seeded RAFT checkpoint; keys carry ``module.`` like the released file when asked.

    ``flow_head_gain`` scales the last flow-head conv: 0.15 (default, the bench weights) keeps the per-iteration
    flow update small; 1.3 is the same Kaiming-like gain as every other layer ("un-damped", used by the
    raft_iter=20 parity case to measure fp16 error growth over the iterations)."""
    def gain(key, shape):
        if "flow_head.conv2" in key:
            return flow_head_gain
        if "mask.2" in key:
            return 2.0
        if "gru." in key:
            return 1.0
        return 1.3
    sd = _fill(raft_spec(), seed, gain)
    # norm3 and downsample.1 are the same module in the reference; keep the tensors identical
    for k in list(sd):
        if ".downsample.1." in k:
            sd[k] = sd[k.replace(".downsample.1.", ".norm3.")].clone()
    if module_prefix:
        sd = OrderedDict(("module." + k, v) for k, v in sd.items())
    return sd


def synthetic_rfc_state_dict(seed: int = 1):
    def gain(key, shape):
        if "backbone" in key and key.endswith(".2.weight"):
            return 0.25  # damp the recurrent residual branch (up to ~90 serial steps)
        if "conv_offset.6" in key:
            return 1.0
        if "deform_align" in key and "conv_offset" not in key:
            return 0.9
        if "upsample.2.conv" in key:
            return 2.0
        return 1.3
    return _fill(rfc_spec(), seed, gain)


def synthetic_generator_state_dict(seed: int = 2, attn_logit_gain: float = 1.0):
    """Seeded generator checkpoint.  ``attn_logit_gain`` scales the attention's query and key weights, so the logits by
    its square: at 1.0 (default, the bench weights) the attention over ~1,600 keys is nearly uniform; a larger gain makes
    it sharp, so that a key gathered from the wrong token moves the output by O(|v|)."""
    def gain(key, shape):
        if "attention.query.weight" in key or "attention.key.weight" in key:
            return attn_logit_gain
        if "backbone" in key and key.endswith(".2.weight"):
            return 0.3
        if "conv_offset.6" in key:
            return 1.0
        if "pool_layer.weight" in key:
            return 1.0
        if "mlp.fc2" in key or "attention.proj" in key:
            return 0.5
        if "sc.embedding" in key:
            return 0.6
        if "ss.embedding" in key:
            return 1.0
        if "transformers" in key:
            return 1.0
        return 1.3
    sd = _fill(generator_spec(), seed, gain)
    rng = np.random.RandomState(seed + 1000)
    for k in list(sd):
        if k.endswith("pool_layer.weight"):
            # learned depthwise pooling: mean filter plus a perturbation so it is not a plain mean
            w = np.full(sd[k].shape, 1.0 / 16.0, dtype=np.float32)
            w += (0.02 * rng.randn(*w.shape)).astype(np.float32)
            sd[k] = torch.from_numpy(w)
    return sd


def check_state_dict(sd, spec, strip_prefix: str = "") -> None:
    """Raise ``KeyError``/``ValueError`` unless ``sd`` matches ``spec`` exactly (strict load)."""
    keys = {(k[len(strip_prefix):] if strip_prefix and k.startswith(strip_prefix) else k): v
            for k, v in sd.items()}
    missing = [k for k in spec if k not in keys]
    extra = [k for k in keys if k not in spec]
    if missing or extra:
        raise KeyError(f"state_dict mismatch: missing={missing[:5]} unexpected={extra[:5]}")
    for k, shape in spec.items():
        if tuple(keys[k].shape) != tuple(shape):
            raise ValueError(f"{k}: expected {tuple(shape)}, got {tuple(keys[k].shape)}")
