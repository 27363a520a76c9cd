"""ctypes binding of libpropainter_b200.so + checkpoint packing for the sm_90a kernels.

PyTorch is used here only for device memory, streams and host-side weight re-layout; every compute
step goes through the C ABI declared in include/propainter_b200.h.  There is NO fallback path: if the
shared library is missing or the device is not an H100 (sm_90), construction fails loudly.
"""
from __future__ import annotations

import ctypes
import math
import os
from typing import Dict, Tuple

import torch

from . import weights as Wspec

_LIB = None
_PKG_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("PP_LIB_PATH") or os.path.join(_PKG_DIR, "libpropainter_b200.so")   # PP_LIB_PATH: A/B builds

MAX_BN = 256
ACT_NONE, ACT_RELU, ACT_LRELU, ACT_SIGMOID, ACT_TANH, ACT_GELU = range(6)

_VP, _I, _F, _LL, _SZ, _CP = (ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_longlong, ctypes.c_size_t,
                              ctypes.c_char_p)
# name -> (restype, argtypes); must list every symbol declared in include/propainter_b200.h
_SIGNATURES = {
    "pp_last_error": (_CP, []),
    "pp_version": (_CP, []),
    "pp_create": (_I, [_I, _VP, _SZ, ctypes.POINTER(_VP)]),
    "pp_destroy": (_I, [_VP]),
    "pp_set_workspace": (_I, [_VP, _VP, _SZ]),
    "pp_comm_unique_id": (_I, [_VP]),
    "pp_comm_init": (_I, [_VP, _VP, _I, _I]),
    "pp_comm_destroy": (_I, [_VP]),
    "pp_comm_all_gather_rows": (_I, [_VP, _VP, ctypes.POINTER(_LL), _SZ, _I, _I, _VP]),
    "pp_register_conv": (_I, [_VP, _CP, _VP, _VP, _I, _I, _I, _I, _I, _I, _I]),
    "pp_register_tensor": (_I, [_VP, _CP, _VP, _SZ]),
    "pp_set_conv_macs": (_I, [_VP, _CP, ctypes.c_double]),
    "pp_raft_bidir": (_I, [_VP, _VP, _I, _I, _I, _I, _VP, _VP, _VP]),
    "pp_raft_bidir_fp32": (_I, [_VP, _VP, _I, _I, _I, _I, _VP, _VP, _VP]),
    "pp_flow_complete": (_I, [_VP, _VP, _VP, _VP, _I, _I, _I, _VP, _VP, _VP]),
    "pp_flow_complete_dist": (_I, [_VP, _VP, _VP, _VP, _I, _I, _I, _VP, _VP, _I, _I, _VP]),
    "pp_flow_complete_fp32": (_I, [_VP, _VP, _VP, _VP, _I, _I, _I, _VP, _VP, _VP]),
    "pp_flow_complete_dist_fp32": (_I, [_VP, _VP, _VP, _VP, _I, _I, _I, _VP, _VP, _I, _I, _VP]),
    "pp_image_propagate": (_I, [_VP, _VP, _VP, _VP, _VP, _I, _I, _I, _VP, _VP, _VP]),
    "pp_image_propagate_fp32": (_I, [_VP, _VP, _VP, _VP, _VP, _I, _I, _I, _VP, _VP, _VP]),
    "pp_gen_begin": (_I, [_VP, _VP, _VP, _VP, _VP, _VP, _I, _I, _I, _VP]),
    "pp_gen_begin_subset": (_I, [_VP, _VP, _VP, _VP, _VP, _VP, _I, _I, _I, ctypes.c_char_p, _VP]),
    "pp_gen_window": (_I, [_VP, ctypes.POINTER(_I), _I, _I, _VP, _VP]),
    "pp_gen_run": (_I, [_VP, ctypes.POINTER(_I), ctypes.POINTER(_I), ctypes.POINTER(_I), _I, _VP, _VP]),
    "pp_gen_end": (_I, [_VP]),
    "pp_composite": (_I, [_VP, _VP, _VP, _VP, _VP, _VP, _VP, _I, _I, _I, _I, _VP]),
    "pp_preprocess": (_I, [_VP, _VP, _VP, _I, _I, _I, _I, _I, _I, _VP, _VP, _VP, _VP, _VP]),
    "pp_preprocess_resize": (_I, [_VP, _VP, _VP, _I, _I, _I, _I, _I, _I, _I, _I, _VP, _VP, _VP, _VP, _VP]),
    "pp_preprocess_u8": (_I, [_VP, _VP, _VP, _I, _I, _I, _I, _I, _I, _I, _I, _VP, _VP, _VP, _VP, _VP]),
    "pp_host_quantize_u8": (_I, [_VP, _VP, _LL, _I]),
    "pp_quantize_u8": (_I, [_VP, _VP, _VP, _LL, _VP]),
    "pp_preprocess_outpaint_u8": (_I, [_VP, _VP, _I, _I, _I, _I, _I, _I, _I, _VP, _VP, _VP, _VP, _VP]),
    "pp_postprocess": (_I, [_VP, _VP, _VP, _LL, _VP]),
    "pp_launch_count": (_LL, [_VP]),
    "pp_workspace_peak": (_SZ, [_VP]),
    "pp_profile_enable": (_I, [_VP, _I]),
    "pp_profile_dump": (_I, [_VP, ctypes.c_char_p, _SZ]),
    "pp_op_conv": (_I, [_VP, _CP, _VP, _I, _I, _I, _I, _I, _I, _I, _I, _F, _VP, _VP, _VP]),
    "pp_op_conv_ex": (_I, [_VP, _CP, _VP, _I, _I, _I, _I, _I, _I, _I, _I, _I, _F, _F, _I, _VP, _I, _I, _VP, _I, _I, _VP,
                           _I, _I, _VP]),
    "pp_op_conv_segs": (_I, [_VP, _CP, _I, ctypes.POINTER(_VP)] + [ctypes.POINTER(_I)] * 4 + [_I] * 12 + [_F, _F, _I, _VP,
                             _I, _I, _VP, _I, _I, _VP, _I, _I, _I, _I, _VP]),
    "pp_op_conv_last_plan": (_I, [ctypes.POINTER(_I), _I]),
    "pp_op_corr_lookup": (_I, [_VP, _VP, _VP, _VP, _VP, _VP, _VP, _LL, _I, _I, _VP]),
    "pp_op_conv_tf32": (_I, [_VP, _CP, _VP, _I, _I, _I, _VP, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I,
                             _F, _F, _I, _VP, _I, _I, _VP, _I, _I, _VP, _I, _I, _I, _VP]),
    "pp_op_dcn_sample_f32": (_I, [_VP, _VP, _I, _VP, _I, _VP, _I, _I, _I, _F, _VP, _VP]),
    "pp_op_upsample2x_f32": (_I, [_VP, _VP, _VP, _I, _I, _I, _I, _VP]),
    "pp_op_instnorm": (_I, [_VP, _VP, _VP, _VP, _I, _I, _I, _I, _I, _VP]),
    "pp_op_corr_pyramid": (_I, [_VP, _VP, _VP, _I, _I, _I, _I, _VP, _VP, _VP, _VP, _VP]),
    "pp_op_corr_lookup_f32": (_I, [_VP, _VP, _VP, _VP, _VP, _VP, _VP, _LL, _I, _I, _VP]),
    "pp_op_convex_upsample": (_I, [_VP, _VP, _VP, _VP, _I, _I, _I, _I, _VP]),
    "pp_op_imgprop_step": (_I, [_VP, _VP, _VP, _VP, _VP, _VP, _I, _I, _VP]),
    "pp_op_imgprop_step_f32": (_I, [_VP, _VP, _VP, _VP, _VP, _VP, _I, _I, _VP]),
    "pp_op_attention": (_I, [_VP, _VP, _VP, _VP, _VP, ctypes.POINTER(_I), _I, _I, _I, _I, _I, _VP]),
    "pp_op_layernorm": (_I, [_VP, _VP, _VP, _VP, _VP, _I, _I, _I, _I, _I, _VP]),
    "pp_op_pool_tokens": (_I, [_VP, _VP, _VP, _VP, _VP, _I, _I, _I, _I, _VP]),
    "pp_op_window_flags": (_I, [_VP, _VP, _I, _I, ctypes.POINTER(_I), ctypes.POINTER(_I), _I, _I, _I, _VP, _VP]),
    "pp_op_fold": (_I, [_VP, _VP, _I, _VP, _I, _I, _I, _I, _I, _I, _VP]),
    "pp_op_featprop_cond": (_I, [_VP, _VP, _VP, _VP, _VP, _VP, _VP, _I, _I, _I, _VP]),
    "pp_op_dcn_sample": (_I, [_VP, _VP, _I, _I, _VP, _I, _I, _VP, _VP, _I, _I, _F, _VP, _I, _I, _I, _VP]),
    "pp_op_downsample4": (_I, [_VP, _VP, _VP, _I, _VP, _VP, _I, _I, _I, _I, _VP]),
    "pp_op_upsample2x": (_I, [_VP, _VP, _VP, _I, _I, _I, _I, _VP]),
}


def load_library() -> ctypes.CDLL:
    """Load the CUDA library (built in-tree by ``__graft_entry__.build()`` / ``make -C csrc``)."""
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `make -C {os.path.join(_PKG_DIR, 'csrc')}` "
                "(there is no CPU or PyTorch fallback for the ProPainter hot path)")
        lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError if the symbol is not exported
            fn.restype = res
            fn.argtypes = args
        _LIB = lib
    return _LIB


def exported_symbols():
    return sorted(_SIGNATURES)


# ----------------------------------------------------------------------------------------------
# weight packing (host side)
# ----------------------------------------------------------------------------------------------


def choose_bn(cout: int) -> Tuple[int, int]:
    """N-tile of the wgmma GEMM: tiles of <= MAX_BN columns (multiple of 16) with the least padding.

    MAX_BN = 256: a 64 x 256 fp32 accumulator is 128 registers per consumer thread, and a wide
    N tile halves the im2col (A operand) traffic per output for the Cout >= 256 layers."""
    best = None
    t0 = (cout + MAX_BN - 1) // MAX_BN
    for n_tiles in (t0, t0 + 1):
        bn = ((cout + n_tiles - 1) // n_tiles + 15) // 16 * 16
        if bn > MAX_BN:
            continue
        cand = (bn * n_tiles, n_tiles, bn)
        if best is None or cand < best:
            best = cand
    return best[2], best[0]


def pack_conv_weight(w: torch.Tensor, groups: int = 1, cin_map=None):
    """[Cout, Cin_g, kh, kw] fp32 -> swizzled B-operand image + metadata.

    K is ordered (ky, kx, ci) with ci running over the *kernel's* input channels: ``cin_map[ci]`` is
    the reference input channel feeding kernel channel ci, or -1 for a zero (padding) channel.
    Layout: [groups][K_pad/64][cout_g_pad] rows of 64 fp16; inside each 128-byte row the 16-byte chunk
    c is stored at position c ^ (row & 7) (the 128B swizzle the wgmma descriptor expects)."""
    w = w.detach().float().cpu()
    cout, cin_ref, kh, kw = w.shape
    if cin_map is None:
        cin_map = list(range(cin_ref)) + [-1] * ((-cin_ref) % 8)
    assert len(cin_map) % 8 == 0
    cin_k = len(cin_map)
    idx = torch.tensor([max(i, 0) for i in cin_map], dtype=torch.long)
    keep = torch.tensor([1.0 if i >= 0 else 0.0 for i in cin_map])
    wk = w[:, idx] * keep.view(1, -1, 1, 1)                # [Cout, cin_k, kh, kw]
    wk = wk.permute(0, 2, 3, 1).reshape(cout, kh * kw * cin_k)   # K = (ky, kx, ci)
    cout_g = cout // groups
    bn, cout_g_pad = choose_bn(cout_g)
    K = wk.shape[1]
    K_pad = (K + 63) // 64 * 64
    buf = torch.zeros(groups, cout_g_pad, K_pad)
    buf[:, :cout_g, :K] = wk.view(groups, cout_g, K)
    num_kc = K_pad // 64
    buf = buf.view(groups, cout_g_pad, num_kc, 8, 8).permute(0, 2, 1, 3, 4).contiguous()  # [G, kc, row, chunk, 8]
    rows = torch.arange(cout_g_pad)
    pos = torch.arange(8).view(1, 8) ^ (rows.view(-1, 1) & 7)                               # position p holds chunk p^(r&7)
    buf = torch.gather(buf, 3, pos.view(1, 1, cout_g_pad, 8, 1).expand(groups, num_kc, cout_g_pad, 8, 8))
    meta = dict(cout_g=cout_g, cout_g_pad=cout_g_pad, bn=bn, cin_g=cin_k, kh=kh, kw=kw, groups=groups)
    return buf.to(torch.float16).contiguous(), meta


def split_tf32(x: torch.Tensor):
    """fp32 x -> (hi, lo): hi = x rounded to tf32 (10 explicit mantissa bits, nearest, ties away from zero, as
    cvt.rna.tf32.f32 does), lo = x - hi.  hi has its low 13 mantissa bits zero and hi + lo == x exactly."""
    x = x.detach().float().contiguous()
    hi = ((x.view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)
    return hi, x - hi


def pack_conv_weight_tf32(w, cin_map=None):
    """[Cout, Cin, kh, kw] fp32 -> split-tf32 B-operand image of the fp32 RAFT path + metadata.

    The kernel reads its inputs as the segments (hi, lo, hi) of split activation pairs (csrc/conv_igemm.cuh), so the K
    rows of one filter tap are [W_hi; W_hi; W_lo] over the kernel's input channels (``cin_map`` as in
    pack_conv_weight, padded to a multiple of 4 channels), and the GEMM sums hi*W_hi + lo*W_hi + hi*W_lo.  K is
    ordered (ky, kx, pass, ci).  Layout: [K_pad/32][cout_pad] rows of 32 fp32 (128 bytes, the same byte geometry as the
    fp16 image); inside a row the 16-byte unit u is stored at position u ^ (row & 7).  ``cin_g`` of the metadata counts
    the kernel's 2-byte units (two per fp32 value)."""
    w = w.detach().float().cpu()
    cout, cin_ref, kh, kw = w.shape
    if cin_map is None:
        cin_map = list(range(cin_ref)) + [-1] * ((-cin_ref) % 4)
    assert len(cin_map) % 4 == 0
    cin_k = len(cin_map)
    idx = torch.tensor([max(i, 0) for i in cin_map], dtype=torch.long)
    keep = torch.tensor([1.0 if i >= 0 else 0.0 for i in cin_map])
    hi, lo = split_tf32(w[:, idx] * keep.view(1, -1, 1, 1))               # [Cout, cin_k, kh, kw]
    wk = torch.cat([hi, hi, lo], 1).permute(0, 2, 3, 1).reshape(cout, kh * kw * 3 * cin_k)
    bn, cout_pad = choose_bn(cout)
    K = wk.shape[1]
    K_pad = (K + 31) // 32 * 32
    buf = torch.zeros(cout_pad, K_pad)
    buf[:cout, :K] = wk
    num_kc = K_pad // 32
    buf = buf.view(cout_pad, num_kc, 8, 4).permute(1, 0, 2, 3).contiguous()           # [kc, row, unit, 4]
    rows = torch.arange(cout_pad)
    pos = torch.arange(8).view(1, 8) ^ (rows.view(-1, 1) & 7)                          # position p holds unit p^(r&7)
    buf = torch.gather(buf, 2, pos.view(1, cout_pad, 8, 1).expand(num_kc, cout_pad, 8, 4))
    meta = dict(cout_g=cout, cout_g_pad=cout_pad, bn=bn, cin_g=2 * 3 * cin_k, kh=kh, kw=kw, groups=1)
    return buf.contiguous(), meta


def _fold_bn(w, b, sd, p, eps=1e-5):
    scale = sd[p + ".weight"] / torch.sqrt(sd[p + ".running_var"] + eps)
    return w * scale.view(-1, 1, 1, 1), (b - sd[p + ".running_mean"]) * scale + sd[p + ".bias"]


def _pad_map(n_real: int, total: int):
    return list(range(n_real)) + [-1] * (total - n_real)


def build_layers(raft_sd, rfc_sd, gen_sd):
    """-> (convs: name -> (weight[Cout,Cin,kh,kw], bias, groups, cin_map), tensors: name -> fp32 tensor)."""
    convs: Dict[str, tuple] = {}
    tens: Dict[str, torch.Tensor] = {}

    def add(name, w, b, groups=1, cin_map=None, macs=None):
        # macs: multiply-adds per output pixel of the reference layer (default: the weight tensor as given)
        convs[name] = (w.float(), None if b is None else b.float(), groups, cin_map,
                       float(w.shape[0] * w.shape[1] * w.shape[2] * w.shape[3]) if macs is None else float(macs))

    # ------------------------------------------------------------------ RAFT
    r = {(k[7:] if k.startswith("module.") else k): v.float() for k, v in raft_sd.items()}
    Wspec.check_state_dict(r, Wspec.raft_spec())
    for net, bn in (("fnet", False), ("cnet", True)):
        def cv(dst, src, norm=None, cin_map=None):
            w, b = r[f"{net}.{src}.weight"], r[f"{net}.{src}.bias"]
            if bn and norm is not None:
                w, b = _fold_bn(w, b, r, f"{net}.{norm}")
            add(f"raft.{net}.{dst}", w, b, 1, cin_map)
        cv("conv1", "conv1", "norm1", _pad_map(3, 8))
        for li in (1, 2, 3):
            for bi in (0, 1):
                q = f"layer{li}.{bi}."
                cv(q + "conv1", q + "conv1", q + "norm1")
                cv(q + "conv2", q + "conv2", q + "norm2")
                if li > 1 and bi == 0:
                    cv(q + "downsample", q + "downsample.0", q + "norm3")
        cv("conv2", "conv2")
    u = "update_block."
    add("raft.update.convc1", r[u + "encoder.convc1.weight"], r[u + "encoder.convc1.bias"], 1, _pad_map(324, 328))
    add("raft.update.convc2", r[u + "encoder.convc2.weight"], r[u + "encoder.convc2.bias"])
    # convf1 (7x7 over the 2-channel flow) as a linear layer over explicit 7x7x2 patches in (ky, kx, channel) order,
    # zero-padded 98 -> 128 (kernels_raft.cu: flow_patch7x7)
    wf1 = r[u + "encoder.convf1.weight"]                                   # [128, 2, 7, 7]
    wf1 = torch.cat([wf1.permute(0, 2, 3, 1).reshape(128, 98), torch.zeros(128, 30)], 1).view(128, 128, 1, 1)
    add("raft.update.convf1", wf1, r[u + "encoder.convf1.bias"], 1, None, macs=128 * 98)
    add("raft.update.convf2", r[u + "encoder.convf2.weight"], r[u + "encoder.convf2.bias"])
    add("raft.update.conv", r[u + "encoder.conv.weight"], r[u + "encoder.conv.bias"])
    for s in ("1", "2"):
        add("raft.update.gru.zr" + s, torch.cat([r[u + f"gru.convz{s}.weight"], r[u + f"gru.convr{s}.weight"]], 0),
            torch.cat([r[u + f"gru.convz{s}.bias"], r[u + f"gru.convr{s}.bias"]], 0))
        add("raft.update.gru.q" + s, r[u + f"gru.convq{s}.weight"], r[u + f"gru.convq{s}.bias"])
    add("raft.update.fh1", r[u + "flow_head.conv1.weight"], r[u + "flow_head.conv1.bias"])
    add("raft.update.fh2", r[u + "flow_head.conv2.weight"], r[u + "flow_head.conv2.bias"])
    add("raft.update.mask0", r[u + "mask.0.weight"], r[u + "mask.0.bias"])
    add("raft.update.mask2", r[u + "mask.2.weight"], r[u + "mask.2.bias"])

    # ------------------------------------------------------------------ flow completion
    f = {k: v.float() for k, v in rfc_sd.items()}
    Wspec.check_state_dict(f, Wspec.rfc_spec())
    add("rfc.downsample", f["downsample.0.weight"][:, :, 0], f["downsample.0.bias"], 1, _pad_map(3, 8))
    for enc in ("encoder1", "encoder2"):
        for i in (0, 2):
            add(f"rfc.{enc}.{i}.conv1", f[f"{enc}.{i}.conv1.0.weight"][:, :, 0], f[f"{enc}.{i}.conv1.0.bias"])
            add(f"rfc.{enc}.{i}.conv2", f[f"{enc}.{i}.conv2.0.weight"][:, :, :, :, 0], f[f"{enc}.{i}.conv2.0.bias"])
    for j, i in enumerate((0, 2, 4)):
        add(f"rfc.mid.{j}", f[f"mid_dilation.{i}.weight"][:, :, 0], f[f"mid_dilation.{i}.bias"])

    def add_align(dst, sd, src):
        for j, i in enumerate((0, 2, 4, 6)):
            w = sd[f"{src}.conv_offset.{i}.weight"]
            cm = None if w.shape[1] % 8 == 0 else _pad_map(w.shape[1], (w.shape[1] + 7) // 8 * 8)
            add(f"{dst}.offset.{j}", w, sd[f"{src}.conv_offset.{i}.bias"], 1, cm)
        w = sd[src + ".weight"]                                        # [Cout, Cin, 3, 3] -> K = (tap, ci)
        add(f"{dst}.dcn", w.permute(0, 2, 3, 1).reshape(w.shape[0], -1, 1, 1), sd[src + ".bias"])

    fp = "feat_prop_module."
    for d in ("backward_", "forward_"):
        add_align(f"rfc.fp.{d}", f, fp + "deform_align." + d)
        add(f"rfc.fp.{d}.backbone.0", f[fp + f"backbone.{d}.0.weight"], f[fp + f"backbone.{d}.0.bias"])
        add(f"rfc.fp.{d}.backbone.1", f[fp + f"backbone.{d}.2.weight"], f[fp + f"backbone.{d}.2.bias"])
    add("rfc.fp.fusion", f[fp + "fusion.weight"], f[fp + "fusion.bias"])
    for dst, src in (("decoder2.0", "decoder2.0"), ("decoder2.deconv", "decoder2.2.conv"), ("decoder1.0", "decoder1.0"),
                     ("decoder1.deconv", "decoder1.2.conv"), ("upsample.0", "upsample.0"),
                     ("upsample.deconv", "upsample.2.conv")):
        add("rfc." + dst, f[src + ".weight"], f[src + ".bias"])

    # ------------------------------------------------------------------ generator
    g = {k: v.float() if v.is_floating_point() else v for k, v in gen_sd.items()}
    Wspec.check_state_dict(g, Wspec.generator_spec())
    enc_groups = {0: 1, 2: 1, 4: 1, 6: 1, 8: 1, 10: 2, 12: 4, 14: 8, 16: 1}
    for i, gr in enc_groups.items():
        w = g[f"encoder.layers.{i}.weight"]
        if i == 14:
            # groups of 80 input / 32 output channels are too small for 64-wide K chunks and 128-column tiles: run the
            # layer dense with block-diagonal weights (8x the MACs, all of them on the TMA halo-tile kernel at >10x the
            # rate).  Kernel channel order = cat(x0[256], previous output[384]); group k owns x0[32k:32k+32] and
            # prev[48k:48k+48] (propainter.py:268-273).
            cout, cg = w.shape[0], w.shape[1]
            nx, npv = 256 // gr, 384 // gr
            assert cg == nx + npv and cout % gr == 0
            dense = torch.zeros(cout, 640, w.shape[2], w.shape[3])
            for k in range(gr):
                rows = slice(k * (cout // gr), (k + 1) * (cout // gr))
                dense[rows, k * nx:(k + 1) * nx] = w[rows, :nx]
                dense[rows, 256 + k * npv:256 + (k + 1) * npv] = w[rows, nx:]
            add("gen.encoder.14", dense, g["encoder.layers.14.bias"], 1, None, macs=w.numel())
            continue
        add(f"gen.encoder.{i}", w, g[f"encoder.layers.{i}.bias"], gr, _pad_map(5, 8) if i == 0 else None)
    for dst, src in (("0", "0.conv"), ("2", "2"), ("4", "4.conv"), ("6", "6")):
        add("gen.decoder." + dst, g[f"decoder.{src}.weight"], g[f"decoder.{src}.bias"])
    add("gen.ss", g["ss.embedding.weight"].view(512, 128, 7, 7), g["ss.embedding.bias"])
    # SoftComp Linear: output column c*49+k -> k*128+c, so the fold kernel reads contiguous channels
    perm = (torch.arange(49).view(49, 1) + 49 * torch.arange(128).view(1, 128)).reshape(-1)
    add("gen.sc.embedding", g["sc.embedding.weight"][perm].view(6272, 512, 1, 1), g["sc.embedding.bias"][perm])
    add("gen.sc.bias_conv", g["sc.bias_conv.weight"], g["sc.bias_conv.bias"])
    for d in ("backward_1", "forward_1"):
        add_align(f"gen.fp.{d}", g, fp + "deform_align." + d)
        add(f"gen.fp.{d}.backbone.0", g[fp + f"backbone.{d}.0.weight"], g[fp + f"backbone.{d}.0.bias"], 1,
            _pad_map(258, 264))
        add(f"gen.fp.{d}.backbone.1", g[fp + f"backbone.{d}.2.weight"], g[fp + f"backbone.{d}.2.bias"])
    add("gen.fp.fuse.0", g[fp + "fuse.0.weight"], g[fp + "fuse.0.bias"], 1, _pad_map(258, 264))
    add("gen.fp.fuse.1", g[fp + "fuse.2.weight"], g[fp + "fuse.2.bias"])
    perm40 = (torch.arange(49).view(49, 1) + 49 * torch.arange(40).view(1, 40)).reshape(-1)
    for b in range(Wspec.N_TRANSFORMER_BLOCKS):
        t = f"transformers.transformer.{b}."
        a = t + "attention."
        o = f"gen.tf.{b}."
        qkv_w = torch.cat([g[a + "query.weight"], g[a + "key.weight"], g[a + "value.weight"]], 0)
        qkv_b = torch.cat([g[a + "query.bias"], g[a + "key.bias"], g[a + "value.bias"]], 0)
        add(o + "qkv", qkv_w.view(1536, 512, 1, 1), qkv_b)
        add(o + "kv", qkv_w[512:].reshape(1024, 512, 1, 1), qkv_b[512:])
        add(o + "proj", g[a + "proj.weight"].view(512, 512, 1, 1), g[a + "proj.bias"])
        add(o + "fc1", g[t + "mlp.fc1.0.weight"][perm40].view(1960, 512, 1, 1), g[t + "mlp.fc1.0.bias"][perm40])
        add(o + "fc2", g[t + "mlp.fc2.1.weight"].view(512, 40, 7, 7), g[t + "mlp.fc2.1.bias"])
        for n in ("norm1", "norm2"):
            tens[o + n + ".weight"] = g[t + n + ".weight"].float()
            tens[o + n + ".bias"] = g[t + n + ".bias"].float()
        tens[o + "pool.weight"] = g[a + "pool_layer.weight"].reshape(512, 16).float().t().contiguous()   # [tap][C]
        tens[o + "pool.bias"] = g[a + "pool_layer.bias"].float()
        expect = torch.from_numpy(Wspec.rolled_valid_indices())
        if not torch.equal(g[a + "valid_ind_rolled"].cpu().long(), expect):
            raise ValueError("checkpoint's valid_ind_rolled differs from the 5x9 window ring this engine implements")
    return convs, tens


# ----------------------------------------------------------------------------------------------
# engine
# ----------------------------------------------------------------------------------------------


def _ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


class Engine:
    """One engine per process/GPU.  Owns the workspace arena and the packed weights."""

    MIN_WORKSPACE = 256 << 20

    def __init__(self, device: torch.device | str | int = "cuda:0", workspace_gb: float | None = None):
        """``workspace_gb``: fixed size of the scratch arena; None = start at 256 MiB and let ``reserve_for_clip``
        size it from (T, H, W) before each clip (what the node path does)."""
        self.lib = load_library()
        self.device = torch.device(device)
        if self.device.type != "cuda" or not torch.cuda.is_available():
            raise RuntimeError("the ProPainter CUDA engine needs a CUDA device (no CPU fallback)")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self._keep = []
        self._total_mem = torch.cuda.get_device_properties(self.device).total_memory
        self.fixed_workspace = workspace_gb is not None
        nbytes = self.MIN_WORKSPACE if workspace_gb is None else int(min(workspace_gb * (1 << 30), self._total_mem * 0.8))
        self.workspace = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        h = ctypes.c_void_p()
        self._check(self.lib.pp_create(self.device.index, _ptr(self.workspace), nbytes, ctypes.byref(h)))
        self.h = h
        self.conv_meta: Dict[str, dict] = {}

    # -- workspace sizing
    @staticmethod
    def clip_workspace_bytes(T: int, H: int, W: int) -> int:
        """Arena size that lets every stage of a T x H x W clip run in its widest batching (~1.4 kB per frame-pixel;
        clips beyond ~100 frames are processed in sub-batches of windows / chunks of sub-videos, so the estimate
        saturates there).  reserve_for_clip caps it at 80 % of the device memory; above the cap the stages run smaller
        batches."""
        return int(1400 * min(T, 100) * H * W + (2 << 30))

    def set_workspace_bytes(self, nbytes: int) -> None:
        """Re-allocate the arena (no generator session may be open)."""
        nbytes = max(int(nbytes), self.MIN_WORKSPACE)
        torch.cuda.current_stream(self.device).synchronize()
        self.workspace = None                       # release before allocating: never hold old + new together
        torch.cuda.empty_cache()
        ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        self._check(self.lib.pp_set_workspace(self.h, _ptr(ws), nbytes))
        self.workspace = ws

    def reserve_for_clip(self, T: int, H: int, W: int) -> int:
        """Grow the arena for a clip when it was created without a fixed size.  Capped at 80 % of the device memory;
        when the cap (or a fixed size) is below the estimate the stages fall back to smaller batches
        (RAFT pair batches, encoder / decoder frame chunks, sub-batches of sliding windows)."""
        if self.fixed_workspace:
            return self.workspace.numel()
        free, _ = torch.cuda.mem_get_info(self.device)
        have = self.workspace.numel()
        want = min(self.clip_workspace_bytes(T, H, W), int(self._total_mem * 0.8), int((free + have) * 0.9))
        if want > have:
            self.set_workspace_bytes(want)
        return self.workspace.numel()

    def release_workspace(self) -> None:
        """Shrink the arena back to its minimum (gives the HBM back between node executions when asked to)."""
        if not self.fixed_workspace and self.workspace.numel() > self.MIN_WORKSPACE:
            self.set_workspace_bytes(self.MIN_WORKSPACE)

    # -- helpers
    def _check(self, rc: int):
        if rc != 0:
            raise RuntimeError("propainter_b200: " + self.lib.pp_last_error().decode())

    def _stream(self):
        return ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def close(self):
        if getattr(self, "h", None):
            self.lib.pp_destroy(self.h)
            self.h = None
        self.workspace = None
        self._keep = []

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- weights
    def _register_packed(self, name, packed, meta, w, b, macs):
        packed = packed.to(self.device)
        bias = None if b is None else b.detach().float().contiguous().to(self.device)
        self._keep += [packed, bias]
        self.conv_meta[name] = meta
        self._check(self.lib.pp_register_conv(self.h, name.encode(), _ptr(packed), _ptr(bias), meta["cout_g"],
                                              meta["cout_g_pad"], meta["bn"], meta["cin_g"], meta["kh"], meta["kw"],
                                              meta["groups"]))
        self._check(self.lib.pp_set_conv_macs(self.h, name.encode(), float(w.numel() if macs is None else macs)))

    def register_conv(self, name, w, b, groups=1, cin_map=None, macs=None):
        self._register_packed(name, *pack_conv_weight(w, groups, cin_map), w, b, macs)

    def register_conv_tf32(self, name, w, b, cin_map=None, macs=None):
        """Split-tf32 image of a layer (pack_conv_weight_tf32), registered as ``name + ".tf32"``."""
        self._register_packed(name + ".tf32", *pack_conv_weight_tf32(w, cin_map), w, b, macs)

    def register_tensor(self, name, t):
        t = t.detach().float().contiguous().to(self.device)
        self._keep.append(t)
        self._check(self.lib.pp_register_tensor(self.h, name.encode(), _ptr(t), t.numel() * 4))

    # Stride-1 k>1 layers whose input channels are not a multiple of 64: kernel channels zero-padded to the next
    # multiple so they run on the TMA halo-tile kernel (64-channel K chunks); the activation tensors keep their real
    # channel count, TMA zero-fills the rest of the last segment (PPConvSeg.cvalid)
    PAD64_CONVS = ("rfc.encoder1.0.conv1", "rfc.encoder1.0.conv2", "rfc.upsample.0", "rfc.upsample.deconv") + tuple(
        f"raft.{net}.layer2.{blk}" for net in ("fnet", "cnet") for blk in ("0.conv2", "1.conv1", "1.conv2")) + (  # 96 ch
        # cat(features[256], mask/flow[8]) = 264 kernel channels -> 320: the 8-channel tail segment fills one chunk
        "gen.fp.backward_1.offset.0", "gen.fp.forward_1.offset.0", "gen.fp.backward_1.backbone.0",
        "gen.fp.forward_1.backbone.0", "gen.fp.fuse.0")

    # fp32 RAFT and flow-completion paths: kernel input channels of the split images whose reference channels are not a multiple of 32
    # (the frames: 3 -> 4, one 16-byte vector; the correlation lookup: 324 -> 352, whole 32-channel K chunks per pass)
    TF32_CIN_MAPS = {"raft.fnet.conv1": (3, 4), "raft.cnet.conv1": (3, 4), "raft.update.convc1": (324, 352),
                     "rfc.downsample": (3, 4)}

    def load_weights(self, raft_sd, rfc_sd, gen_sd):
        convs, tens = build_layers(raft_sd, rfc_sd, gen_sd)
        for name, (w, b, groups, cin_map, macs) in convs.items():
            if name.startswith(("raft.", "rfc.")):
                tm = self.TF32_CIN_MAPS.get(name)
                self.register_conv_tf32(name, w, b, None if tm is None else _pad_map(*tm), macs)
            if name in self.PAD64_CONVS:
                cin_map = list(cin_map) if cin_map is not None else list(range(w.shape[1]))
                cin_map += [-1] * ((-len(cin_map)) % 64)
            self.register_conv(name, w, b, groups, cin_map, macs)
        for name, t in tens.items():
            self.register_tensor(name, t)
        return self

    # -- stages (float32 contiguous CUDA tensors in the reference's layouts)
    def _f32(self, t):
        return t.to(device=self.device, dtype=torch.float32).contiguous()

    def raft_bidir(self, frames: torch.Tensor, iters: int, out=None, fp32: bool = False):
        """frames [T,3,H,W] in [-1,1] -> (flows_f, flows_b) [T-1,2,H,W] (written into `out` when given: contiguous
        float32 views, e.g. a rank's shard of the full flow buffers).  fp32=False: fp16 activations with fp32
        accumulation; fp32=True: fp32 activations and 3xTF32 GEMMs (pp_raft_bidir_fp32), what the node runs for
        fp16="disable"."""
        frames = self._f32(frames)
        T, _, H, W = frames.shape
        if out is not None:
            ff, fb = out
            assert ff.is_contiguous() and fb.is_contiguous() and ff.dtype == torch.float32 and ff.shape == (T - 1, 2, H, W)
        else:
            ff = torch.empty(T - 1, 2, H, W, device=self.device, dtype=torch.float32)
            fb = torch.empty_like(ff)
        fn = self.lib.pp_raft_bidir_fp32 if fp32 else self.lib.pp_raft_bidir
        self._check(fn(self.h, _ptr(frames), T, H, W, int(iters), _ptr(ff), _ptr(fb), self._stream()))
        return ff, fb

    def flow_complete(self, flows_f, flows_b, flow_masks, fp32: bool = False):
        """flows [T-1,2,H,W], flow_masks [T,1,H,W] -> completed (flows_f, flows_b).  fp32=False: fp16 activations;
        fp32=True: fp32 activations and 3xTF32 convolutions (pp_flow_complete_fp32), what the node runs for
        fp16="disable"."""
        flows_f, flows_b, flow_masks = self._f32(flows_f), self._f32(flows_b), self._f32(flow_masks)
        T, _, H, W = flow_masks.shape
        assert flows_f.shape[0] == T - 1
        of, ob = torch.empty_like(flows_f), torch.empty_like(flows_b)
        fn = self.lib.pp_flow_complete_fp32 if fp32 else self.lib.pp_flow_complete
        self._check(fn(self.h, _ptr(flows_f), _ptr(flows_b), _ptr(flow_masks), T, H, W, _ptr(of), _ptr(ob),
                       self._stream()))
        return of, ob

    def flow_complete_dist(self, flows_f, flows_b, flow_masks, team_first: int, team_size: int, out=None,
                           fp32: bool = False):
        """Collective flow completion of one chunk by the ranks [team_first, team_first + team_size) (see
        pp_flow_complete_dist); every team member gets the full completed flows.  fp32 as in flow_complete."""
        flows_f, flows_b, flow_masks = self._f32(flows_f), self._f32(flows_b), self._f32(flow_masks)
        T, _, H, W = flow_masks.shape
        assert flows_f.shape[0] == T - 1
        of, ob = out if out is not None else (torch.empty_like(flows_f), torch.empty_like(flows_b))
        assert of.is_contiguous() and ob.is_contiguous() and of.dtype == torch.float32
        fn = self.lib.pp_flow_complete_dist_fp32 if fp32 else self.lib.pp_flow_complete_dist
        self._check(fn(self.h, _ptr(flows_f), _ptr(flows_b), _ptr(flow_masks), T, H, W, _ptr(of), _ptr(ob),
                       int(team_first), int(team_size), self._stream()))
        return of, ob

    def image_propagate(self, frames, masks, flows_f, flows_b, fp32: bool = False):
        """frames [T,3,H,W], masks [T,1,H,W], completed flows [T-1,2,H,W] -> (updated frames, updated masks).
        fp32=False stores frames and flows in fp16 inside the propagation; fp32=True keeps them in fp32
        (pp_image_propagate_fp32), what the node runs for fp16="disable"."""
        frames, masks, flows_f, flows_b = map(self._f32, (frames, masks, flows_f, flows_b))
        T, _, H, W = frames.shape
        uf, um = torch.empty_like(frames), torch.empty_like(masks)
        fn = self.lib.pp_image_propagate_fp32 if fp32 else self.lib.pp_image_propagate
        self._check(fn(self.h, _ptr(frames), _ptr(masks), _ptr(flows_f), _ptr(flows_b), T, H, W, _ptr(uf), _ptr(um),
                       self._stream()))
        return uf, um

    def gen_begin(self, updated_frames, masks_dilated, updated_masks, flows_f, flows_b, frames_needed=None):
        """Open a generator session over the clip.  ``frames_needed``: frame ids to encode (default all); the windows
        given to gen_run must only touch those."""
        a = [self._f32(x) for x in (updated_frames, masks_dilated, updated_masks, flows_f, flows_b)]
        T, _, H, W = a[0].shape
        self._gen_shape = (T, H, W)
        self._gen_inputs = a  # keep alive for the session
        self._gen_needed = None if frames_needed is None else set(int(i) for i in frames_needed)
        if frames_needed is None:
            self._check(self.lib.pp_gen_begin(self.h, *[_ptr(x) for x in a], T, H, W, self._stream()))
        else:
            need = bytes(1 if i in self._gen_needed else 0 for i in range(T))
            self._check(self.lib.pp_gen_begin_subset(self.h, *[_ptr(x) for x in a], T, H, W, need, self._stream()))

    def gen_window(self, frame_ids, l_t: int) -> torch.Tensor:
        """-> fp16 [l_t,H,W,4] (rgb in [-1,1], lane 3 unused)."""
        T, H, W = self._gen_shape
        ids = (ctypes.c_int * len(frame_ids))(*[int(i) for i in frame_ids])
        pred = torch.empty(l_t, H, W, 4, device=self.device, dtype=torch.float16)
        self._check(self.lib.pp_gen_window(self.h, ids, len(frame_ids), int(l_t), _ptr(pred), self._stream()))
        return pred

    @staticmethod
    def gen_slot_bytes(H: int, W: int) -> int:
        """Workspace one (window, frame) slot of pp_gen_run needs (generator.cu): window-major features and the token /
        qkv / FFN rows of the transformer (all slots alive together), plus an upper bound of the feature-propagation
        buffers (4 feature-sized tensors per LOCAL slot of the largest equal-length group, and the per-step condition /
        offset / sampled-column tensors, one set per window ~ 1/8 of a slot)."""
        p4 = (H // 4) * (W // 4)
        gh, gw = (H // 4 + 6 - 7) // 3 + 1, (W // 4 + 6 - 7) // 3 + 1
        rows_pad = -(-gh // 5) * 5 * (-(-gw // 9) * 9)
        xfmr = p4 * (256 + 80) + gh * gw * 2 * (512 * 3 + 1960) + rows_pad * 2 * (512 + 1536)
        featprop = p4 * 2 * (128 * 4) + p4 * 2 * (264 + 432 + 1152 + 128 * 3) // 8
        return int(1.25 * (xfmr + featprop))

    def gen_batches(self, windows, budget_bytes: int, shape=None):
        """Split the schedule into consecutive sub-batches whose slots fit `budget_bytes` (windows are independent;
        the composite order is the window order, which consecutive sub-batches keep)."""
        T, H, W = shape if shape is not None else self._gen_shape
        per_slot = self.gen_slot_bytes(H, W)
        out, cur, used = [], [], 0
        for w in windows:
            need = (len(w[0]) + len(w[1])) * per_slot
            if cur and used + need > budget_bytes:
                out.append(cur)
                cur, used = [], 0
            cur.append(w)
            used += need
        if cur:
            out.append(cur)
        return out

    def gen_run(self, windows) -> torch.Tensor:
        """Sliding windows in batched passes.  windows = [(neighbor_ids, ref_ids), ...]
        -> fp16 [sum(len(neighbor_ids)), H, W, 4] in window order.

        One engine pass covers as many windows as the workspace holds (all 16 of an 80-frame 640x360 clip); a long
        or large clip is split into consecutive sub-batches, down to one window per pass, before giving up --
        the reference runs one window at a time, so anything it can process this can too."""
        T, H, W = self._gen_shape
        enc_bytes = T * (H // 4) * (W // 4) * (256 + 32) + (64 << 20)          # the session's resident part
        decoder_reserve = 24 * H * W * 2 * 200                                   # room for a useful decoder chunk
        budget = max(self.workspace.numel() - enc_bytes - decoder_reserve, self.gen_slot_bytes(H, W))
        out = [self._gen_run_or_split(b) for b in self.gen_batches(list(windows), budget)]
        return out[0] if len(out) == 1 else torch.cat(out, 0)

    def _gen_run_or_split(self, windows) -> torch.Tensor:
        try:
            return self._gen_run_once(windows)
        except RuntimeError as ex:
            if "workspace" not in str(ex) or len(windows) == 1:
                raise
        half = len(windows) // 2                     # the estimate was too optimistic: halve and retry
        return torch.cat([self._gen_run_or_split(windows[:half]), self._gen_run_or_split(windows[half:])], 0)

    gen_run_calls = 0       # engine passes issued by gen_run (1 per clip unless the workspace forced sub-batches)

    def _gen_run_once(self, windows) -> torch.Tensor:
        self.gen_run_calls += 1
        T, H, W = self._gen_shape
        flat, wt, wl = [], [], []
        if getattr(self, "_gen_needed", None) is not None:
            missing = {int(i) for nb, refs in windows for i in list(nb) + list(refs)} - self._gen_needed
            if missing:
                raise ValueError(f"gen_run: frames {sorted(missing)} were not encoded by gen_begin(frames_needed=...)")
        for nb, refs in windows:
            flat += [int(i) for i in nb] + [int(i) for i in refs]
            wt.append(len(nb) + len(refs))
            wl.append(len(nb))
        arr = lambda v: (ctypes.c_int * len(v))(*v)
        pred = torch.empty(sum(wl), H, W, 4, device=self.device, dtype=torch.float16)
        self._check(self.lib.pp_gen_run(self.h, arr(flat), arr(wt), arr(wl), len(windows), _ptr(pred), self._stream()))
        return pred

    def gen_end(self):
        self._check(self.lib.pp_gen_end(self.h))
        self._gen_inputs = None

    def composite(self, pred, masks_dilated, orig_u8, comp_u8, frame_ids_dev, first_visit_dev, half_math=False):
        """half_math: reproduce the half-precision roundings of the reference's fp16="enable" mode before the uint8
        truncation (reference propainter_inference.py:285-286 on a half tensor)."""
        l_t, H, W, _ = pred.shape
        self._check(self.lib.pp_composite(self.h, _ptr(pred), _ptr(masks_dilated), _ptr(orig_u8), _ptr(comp_u8),
                                          _ptr(frame_ids_dev), _ptr(first_visit_dev), l_t, H, W, int(bool(half_math)),
                                          self._stream()))

    def preprocess(self, image, mask, flow_mask_dilates: int, mask_dilates: int, process_size=None):
        """Device version of convert_image_to_frames + prepare_frames_and_masks (reference utils/image_utils.py:98-197).
        image [T,H,W,3] float 0..1, mask [T or 1,H,W] float32 (host or device); ``process_size`` = (width, height) to
        resize to (PIL's 8-bit bicubic resampler, reproduced bit for bit on the device), default: the input size.
        -> frames [1,T,3,h,w], flow_masks [1,T,1,h,w], masks_dilated [1,T,1,h,w] (float32), originals uint8 [T,h,w,3]."""
        T, H, W, _ = image.shape
        ow, oh = (W, H) if process_size is None else (int(process_size[0]), int(process_size[1]))
        if image.device.type == "cpu" and mask.device.type == "cpu" and image.dtype == torch.float32 and mask.dtype == torch.float32:
            # host tensors (what ComfyUI hands a node): the float -> uint8 truncation is the first thing the reference does
            # with them, so do it on the host cores straight into page-locked staging buffers and move 1/4 of the bytes
            return self._preprocess_host(image.contiguous(), mask.contiguous(), flow_mask_dilates, mask_dilates, ow, oh)
        img = image.to(self.device, torch.float32, non_blocking=True).contiguous()
        msk = mask.to(self.device, torch.float32, non_blocking=True).contiguous()
        orig = torch.empty(T, oh, ow, 3, device=self.device, dtype=torch.uint8)
        frames = torch.empty(T, 3, oh, ow, device=self.device, dtype=torch.float32)
        fm = torch.empty(T, 1, oh, ow, device=self.device, dtype=torch.float32)
        md = torch.empty_like(fm)
        if (ow, oh) == (W, H):
            self._check(self.lib.pp_preprocess(self.h, _ptr(img), _ptr(msk), msk.shape[0], T, H, W, int(flow_mask_dilates),
                                               int(mask_dilates), _ptr(orig), _ptr(frames), _ptr(fm), _ptr(md),
                                               self._stream()))
        else:
            self._check(self.lib.pp_preprocess_resize(self.h, _ptr(img), _ptr(msk), msk.shape[0], T, H, W, oh, ow,
                                                      int(flow_mask_dilates), int(mask_dilates), _ptr(orig), _ptr(frames),
                                                      _ptr(fm), _ptr(md), self._stream()))
        return frames.unsqueeze(0), fm.unsqueeze(0), md.unsqueeze(0), orig

    def _preprocess_host(self, image, mask, flow_mask_dilates, mask_dilates, ow, oh):
        T, H, W, _ = image.shape
        (img8d, img8), (msk8d, msk8) = self._upload_u8(image), self._upload_u8(mask)
        orig = torch.empty(T, oh, ow, 3, device=self.device, dtype=torch.uint8)
        frames = torch.empty(T, 3, oh, ow, device=self.device, dtype=torch.float32)
        fm = torch.empty(T, 1, oh, ow, device=self.device, dtype=torch.float32)
        md = torch.empty_like(fm)
        self._check(self.lib.pp_preprocess_u8(self.h, _ptr(img8d), _ptr(msk8d), mask.shape[0], T, H, W, oh, ow,
                                              int(flow_mask_dilates), int(mask_dilates), _ptr(orig), _ptr(frames), _ptr(fm),
                                              _ptr(md), self._stream()))
        self._keep_staging = (img8, msk8)      # the async copies read them; released at the next call
        return frames.unsqueeze(0), fm.unsqueeze(0), md.unsqueeze(0), orig

    def _upload_u8(self, x):
        """Contiguous float32 host tensor -> (uint8 device tensor, host staging): the reference's truncation on the host
        cores (pp_host_quantize_u8) straight into page-locked staging, then an asynchronous copy of 1/4 of the bytes.  The
        caller keeps the staging tensor alive until the copy has run."""
        threads = min(os.cpu_count() or 1, int(os.environ.get("PP_HOST_THREADS", 16)))
        try:
            x8 = torch.empty(x.shape, dtype=torch.uint8, pin_memory=True)
        except RuntimeError:        # locked-memory limit: pageable staging still moves 1/4 of the bytes
            x8 = torch.empty(x.shape, dtype=torch.uint8)
        self._check(self.lib.pp_host_quantize_u8(_ptr(x), _ptr(x8), x.numel(), threads))
        return x8.to(self.device, non_blocking=True), x8

    def preprocess_outpaint(self, image, icfg):
        """Device version of convert_image_to_frames + extrapolation + prepare_frames_and_masks_for_outpaint (reference
        utils/image_utils.py:98-116, 178-252), bit for bit: the frames, resized to ``icfg.process_size`` when that is not
        their size (PIL's 8-bit bicubic resampler), centred on a zero canvas of ``icfg.outpaint_size`` with the band
        masks around them.  image [T,H,W,3] float 0..1 (host or device).
        -> frames [1,T,3,ph,pw], flow_masks [1,T,1,ph,pw], masks_dilated [1,T,1,ph,pw] (float32), originals uint8
        [T,ph,pw,3], all on the device."""
        T, H, W, _ = image.shape
        rw, rh = (int(v) for v in icfg.process_size)
        pw, ph = (int(v) for v in icfg.outpaint_size)
        if image.device.type == "cpu" and image.dtype == torch.float32:
            img8d, staging = self._upload_u8(image.contiguous())        # as in preprocess: 1/4 of the bytes over PCIe
        else:
            img = image.to(self.device, torch.float32, non_blocking=True).contiguous()
            img8d, staging = torch.empty(img.shape, device=self.device, dtype=torch.uint8), None
            self._check(self.lib.pp_quantize_u8(self.h, _ptr(img), _ptr(img8d), img.numel(), self._stream()))
        orig = torch.empty(T, ph, pw, 3, device=self.device, dtype=torch.uint8)
        frames = torch.empty(T, 3, ph, pw, device=self.device, dtype=torch.float32)
        fm = torch.empty(T, 1, ph, pw, device=self.device, dtype=torch.float32)
        md = torch.empty_like(fm)
        self._check(self.lib.pp_preprocess_outpaint_u8(self.h, _ptr(img8d), T, H, W, rw, rh, pw, ph, _ptr(orig),
                                                       _ptr(frames), _ptr(fm), _ptr(md), self._stream()))
        self._keep_staging = staging
        return frames.unsqueeze(0), fm.unsqueeze(0), md.unsqueeze(0), orig

    def postprocess(self, comp_u8: torch.Tensor) -> torch.Tensor:
        """uint8 [T,H,W,3] -> float32/255 on the device (handle_output)."""
        out = torch.empty(comp_u8.shape, device=self.device, dtype=torch.float32)
        self._check(self.lib.pp_postprocess(self.h, _ptr(comp_u8), _ptr(out), comp_u8.numel(), self._stream()))
        return out

    # -- multi-GPU exchange (NCCL communicator inside the C library)
    rank, world = 0, 1

    def comm_unique_id(self) -> bytes:
        buf = ctypes.create_string_buffer(128)
        self._check(self.lib.pp_comm_unique_id(buf))
        return buf.raw

    def comm_init(self, unique_id: bytes, rank: int, world: int):
        assert len(unique_id) == 128
        self._check(self.lib.pp_comm_init(self.h, ctypes.create_string_buffer(unique_id, 128), int(rank), int(world)))
        self.rank, self.world = int(rank), int(world)

    def comm_destroy(self):
        self._check(self.lib.pp_comm_destroy(self.h))
        self.rank, self.world = 0, 1

    def comm_all_gather_rows(self, buf: torch.Tensor, rows, first_rank: int = 0):
        """In-place all-gather along dim 0 of the contiguous tensor `buf` among ranks
        [first_rank, first_rank + len(rows)): member m owns rows [sum(rows[:m]), +rows[m])."""
        assert buf.is_contiguous() and buf.shape[0] == sum(rows)
        row_bytes = buf[0].numel() * buf.element_size() if buf.shape[0] else 0
        if len(rows) <= 1 or row_bytes == 0:
            return buf
        arr = (ctypes.c_longlong * len(rows))(*[int(r) for r in rows])
        self._check(self.lib.pp_comm_all_gather_rows(self.h, _ptr(buf), arr, row_bytes, int(first_rank), len(rows),
                                                     self._stream()))
        return buf

    @property
    def launch_count(self) -> int:
        return int(self.lib.pp_launch_count(self.h))

    @property
    def workspace_peak(self) -> int:
        return int(self.lib.pp_workspace_peak(self.h))

    def profile_enable(self, on: bool):
        self._check(self.lib.pp_profile_enable(self.h, int(on)))

    def profile_dump(self):
        """-> {kernel name: dict(count, ms, rows, flops, bytes)} since profile_enable(True)."""
        buf = ctypes.create_string_buffer(1 << 20)
        self._check(self.lib.pp_profile_dump(self.h, buf, len(buf)))
        out = {}
        for line in buf.value.decode().splitlines():
            name, n, ms, rows, flops, nbytes = line.split("\t")
            out[name] = dict(count=int(n), ms=float(ms), rows=float(rows), flops=float(flops), bytes=float(nbytes))
        return out

    # -- single operators (tests / micro-benchmarks)
    def op_conv(self, name, x_nhwc, stride=1, pad=0, dil=1, replicate=False, act=ACT_NONE, slope=0.0, residual=None):
        m = self.conv_meta[name]
        N, H, W, _ = x_nhwc.shape
        kh, kw = m["kh"], m["kw"]
        OH = (H + 2 * pad - dil * (kh - 1) - 1) // stride + 1
        OW = (W + 2 * pad - dil * (kw - 1) - 1) // stride + 1
        out = torch.empty(N, OH, OW, m["cout_g"] * m["groups"], device=self.device, dtype=torch.float16)
        self._check(self.lib.pp_op_conv(self.h, name.encode(), _ptr(x_nhwc), N, H, W, stride, pad, dil, int(replicate),
                                        act, float(slope), _ptr(residual), _ptr(out), self._stream()))
        return out

    def op_conv_ex(self, name, x, out, x_co=0, out_co=0, pad=(0, 0), act=ACT_NONE, slope=0.0, scale=1.0, act2=ACT_NONE,
                   residual=None, gru_zr=None, gru_h=None):
        """One stride-1 fp16 convolution (weights from register_conv) of x [N,H,W,C] from channel x_co into out
        [N,OH,OW,C'] from channel out_co.  Epilogue: act / slope / scale / act2 and an optional residual (tensor, co); or
        gru_zr = (h, h_co, rh, rh_co) (z -> out, r * h -> rh); or gru_h = (h, h_co, z, z_co)."""
        N, H, W, xC = x.shape
        C = lambda t: 0 if t is None else t.shape[-1]
        epi, a0, a0_co, a1, a1_co = self.EPI_STD, None, 0, None, 0
        if residual is not None:
            a0, a0_co = residual
        if gru_zr is not None:
            epi, (a0, a0_co, a1, a1_co) = self.EPI_GRU_ZR, gru_zr
        if gru_h is not None:
            epi, (a0, a0_co, a1, a1_co) = self.EPI_GRU_H, gru_h
        self._check(self.lib.pp_op_conv_ex(
            self.h, name.encode(), _ptr(x), xC, x_co, N, H, W, pad[0], pad[1], epi, act, float(slope), float(scale), act2,
            _ptr(a0), C(a0), a0_co, _ptr(a1), C(a1), a1_co, _ptr(out), C(out), out_co, self._stream()))
        return out

    def op_conv_segs(self, name, segs, out, out_co=0, out_gstep=0, out_f32=False, stride=(1, 1), pad=(0, 0),
                     dilation=(1, 1), replicate=False, act=ACT_NONE, slope=0.0, scale=1.0, act2=ACT_NONE, residual=None,
                     gru_zr=None, gru_h=None):
        """One fp16 convolution (weights from register_conv) built as the stages build it (pp_op_conv_segs).
        segs: 1..6 input segments (x [N,H,W,C] fp16, first channel, channels, gstep): the layer's input is their channel
        concatenation, group g reading each segment from channel co + g * gstep.  out [N,OH,OW,C'] fp16 written from
        channel out_co (+ g * out_gstep), or with out_f32 float32.  Epilogue as in op_conv_ex."""
        N, H, W = segs[0][0].shape[:3]
        n = len(segs)
        ints = lambda v: (ctypes.c_int * n)(*[int(i) for i in v])
        ptrs = (ctypes.c_void_p * n)(*[t.data_ptr() for t, *_ in segs])
        C = lambda t: 0 if t is None else t.shape[-1]
        epi, a0, a0_co, a1, a1_co = self.EPI_STD, None, 0, None, 0
        if residual is not None:
            a0, a0_co = residual
        if gru_zr is not None:
            epi, (a0, a0_co, a1, a1_co) = self.EPI_GRU_ZR, gru_zr
        if gru_h is not None:
            epi, (a0, a0_co, a1, a1_co) = self.EPI_GRU_H, gru_h
        self._check(self.lib.pp_op_conv_segs(
            self.h, name.encode(), n, ptrs, ints(t.shape[-1] for t, *_ in segs), ints(s[1] for s in segs),
            ints(s[2] for s in segs), ints(s[3] for s in segs), N, H, W, stride[0], stride[1], pad[0], pad[1],
            dilation[0], dilation[1], int(replicate), epi, act, float(slope), float(scale), act2, _ptr(a0), C(a0), a0_co,
            _ptr(a1), C(a1), a1_co, _ptr(out), C(out), out_co, out_gstep, int(out_f32), self._stream()))
        return out

    def op_conv_last_plan(self) -> dict:
        """The tile plan of this thread's last convolution launch (pp_op_conv_last_plan): kernel 'g' / 'h' / 'i' / 'p',
        m (halo MT or gemm MB), bn, tps, flat, tma_out, sa, sb."""
        v = (ctypes.c_int * 8)()
        self._check(self.lib.pp_op_conv_last_plan(v, 8))
        return dict(kernel=chr(v[0]), m=v[1], bn=v[2], tps=v[3], flat=v[4], tma_out=v[5], sa=v[6], sb=v[7])

    def op_corr_lookup(self, levels, coords, h8, w8):
        nq = coords.shape[0]
        out = torch.empty(nq, 328, device=self.device, dtype=torch.float16)
        self._check(self.lib.pp_op_corr_lookup(self.h, *[_ptr(l) for l in levels], _ptr(coords), _ptr(out), nq, h8, w8,
                                               self._stream()))
        return out

    EPI_STD, EPI_GRU_ZR, EPI_GRU_H = range(3)

    def op_conv_tf32(self, name, inputs, out, out_co=0, stride=(1, 1), pad=(0, 0), act=ACT_NONE, slope=0.0, scale=1.0,
                     act2=ACT_NONE, residual=None, gru_zr=None, gru_h=None, out_fp32=False, dilation=(1, 1),
                     replicate=False):
        """One split-tf32 convolution (weights from register_conv_tf32) on split tensors [N,H,W,2C] float32 (split_tf32:
        hi channels, then lo).  inputs: one or two (tensor, first channel, channels); out: split tensor written at channel
        out_co, or with out_fp32 a plain [N,OH,OW,C] float32 tensor; padding is zeros or, with replicate, the edge
        pixels.  Epilogue: act / slope / scale / act2 and an optional
        residual (tensor, co); or gru_zr = (h, h_co, rh, rh_co) (z -> out, r * h -> rh); or gru_h = (h, h_co, z, z_co)."""
        N, H, W = inputs[0][0].shape[:3]
        (x0, c0, n0), (x1, c1, n1) = inputs[0], (inputs[1] if len(inputs) > 1 else (None, 0, 0))
        C = lambda t: 0 if t is None else t.shape[-1] // 2
        epi, a0, a0_co, a1, a1_co = self.EPI_STD, None, 0, None, 0
        if residual is not None:
            a0, a0_co = residual
        if gru_zr is not None:
            epi, (a0, a0_co, a1, a1_co) = self.EPI_GRU_ZR, gru_zr
        if gru_h is not None:
            epi, (a0, a0_co, a1, a1_co) = self.EPI_GRU_H, gru_h
        self._check(self.lib.pp_op_conv_tf32(
            self.h, (name + ".tf32").encode(), _ptr(x0), C(x0), c0, n0, _ptr(x1), C(x1), c1, n1, N, H, W, stride[0],
            stride[1], pad[0], pad[1], dilation[0], dilation[1], int(replicate), epi, act, float(slope), float(scale), act2, _ptr(a0), C(a0), a0_co, _ptr(a1), C(a1),
            a1_co, _ptr(out), out.shape[-1] if out_fp32 else C(out), out_co, int(out_fp32), self._stream()))
        return out

    def op_dcn_sample_f32(self, x0, x1, offs, max_mag=5.0):
        """fp32 deformable sampler of flow completion: split x0 [N,H,W,2*C0] and x1 [N,H,W,2*C1] (C0 + C1 = 256), offs
        float32 [N,H,W,432] -> split columns [N,H,W,2*2304] (hi 2304 | lo 2304, K ordered (tap, channel)).  x1 may be
        None when x0 holds all 256 channels."""
        N, H, W = x0.shape[:3]
        cols = torch.empty(N, H, W, 2 * 2304, device=self.device, dtype=torch.float32)
        C1 = 0 if x1 is None else x1.shape[-1] // 2
        self._check(self.lib.pp_op_dcn_sample_f32(self.h, _ptr(x0), x0.shape[-1] // 2, _ptr(x1), C1, _ptr(offs), N, H,
                                                  W, float(max_mag), _ptr(cols), self._stream()))
        return cols

    def op_upsample2x_f32(self, x):
        """bilinear x2 (align_corners=True) of a split tensor [N,H,W,2C] -> [N,2H,2W,2C]."""
        N, H, W, C2 = x.shape
        out = torch.empty(N, 2 * H, 2 * W, C2, device=self.device, dtype=torch.float32)
        self._check(self.lib.pp_op_upsample2x_f32(self.h, _ptr(x), _ptr(out), N, H, W, C2 // 2, self._stream()))
        return out

    def op_instnorm(self, x, C, relu=False, residual=None, out=None, fp32=True):
        """InstanceNorm2d of x [N,HW,C] fp16 (fp32=False) or [N,HW,2C] split float32, + relu, then relu(residual + .)."""
        out = torch.empty_like(x) if out is None else out
        N, HW = x.shape[:2]
        self._check(self.lib.pp_op_instnorm(self.h, _ptr(x), _ptr(residual), _ptr(out), N, HW, C, int(relu), int(fp32),
                                            self._stream()))
        return out

    def op_corr_pyramid(self, fmap1, fmap2, h8, w8, fp32=True):
        """fmap1 / fmap2 [pairs, h8*w8, 256] fp16 or [pairs, h8*w8, 512] split float32 -> the 4 pyramid levels
        [pairs*h8*w8, (h8 >> l) * (w8 >> l)] (fp16 / float32)."""
        pairs = fmap1.shape[0]
        dt = torch.float32 if fp32 else torch.float16
        lv = [torch.empty(pairs * h8 * w8, (h8 >> l) * (w8 >> l), device=self.device, dtype=dt) for l in range(4)]
        self._check(self.lib.pp_op_corr_pyramid(self.h, _ptr(fmap1), _ptr(fmap2), pairs, h8, w8, int(fp32),
                                                *[_ptr(t) for t in lv], self._stream()))
        return lv

    def op_corr_lookup_f32(self, levels, coords, h8, w8):
        """fp32 pyramid -> split [nq, 704] float32 (hi 352 | lo 352)."""
        nq = coords.shape[0]
        out = torch.empty(nq, 704, device=self.device, dtype=torch.float32)
        self._check(self.lib.pp_op_corr_lookup_f32(self.h, *[_ptr(l) for l in levels], _ptr(coords), _ptr(out), nq, h8,
                                                   w8, self._stream()))
        return out

    def op_convex_upsample(self, coords1, mask, B, h8, w8, fp32=True):
        """coords1 [B*h8*w8, 2], mask [B*h8*w8, 576] fp16 or [B*h8*w8, 1152] split float32 -> [B, 2, 8*h8, 8*w8]."""
        out = torch.empty(B, 2, 8 * h8, 8 * w8, device=self.device, dtype=torch.float32)
        self._check(self.lib.pp_op_convex_upsample(self.h, _ptr(coords1), _ptr(mask), _ptr(out), B, h8, w8, int(fp32),
                                                   self._stream()))
        return out

    def op_imgprop_step(self, cur4, prop4, flow_prop, flow_check):
        H, W, _ = cur4.shape
        out = torch.empty_like(cur4)
        self._check(self.lib.pp_op_imgprop_step(self.h, _ptr(cur4), _ptr(prop4), _ptr(out), _ptr(flow_prop),
                                                _ptr(flow_check), H, W, self._stream()))
        return out

    def op_imgprop_step_f32(self, cur4, prop4, flow_prop, flow_check):
        """One fp32 propagation step: cur4 / prop4 float32 [H,W,4] (r, g, b, mask), flows float32 [H,W,2]."""
        H, W, _ = cur4.shape
        out = torch.empty_like(cur4)
        self._check(self.lib.pp_op_imgprop_step_f32(self.h, _ptr(cur4), _ptr(prop4), _ptr(out), _ptr(flow_prop),
                                                    _ptr(flow_check), H, W, self._stream()))
        return out

    def op_attention(self, qkv, pkv, win_flags, win_t, gh, gw, n_pool, parity):
        """Sparse window attention of sliding windows with win_t[w] frames each, concatenated: qkv fp16
        [sum(win_t), nh*nw, 1536], pkv fp16 [sum(win_t), n_pool, 1024], win_flags int32 [len(win_t), nwh*nww]
        -> [sum(win_t), gh, gw, 512].  An int win_t is one sliding window of that many frames."""
        win_t = [int(win_t)] if isinstance(win_t, int) else [int(t) for t in win_t]
        out = torch.zeros(sum(win_t), gh, gw, 512, device=self.device, dtype=torch.float16)
        self._check(self.lib.pp_op_attention(self.h, _ptr(qkv), _ptr(pkv), _ptr(out), _ptr(win_flags),
                                             (ctypes.c_int * len(win_t))(*win_t), len(win_t), gh, gw, n_pool, parity,
                                             self._stream()))
        return out

    def op_layernorm(self, x, gamma, beta, gh, gw, nh, nw, fill=0.0):
        """LayerNorm(512) of x fp16 [t*gh*gw, 512] -> fp16 [t, nh, nw, 512]; padding rows keep `fill`."""
        t = x.shape[0] // (gh * gw)
        out = torch.full((t, nh, nw, 512), fill, device=self.device, dtype=torch.float16)
        self._check(self.lib.pp_op_layernorm(self.h, _ptr(x), _ptr(gamma), _ptr(beta), _ptr(out), t, gh, gw, nh, nw,
                                             self._stream()))
        return out

    def op_pool_tokens(self, x, w, b):
        """Depthwise 4x4 stride-4 pooling of x fp16 [t, nh, nw, C], w float32 [16, C] (tap-major), b float32 [C]."""
        t, nh, nw, C = x.shape
        out = torch.empty(t, (nh - 4) // 4 + 1, (nw - 4) // 4 + 1, C, device=self.device, dtype=torch.float16)
        self._check(self.lib.pp_op_pool_tokens(self.h, _ptr(x), _ptr(w), _ptr(b), _ptr(out), t, nh, nw, C,
                                               self._stream()))
        return out

    def op_window_flags(self, mask4, co, win_f0, win_lt):
        """mask4 fp16 [T, h4, w4, cs] (channel co) -> int32 [len(win_f0), nwh*nww] masked-window flags."""
        _, h4, w4, cs = mask4.shape
        gh, gw = (h4 - 1) // 3 + 1, (w4 - 1) // 3 + 1
        n = len(win_f0)
        flags = torch.full((n, -(-gh // 5) * -(-gw // 9)), -1, device=self.device, dtype=torch.int32)
        arr = lambda v: (ctypes.c_int * n)(*[int(i) for i in v])
        self._check(self.lib.pp_op_window_flags(self.h, _ptr(mask4), cs, co, arr(win_f0), arr(win_lt), n, h4, w4,
                                                _ptr(flags), self._stream()))
        return flags

    def op_fold(self, x, t, H, W, C, normalise, gelu):
        """F.fold(7, stride 3, pad 3) of x fp16 [t*gh*gw, cs] -> fp16 [t, H, W, C]."""
        out = torch.empty(t, H, W, C, device=self.device, dtype=torch.float16)
        self._check(self.lib.pp_op_fold(self.h, _ptr(x), x.shape[-1], _ptr(out), t, H, W, C, int(normalise), int(gelu),
                                        self._stream()))
        return out

    def op_featprop_cond(self, cur, prop, flow_prop, flow_check, mask2):
        """cur / prop fp16 [N, H, W, 128], flows fp16 [N, H, W, 2], mask2 fp16 [N, H, W, 8] -> cond fp16 [N, H, W, 264]."""
        N, H, W, _ = cur.shape
        cond = torch.full((N, H, W, 264), float("nan"), device=self.device, dtype=torch.float16)
        self._check(self.lib.pp_op_featprop_cond(self.h, _ptr(cur), _ptr(prop), _ptr(flow_prop), _ptr(flow_check),
                                                 _ptr(mask2), _ptr(cond), N, H, W, self._stream()))
        return cond

    def op_dcn_sample(self, x0, offs, max_mag, x1=None, flow=None):
        """fp16 deformable sampler: x0 [N, H, W, C0] (+ x1 [N, H, W, C1]), offs [N, H, W, 432], flow = (tensor
        [N, H, W, cs], co) or None -> columns fp16 [N, H, W, 9 * (C0 + C1)]."""
        N, H, W, C0 = x0.shape
        C1 = 0 if x1 is None else x1.shape[-1]
        ft, fco = flow if flow is not None else (None, 0)
        cols = torch.empty(N, H, W, 9 * (C0 + C1), device=self.device, dtype=torch.float16)
        self._check(self.lib.pp_op_dcn_sample(self.h, _ptr(x0), C0, C0, _ptr(x1), C1, C1, _ptr(offs), _ptr(ft),
                                              0 if ft is None else ft.shape[-1], fco, float(max_mag), _ptr(cols), N, H,
                                              W, self._stream()))
        return cols

    def op_downsample4(self, flows=None, masks=None, mask_co=0):
        """flows float32 [n, 2, H, W] -> fp16 [n, H/4, W/4, 2]; masks float32 [n, 1, H, W] -> fp16 [n, H/4, W/4, 8]
        (channel mask_co written, the others zero)."""
        H, W = (flows if flows is not None else masks).shape[-2:]
        f4 = None if flows is None else torch.empty(flows.shape[0], H // 4, W // 4, 2, device=self.device,
                                                    dtype=torch.float16)
        m4 = None if masks is None else torch.zeros(masks.shape[0], H // 4, W // 4, 8, device=self.device,
                                                    dtype=torch.float16)
        self._check(self.lib.pp_op_downsample4(self.h, _ptr(flows), _ptr(f4), 0 if flows is None else flows.shape[0],
                                               _ptr(masks), _ptr(m4), mask_co, 0 if masks is None else masks.shape[0],
                                               H, W, self._stream()))
        return f4, m4

    def op_upsample2x(self, x):
        """bilinear x2 (align_corners=True) of fp16 [N, H, W, C] -> [N, 2H, 2W, C]."""
        N, H, W, C = x.shape
        out = torch.empty(N, 2 * H, 2 * W, C, device=self.device, dtype=torch.float16)
        self._check(self.lib.pp_op_upsample2x(self.h, _ptr(x), _ptr(out), N, H, W, C, self._stream()))
        return out
