"""CPU tests: C-ABI library exports, weight packing, node surface, window scheduling, image utils."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from comfyui_propainter_nodes_b200 import engine as E
from comfyui_propainter_nodes_b200 import weights as Wt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "propainter_b200.h")).read()
    declared = sorted(set(re.findall(r"PP_API [a-z_ \*]+?(pp_[a-z_0-9]+)\(", hdr)))
    assert declared, "no declarations found"
    assert declared == E.exported_symbols(), (declared, E.exported_symbols())
    lib = ctypes.CDLL(E.LIB_PATH)          # loads without a GPU
    for name in declared:
        getattr(lib, name)                 # raises if not exported
    E.load_library()
    assert b"sm_90a" in E.load_library().pp_version()


def _unpack(packed, meta):
    G, kc, rows = packed.shape[0], packed.shape[1], packed.shape[2]
    pos = torch.arange(8).view(1, 8) ^ (torch.arange(rows).view(-1, 1) & 7)
    un = torch.gather(packed.float(), 3, pos.view(1, 1, rows, 8, 1).expand(G, kc, rows, 8, 8))  # xor is an involution
    return un.permute(0, 2, 1, 3, 4).reshape(G, rows, kc * 64)


@pytest.mark.parametrize("cout,cin,k,groups,cin_pad", [(64, 3, 7, 1, 8), (384, 768, 3, 4, None), (126, 256, 3, 1, None),
                                                       (432, 128, 3, 1, None), (1960, 512, 1, 1, None)])
def test_pack_conv_weight_roundtrip(cout, cin, k, groups, cin_pad):
    g = torch.Generator().manual_seed(0)
    w = torch.randn(cout, cin // groups, k, k, generator=g)
    cmap = None if cin_pad is None else list(range(cin)) + [-1] * (cin_pad - cin)
    packed, meta = E.pack_conv_weight(w, groups, cmap)
    assert meta["bn"] % 16 == 0 and meta["bn"] <= 256 and meta["cout_g_pad"] % meta["bn"] == 0
    un = _unpack(packed, meta)
    cin_k = meta["cin_g"]
    K = k * k * cin_k
    ref = torch.zeros(cout, k, k, cin_k)
    ref[..., :cin // groups] = w.permute(0, 2, 3, 1)
    ref = ref.reshape(groups, cout // groups, K).half().float()
    assert torch.equal(un[:, :cout // groups, :K], ref)
    assert float(un[:, cout // groups:].abs().max() if un.shape[1] > cout // groups else 0) == 0
    assert float(un[:, :, K:].abs().max() if un.shape[2] > K else 0) == 0


def test_build_layers_covers_checkpoints():
    convs, tens = E.build_layers(Wt.synthetic_raft_state_dict(), Wt.synthetic_rfc_state_dict(),
                                 Wt.synthetic_generator_state_dict())
    assert len(convs) == 150 and len(tens) == 8 * 6
    # every kernel-side input channel count is a multiple of 8
    for name, (w, b, groups, cmap, macs) in convs.items():
        cin = len(cmap) if cmap is not None else w.shape[1]
        assert (cin + (-cin) % 8) % 8 == 0
    # GRU gate merge: z|r stacked along Cout
    assert convs["raft.update.gru.zr1"][0].shape == (256, 384, 1, 5)


def test_bn_folding_matches_batchnorm():
    sd = {k[7:]: v for k, v in Wt.synthetic_raft_state_dict().items()}
    convs, _ = E.build_layers(Wt.synthetic_raft_state_dict(), Wt.synthetic_rfc_state_dict(),
                              Wt.synthetic_generator_state_dict())
    w, b, _, _, _ = convs["raft.cnet.layer1.0.conv1"]
    x = torch.randn(1, 64, 9, 11)
    y = torch.nn.functional.conv2d(x, sd["cnet.layer1.0.conv1.weight"], sd["cnet.layer1.0.conv1.bias"], padding=1)
    y = torch.nn.functional.batch_norm(y, sd["cnet.layer1.0.norm1.running_mean"], sd["cnet.layer1.0.norm1.running_var"],
                                       sd["cnet.layer1.0.norm1.weight"], sd["cnet.layer1.0.norm1.bias"], False, 0.0, 1e-5)
    y2 = torch.nn.functional.conv2d(x, w, b, padding=1)
    assert (y - y2).abs().max() < 1e-4


def test_strict_checkpoint_validation():
    sd = Wt.synthetic_rfc_state_dict()
    sd.pop("fusion.weight", None)
    bad = dict(sd)
    bad.pop("downsample.0.weight")
    with pytest.raises(KeyError):
        Wt.check_state_dict(bad, Wt.rfc_spec())


def test_ring_indices_match_reference_buffer():
    idx = Wt.rolled_valid_indices()
    assert idx.shape == (148,) and idx[0] == 4  # first kept entry of the top-left mask is (row 0, col 4)


def test_node_surface():
    from comfyui_propainter_nodes_b200 import NODE_CLASS_MAPPINGS, NODE_DISPLAY_NAME_MAPPINGS
    assert set(NODE_CLASS_MAPPINGS) == {"ProPainterInpaint", "ProPainterOutpaint"}
    assert NODE_DISPLAY_NAME_MAPPINGS["ProPainterInpaint"] == "ProPainter Inpainting"
    inp = NODE_CLASS_MAPPINGS["ProPainterInpaint"]
    req = inp.INPUT_TYPES()["required"]
    assert list(req) == ["image", "mask", "width", "height", "mask_dilates", "flow_mask_dilates", "ref_stride",
                         "neighbor_length", "subvideo_length", "raft_iter", "fp16"]
    assert req["width"][1] == {"default": 640, "min": 0, "max": 2560} and req["raft_iter"][1]["default"] == 20
    assert inp.RETURN_TYPES == ("IMAGE", "MASK", "MASK") and inp.FUNCTION == "propainter_inpainting"
    out = NODE_CLASS_MAPPINGS["ProPainterOutpaint"]
    assert "mask" not in out.INPUT_TYPES()["required"] and out.RETURN_TYPES == ("IMAGE", "MASK", "INT", "INT")
    assert out.INPUT_TYPES()["required"]["width_scale"][1]["default"] == 1.2


def test_check_inputs_errors():
    from comfyui_propainter_nodes_b200.propainter_nodes import check_inputs
    with pytest.raises(Exception, match="greater than 1"):
        check_inputs(torch.zeros(1, 8, 8, 3), torch.zeros(1, 8, 8))
    with pytest.raises(Exception, match="same length"):
        check_inputs(torch.zeros(4, 8, 8, 3), torch.zeros(3, 8, 8))
    with pytest.raises(Exception, match="same dimensions"):
        check_inputs(torch.zeros(4, 8, 8, 3), torch.zeros(4, 8, 9))
    check_inputs(torch.zeros(4, 8, 8, 3), torch.zeros(1, 8, 8))


def test_window_schedule_matches_oracle():
    from comfyui_propainter_nodes_b200 import propainter_inference as PI
    from oracle import propainter_oracle as O
    for T, nl, rs, sv in ((80, 10, 10, 80), (240, 10, 10, 80), (16, 10, 10, 80), (8, 4, 3, 80), (33, 6, 7, 20)):
        cfg = PI.ProPainterConfig(rs, nl, sv, 20, "enable", T, torch.device("cpu"), (64, 64))
        assert PI.window_schedule(cfg) == O.window_schedule(T, nl, rs, sv)


def test_engine_refuses_without_gpu():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        E.Engine("cuda:0")


def test_outpaint_canvas():
    from comfyui_propainter_nodes_b200.utils import image_utils as IU
    from comfyui_propainter_nodes_b200.synthetic import synthetic_clip
    img = synthetic_clip(3, 64, 96, 1)
    cfg = IU.ImageOutpaintConfig(96, 64, 5, 8, (96, 64), 3, 1.5, 1.0)
    assert cfg.outpaint_size == (144, 64)
    canvas, fm, md = IU.extrapolation(IU.convert_image_to_frames(img), cfg)
    a, f, m = np.array(canvas[0]), np.array(fm[0]), np.array(md[0])
    assert a.shape == (64, 144, 3) and (a[:, :24] == 0).all() and (a[:, 24:120] > 0).any()
    assert (m[:, :24] == 255).all() and (m[:, 24:120] == 0).all()
    assert (f[:, :28] == 255).all() and (f[:, 28:116] == 0).all()   # 4-px inset of the flow mask


def test_outpaint_tensor_path_matches_pil_path():
    """The device-side canvas / band-mask assembly equals the reference-style PIL path bit for bit."""
    from comfyui_propainter_nodes_b200.utils import image_utils as IU
    g = torch.Generator().manual_seed(5)
    for (T, H, W, ws, hs) in ((3, 48, 64, 1.2, 1.0), (2, 40, 56, 1.5, 1.3), (2, 32, 32, 1.0, 1.26)):
        image = torch.rand(T, H, W, 3, generator=g)
        cfg = IU.ImageOutpaintConfig(W, H, 5, 8, (W, H), T, ws, hs)
        canvas, fm_l, md_l = IU.extrapolation(IU.convert_image_to_frames(image), cfg)
        ft0, fm0, md0, orig0 = IU.prepare_frames_and_masks_for_outpaint(canvas, fm_l, md_l, torch.device("cpu"))
        ft1, fm1, md1, orig1 = IU.outpaint_tensors(image, cfg, torch.device("cpu"))
        assert torch.equal(ft0, ft1) and torch.equal(fm0, fm1) and torch.equal(md0, md1)
        assert np.array_equal(np.stack(orig0), orig1.numpy())


def test_encoder14_dense_weights_equal_grouped_conv():
    """gen.encoder.14 (8 groups of 80 -> 32 channels) is registered as a dense conv with block-diagonal weights over
    cat(x0[256], prev[384]); it must reproduce the reference's grouped conv over the interleaved input
    (model/propainter.py:268-273)."""
    import torch.nn.functional as F
    sd = Wt.synthetic_generator_state_dict()
    convs, _ = E.build_layers(Wt.synthetic_raft_state_dict(), Wt.synthetic_rfc_state_dict(), sd)
    w_dense, b, groups, cmap, macs = convs["gen.encoder.14"]
    assert groups == 1 and cmap is None and tuple(w_dense.shape[:2]) == (256, 640)
    g = torch.Generator().manual_seed(11)
    x0, prev = torch.randn(1, 256, 9, 11, generator=g), torch.randn(1, 384, 9, 11, generator=g)
    gr = 8
    # reference: x = cat([x0.view(g, -1), prev.view(g, -1)], 2) per group, then grouped conv
    xi = torch.cat([x0.view(1, gr, -1, 9, 11), prev.view(1, gr, -1, 9, 11)], 2).view(1, -1, 9, 11)
    ref = F.conv2d(xi, sd["encoder.layers.14.weight"].float(), sd["encoder.layers.14.bias"].float(), 1, 1, 1, gr)
    out = F.conv2d(torch.cat([x0, prev], 1), w_dense, b, 1, 1)
    assert torch.allclose(out, ref, atol=1e-5, rtol=1e-5)


def test_pad64_layers_are_registered_with_zero_extended_channels():
    """Layers on the PAD64 list get kernel input channels padded to a multiple of 64 with -1 (zero weight) entries;
    the activation tensors keep their real channel count (TMA zero-fills the rest, PPConvSeg.cvalid)."""
    convs, _ = E.build_layers(Wt.synthetic_raft_state_dict(), Wt.synthetic_rfc_state_dict(),
                              Wt.synthetic_generator_state_dict())
    for name in E.Engine.PAD64_CONVS:
        w, b, groups, cmap, _ = convs[name]
        cmap = list(cmap) if cmap is not None else list(range(w.shape[1]))
        padded = cmap + [-1] * ((-len(cmap)) % 64)
        assert groups == 1 and len(padded) % 64 == 0 and len(padded) - len(cmap) < 64
        packed, meta = E.pack_conv_weight(w, 1, padded)
        assert meta["cin_g"] == len(padded)
        un = _unpack(packed, meta)[0, : w.shape[0]]                       # [cout, kh*kw*cin_k]
        un = un[:, : meta["kh"] * meta["kw"] * len(padded)].view(w.shape[0], meta["kh"] * meta["kw"], len(padded))
        real = [i for i, c in enumerate(padded) if c >= 0]
        pad = [i for i, c in enumerate(padded) if c < 0]
        assert float(un[:, :, pad].abs().max()) == 0.0 if pad else True
        ref = w[:, [padded[i] for i in real]].permute(0, 2, 3, 1).reshape(w.shape[0], -1, len(real)).half().float()
        assert torch.equal(un[:, :, real], ref)


def test_bench_reference_arm_prints_one_json_line(monkeypatch, capfd):
    """bench.py contract: exactly one JSON line on stdout (everything else on stderr) with the agreed keys."""
    import json
    import bench
    monkeypatch.setattr(bench, "cpu_sample", lambda n=3: (0.5, 6.0, "port", 8))
    monkeypatch.setattr(bench, "_OUT_FD", 1)
    args = type("A", (), dict(gpus=1, steps=2, warmup=1, no_ref_cuda=True))()
    print("noise that must not reach the JSON consumer", file=__import__("sys").stderr)
    bench.run_reference(args, rank=0)
    out = capfd.readouterr().out.strip().splitlines()
    assert len(out) == 1
    rec = json.loads(out[0])
    for key in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better",
                "scaling", "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e"):
        assert key in rec, key
    assert rec["impl"] == "reference" and rec["cpu_baseline"]["kind"] == "port" and rec["e2e"]["h2d_bytes_per_step"] == 0
    bench.run_reference(args, rank=1)            # other ranks stay silent
    assert capfd.readouterr().out == ""


def test_pil_bicubic_restatement_matches_pillow():
    """oracle/pil_resize.py (the arithmetic the device resize kernel implements) == Pillow's Image.resize, bit for bit."""
    from PIL import Image
    from oracle import pil_resize as PR
    rng = np.random.RandomState(0)
    for (H, W, oh, ow) in ((180, 320, 176, 320), (64, 96, 48, 72), (50, 70, 120, 200), (97, 131, 40, 57), (36, 64, 48, 64)):
        img = rng.randint(0, 256, (H, W, 3), dtype=np.uint8)
        assert np.array_equal(PR.resize_u8(img, ow, oh), np.array(Image.fromarray(img).resize((ow, oh)))), (H, W, oh, ow)
        m = rng.randint(0, 256, (H, W), dtype=np.uint8)
        assert np.array_equal(PR.resize_u8(m, ow, oh), np.array(Image.fromarray(m).resize((ow, oh)))), (H, W, oh, ow)


def test_host_quantiser_matches_reference_conversion():
    """pp_host_quantize_u8 (host helper of the e2e path, no GPU) == (x * 255).clip(0, 255).astype(uint8) of the reference
    (utils/image_utils.py:106-114), incl. out-of-range values, for every thread count."""
    lib = E.load_library()
    g = torch.Generator().manual_seed(0)
    x = torch.rand(3, 40, 56, 3, generator=g) * 1.4 - 0.2
    x[0, 0, 0, :] = torch.tensor([1.0, 0.0, 0.999999])
    ref = (x.numpy() * 255.0).clip(0, 255).astype(np.uint8)
    for threads in (1, 3, 16):
        out = torch.empty(x.shape, dtype=torch.uint8)
        assert lib.pp_host_quantize_u8(ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(out.data_ptr()), x.numel(), threads) == 0
        assert np.array_equal(out.numpy(), ref), threads
    big = torch.rand(1 << 18, generator=g)
    out = torch.empty(big.shape, dtype=torch.uint8)
    assert lib.pp_host_quantize_u8(ctypes.c_void_p(big.data_ptr()), ctypes.c_void_p(out.data_ptr()), big.numel(), 8) == 0
    assert np.array_equal(out.numpy(), (big.numpy() * 255.0).clip(0, 255).astype(np.uint8))


def test_window_sub_batches_cover_the_schedule_in_order():
    """Engine.gen_batches (host logic of the small-workspace fallback): consecutive sub-batches, nothing dropped or
    reordered, every batch within the budget unless it is a single window."""
    from oracle import propainter_oracle as O
    sched = O.window_schedule(240, 10, 10, 80)
    eng = E.Engine.__new__(E.Engine)            # host-side method only: no device, no library call
    per_slot = E.Engine.gen_slot_bytes(360, 640)
    assert 20e6 < per_slot < 100e6
    for budget_slots in (1000, 120, 40, 5):
        parts = eng.gen_batches(sched, budget_slots * per_slot, (240, 360, 640))
        assert [w for p in parts for w in p] == sched
        for p in parts:
            slots = sum(len(a) + len(b) for a, b in p)
            assert slots <= budget_slots or len(p) == 1
    assert len(eng.gen_batches(sched, 10 ** 15, (240, 360, 640))) == 1
    # the per-clip arena estimate saturates for long clips and covers the measured peaks (24.3 GB at C2, 92 GB at C4)
    assert E.Engine.clip_workspace_bytes(80, 360, 640) > 24.3e9 and E.Engine.clip_workspace_bytes(80, 720, 1280) > 92e9
    assert E.Engine.clip_workspace_bytes(1000, 360, 640) == E.Engine.clip_workspace_bytes(100, 360, 640)
