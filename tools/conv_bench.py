"""Micro-benchmark of the wgmma conv kernels on representative layers (CUDA events, L2 flushed).

1x1 layers (linear layers and 1x1 convolutions) also report torch.nn.functional.linear (cuBLAS, fp16 with bias) on
the same shape in the same process, as a yardstick for the flat GEMM kernel.  PP_CONV_NOEPI=1 in the environment skips
the epilogue math and stores of the conv kernels (main-loop timing; the outputs are then garbage).

EPI_CASES are the bench step's stride-1 layers with their real epilogues and output layouts (GRU gates, channel slices
of the hidden-state tensor, residuals), run through Engine.op_conv_ex."""
import math
import sys
import os

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from comfyui_propainter_nodes_b200 import engine as E

CASES = {
    # name: (N, H, W, Cin, Cout, kh, kw, stride, groups)
    "raft.gru.zr (1x5, 384->256)": (79, 45, 80, 384, 256, 1, 5, 1, 1),
    "raft.convc2 (3x3, 256->192)": (79, 45, 80, 256, 192, 3, 3, 1, 1),
    "raft.fh1 (3x3, 128->256)": (79, 45, 80, 128, 256, 3, 3, 1, 1),
    "raft.convc1 (1x1, 328->256)": (79, 45, 80, 328, 256, 1, 1, 1, 1),
    "gen.encoder.8 (3x3, 256->384)": (32, 90, 160, 256, 384, 3, 3, 1, 1),
    "gen.encoder.2 (3x3, 64->64 @180x320)": (32, 180, 320, 64, 64, 3, 3, 1, 1),
    "gen.decoder.4 (3x3, 64->64 @360x640)": (11, 360, 640, 64, 64, 3, 3, 1, 1),
    "tf.qkv (512->1536)": (1, 1, 29160, 512, 1536, 1, 1, 1, 1),
    "tf.fc1 (512->1960)": (1, 1, 29160, 512, 1960, 1, 1, 1, 1),
    "tf.qkv full (512->1536, M=445k)": (275, 30, 54, 512, 1536, 1, 1, 1, 1),
    "tf.proj full (512->512, M=445k)": (275, 30, 54, 512, 512, 1, 1, 1, 1),
    # flat layers at the shapes of one bench step (80 frames at 640x360)
    "tf.fc1 full (512->1960, M=445k)": (275, 30, 54, 512, 1960, 1, 1, 1, 1),
    "gen.sc.embedding (512->6272, M=275k)": (102, 45, 60, 512, 6272, 1, 1, 1, 1),
    "raft.convc1 full (1x1, 328->256, M=569k)": (158, 45, 80, 328, 256, 1, 1, 1, 1),
    "raft.convf1 (1x1, 128->128, M=569k)": (158, 45, 80, 128, 128, 1, 1, 1, 1),
    "gen.fp.dcn (1x1, 1152->128, M=288k)": (20, 90, 160, 1152, 128, 1, 1, 1, 1),
    "raft.mask2 (1x1, 256->576, M=569k)": (158, 45, 80, 256, 576, 1, 1, 1, 1),
    "raft.update.conv (3x3, 256->126)": (79, 45, 80, 256, 126, 3, 3, 1, 1),
    "raft.gru.q (1x5, 384->128)": (79, 45, 80, 384, 128, 1, 5, 1, 1),
    "raft.convf2 (3x3, 128->64)": (79, 45, 80, 128, 64, 3, 3, 1, 1),
    "gen.fp.offset.3 (3x3, 128->432 @90x160 x5)": (5, 90, 160, 128, 432, 3, 3, 1, 1),
    "gen.fp.backbone (3x3, 128->128 @90x160 x5)": (5, 90, 160, 128, 128, 3, 3, 1, 1),
    "gen.encoder.10 (3x3 g2, 640->512 @90x160)": (16, 90, 160, 640, 512, 3, 3, 1, 2),
    "rfc.offset.0 (3x3, 384->128, M=7200)": (2, 45, 80, 384, 128, 3, 3, 1, 1),
    "step conv (3x3, 128->128, M=7200)": (2, 45, 80, 128, 128, 3, 3, 1, 1),
    "step conv (3x3, 128->128, M=14400)": (1, 90, 160, 128, 128, 3, 3, 1, 1),
}


# name: (N, H, W, Cin, Cout, kh, kw, epilogue, output tensor width, output channel offset) at the shapes of one bench step
# (80 frames at 640x360: RAFT at 1/8 resolution over 79 pairs per direction, the generator's encoder / propagation /
# decoder).  Epilogues: "std" (bias + LReLU), "res" (+ residual), "zr" (GRU z | r * h), "h" (GRU (1 - z) h + z q, in place
# in hx[:, 0:128]).
EPI_CASES = {
    "raft.gru.zr1 (1x5, 384->256, z | r*h)": (158, 45, 80, 384, 256, 1, 5, "zr", 128, 0),
    "raft.gru.zr2 (5x1, 384->256, z | r*h)": (158, 45, 80, 384, 256, 5, 1, "zr", 128, 0),
    "raft.gru.q1 (1x5, 384->128, in place)": (158, 45, 80, 384, 128, 1, 5, "h", 384, 0),
    "raft.gru.q2 (5x1, 384->128, in place)": (158, 45, 80, 384, 128, 5, 1, "h", 384, 0),
    "raft.convc2 (3x3, 256->192 into 256)": (158, 45, 80, 256, 192, 3, 3, "std", 256, 0),
    "raft.convf2 (3x3, 128->64 into 256)": (158, 45, 80, 128, 64, 3, 3, "std", 256, 192),
    "raft.update.conv (3x3, 256->126 into 384)": (158, 45, 80, 256, 126, 3, 3, "std", 384, 256),
    "raft.fh1 (3x3, 128->256)": (158, 45, 80, 128, 256, 3, 3, "std", 256, 0),
    "gen.fp.backbone.1 (3x3, 128->128 +res)": (20, 90, 160, 128, 128, 3, 3, "res", 128, 0),
    "gen.encoder.8 (3x3, 256->384)": (80, 90, 160, 256, 384, 3, 3, "std", 384, 0),
    "gen.decoder.4 (3x3, 64->64 @360x640)": (11, 360, 640, 64, 64, 3, 3, "std", 64, 0),
}


def _epi_case(eng, name, case, flush):
    N, H, W, cin, cout, kh, kw, epi, out_c, out_co = case
    w = torch.randn(cout, cin, kh, kw) / math.sqrt(cin * kh * kw)
    eng.register_conv("b", w, torch.randn(cout) * 0.1, 1)
    dev = "cuda:0"
    x = torch.randn(N, H, W, cin, device=dev, dtype=torch.float16)
    pad = (kh // 2, kw // 2)
    kw_ = {}
    if epi == "zr":
        out = torch.empty(N, H, W, out_c, device=dev, dtype=torch.float16)
        hx = torch.randn(N, H, W, 384, device=dev, dtype=torch.float16)
        rh = torch.empty(N, H, W, 128, device=dev, dtype=torch.float16)
        kw_["gru_zr"] = (hx, 0, rh, 0)
    elif epi == "h":
        out = torch.randn(N, H, W, out_c, device=dev, dtype=torch.float16)
        z = torch.rand(N, H, W, 128, device=dev, dtype=torch.float16)
        kw_["gru_h"] = (out, 0, z, 0)
    else:
        out = torch.empty(N, H, W, out_c, device=dev, dtype=torch.float16)
        kw_.update(act=E.ACT_LRELU, slope=0.2)
        if epi == "res":
            kw_["residual"] = (torch.randn(N, H, W, cout, device=dev, dtype=torch.float16), 0)
    fn = lambda: eng.op_conv_ex("b", x, out, out_co=out_co, pad=pad, **kw_)
    ms = _time_ms(fn, flush)
    fl = 2.0 * N * H * W * cout * cin * kh * kw
    print(f"{name:42s} M={N * H * W:8d} bn={eng.conv_meta['b']['bn']:3d} {ms:8.3f} ms {fl / ms / 1e9:8.1f} TFLOP/s",
          flush=True)


def _time_ms(fn, flush, reps=5):
    """Median of `reps` single launches, each after an L2 flush (CUDA events around the call)."""
    for _ in range(3):
        fn()
    ts = []
    for _ in range(reps):
        flush.fill_(0)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


def main():
    only = sys.argv[1:]
    eng = E.Engine("cuda:0", workspace_gb=2.0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda:0")
    print(f"# {torch.cuda.get_device_name(0)}, PP_CONV_NOEPI={os.environ.get('PP_CONV_NOEPI', '0')}", flush=True)
    for name, (N, H, W, cin, cout, kh, kw, s, g) in CASES.items():
        if only and not any(o in name for o in only):
            continue
        w = torch.randn(cout, cin // g, kh, kw) / math.sqrt(cin * kh * kw)
        bias = torch.randn(cout) * 0.1
        eng.register_conv("b", w, bias, g)
        x = torch.randn(N, H, W, cin, device="cuda:0", dtype=torch.float16)
        if kh != kw:
            x = torch.nn.functional.pad(x, (0, 0, kw // 2, kw // 2, kh // 2, kh // 2)).contiguous()
            pad = 0
        else:
            pad = kh // 2
        y = eng.op_conv("b", x, s, pad)
        ms = _time_ms(lambda: eng.op_conv("b", x, s, pad), flush)
        M = y.shape[0] * y.shape[1] * y.shape[2]
        fl = 2.0 * M * cout * (cin // g) * kh * kw
        line = f"{name:42s} M={M:8d} bn={eng.conv_meta['b']['bn']:3d} {ms:8.3f} ms {fl / ms / 1e9:8.1f} TFLOP/s"
        if kh == 1 and kw == 1 and g == 1:
            x2, w2, b2 = x.reshape(-1, cin), w.reshape(cout, cin).half().cuda(), bias.half().cuda()
            ms_cublas = _time_ms(lambda: torch.nn.functional.linear(x2, w2, b2), flush)
            line += f" | cuBLAS {ms_cublas:8.3f} ms {fl / ms_cublas / 1e9:8.1f} TFLOP/s"
            del x2, w2, b2
        print(line, flush=True)
        del x, y
    for name, case in EPI_CASES.items():
        if only and not any(o in name for o in only):
            continue
        _epi_case(eng, name, case, flush)


if __name__ == "__main__":
    main()
