"""Micro-benchmark of the wgmma implicit-GEMM conv on representative layers (CUDA events, L2 flushed)."""
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


def main():
    only = sys.argv[1:]
    eng = E.Engine("cuda:0", workspace_gb=2.0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda:0")
    for name, (N, H, W, cin, cout, kh, kw, s, g) in CASES.items():
        if only and not any(o in name for o in only):
            continue
        w = torch.randn(cout, cin // g, kh, kw) / math.sqrt(cin * kh * kw)
        eng.register_conv("b", w, torch.zeros(cout), g)
        x = torch.randn(N, H, W, cin, device="cuda:0", dtype=torch.float16)
        if kh != kw:
            x = torch.nn.functional.pad(x, (0, 0, kw // 2, kw // 2, kh // 2, kh // 2)).contiguous()
            pad = 0
        else:
            pad = kh // 2
        for _ in range(3):
            y = eng.op_conv("b", x, s, pad)
        ts = []
        for _ in range(5):
            flush.fill_(0)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            y = eng.op_conv("b", x, s, pad)
            b.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        ms = sorted(ts)[len(ts) // 2]
        M = y.shape[0] * y.shape[1] * y.shape[2]
        fl = 2.0 * M * cout * (cin // g) * kh * kw
        print(f"{name:42s} M={M:8d} bn={eng.conv_meta['b']['bn']:3d} {ms:8.3f} ms {fl / ms / 1e9:8.1f} TFLOP/s", flush=True)


if __name__ == "__main__":
    main()
