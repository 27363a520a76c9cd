"""Image-propagation stage alone at the bench size (80 frames 640x360) in both precisions: fp16 storage
(fp16="enable") and fp32 (fp16="disable", pp_image_propagate_fp32).  Prints one JSON line.

    python tools/imgprop_bench.py [T H W reps]
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from comfyui_propainter_nodes_b200.engine import Engine
from comfyui_propainter_nodes_b200.synthetic import synthetic_clip, synthetic_mask


def main():
    T, H, W, reps = [int(x) for x in (sys.argv[1:5] + [80, 360, 640, 7][len(sys.argv) - 1:])]
    dev = torch.device("cuda:0")
    eng = Engine(dev, workspace_gb=8.0)
    g = torch.Generator().manual_seed(0)
    ff = (torch.randn(T - 1, 2, H // 8, W // 8, generator=g) * 2).to(dev)
    ff = torch.nn.functional.interpolate(ff, size=(H, W), mode="bilinear") + 1.5
    fb = -ff
    frames = (synthetic_clip(T, H, W, 1).permute(0, 3, 1, 2) * 2 - 1).contiguous().to(dev)
    masks = synthetic_mask(T, H, W)[:, None].contiguous().to(dev)
    out = {"T": T, "H": H, "W": W}
    for fp32 in (False, True, False, True):              # alternated, so clock drift does not favour one precision
        for _ in range(2):
            eng.image_propagate(frames, masks, ff, fb, fp32=fp32)
        torch.cuda.synchronize()
        times = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            eng.image_propagate(frames, masks, ff, fb, fp32=fp32)
            b.record()
            torch.cuda.synchronize()
            times.append(a.elapsed_time(b))
        out.setdefault("fp32_ms" if fp32 else "fp16_ms", []).append(round(sorted(times)[len(times) // 2], 3))
    out["workspace_peak_bytes"] = eng.workspace_peak
    print(json.dumps(out))


if __name__ == "__main__":
    main()
