"""Times RAFT in both precisions of the engine: pp_raft_bidir (fp16 activations, fp32 accumulation; fp16="enable")
and pp_raft_bidir_fp32 (fp32 activations, 3xTF32 GEMMs; fp16="disable").

Workload: the bench's clip (80 synthetic frames at 640x360, raft_iter=20, both directions), bench weights.  Each path
is warmed up once, then timed `--reps` times with CUDA events around the whole call; the arena peak of each path is
read from a fresh engine.  Prints one JSON line including the card name and its power limit.

    python tools/raft_precision_bench.py [--frames 80] [--iters 20] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from comfyui_propainter_nodes_b200 import engine as E            # noqa: E402
from comfyui_propainter_nodes_b200 import weights as Wt          # noqa: E402
from comfyui_propainter_nodes_b200.synthetic import synthetic_clip  # noqa: E402


def power_limit_w():
    """Enforced power limit of GPU 0 in W (read only), or None."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=80)
    ap.add_argument("--height", type=int, default=360)
    ap.add_argument("--width", type=int, default=640)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--workspace-gb", type=float, default=40.0)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    T, H, W = a.frames, a.height, a.width
    frames = (synthetic_clip(T, H, W, 7).permute(0, 3, 1, 2) * 2 - 1).contiguous().to(dev)
    sds = (Wt.synthetic_raft_state_dict(), Wt.synthetic_rfc_state_dict(), Wt.synthetic_generator_state_dict())
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(), "frames": T, "size": [W, H],
           "raft_iter": a.iters, "reps": a.reps}
    out = {}
    for tag, fp32 in (("fp16", False), ("fp32", True)):
        eng = E.Engine(dev, workspace_gb=a.workspace_gb).load_weights(*sds)
        out[tag] = eng.raft_bidir(frames, a.iters, fp32=fp32)                 # warm-up; also the arena peak of one call
        torch.cuda.synchronize()
        peak = eng.workspace_peak
        ms = []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            eng.raft_bidir(frames, a.iters, fp32=fp32)
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        res[tag] = {"ms": [round(v, 2) for v in ms], "ms_min": round(min(ms), 2), "arena_peak_mb": round(peak / 2 ** 20, 1)}
        eng.close()
    res["fp32_over_fp16"] = round(res["fp32"]["ms_min"] / res["fp16"]["ms_min"], 2)
    d = (out["fp32"][0] - out["fp16"][0]).abs()
    res["flow_f_fp16_vs_fp32"] = {"max_abs": float(d.max()), "mean_abs": float(d.mean())}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
