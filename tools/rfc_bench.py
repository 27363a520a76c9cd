"""Flow-completion stage alone at the bench size (80 frames 640x360): timing for A/B switches (PP_PROG=0/1), of the two
precisions (fp16 activations / fp32 accuracy, the node's fp16="enable" / "disable"), and a small target for ncu
captures of the propagation-step kernels.

    python tools/rfc_bench.py [T H W reps] [--precision fp16|fp32|both]

With both, the precisions alternate run by run in one process; every line reports the median, the spread, the arena
peak of that precision, and the card with its power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from comfyui_propainter_nodes_b200 import weights as Wt
from comfyui_propainter_nodes_b200.engine import Engine
from comfyui_propainter_nodes_b200.synthetic import synthetic_mask


def _power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("dims", nargs="*", type=int, help="T H W reps (default 80 360 640 5)")
    ap.add_argument("--precision", choices=("fp16", "fp32", "both"), default="fp16")
    a = ap.parse_args()
    T, H, W, reps = (a.dims + [80, 360, 640, 5][len(a.dims):])[:4]
    dev = torch.device("cuda:0")
    eng = Engine(dev, workspace_gb=24.0).load_weights(Wt.synthetic_raft_state_dict(), Wt.synthetic_rfc_state_dict(),
                                                      Wt.synthetic_generator_state_dict())
    g = torch.Generator().manual_seed(0)
    ff = (torch.randn(T - 1, 2, H // 8, W // 8, generator=g) * 2).to(dev)
    ff = torch.nn.functional.interpolate(ff, size=(H, W), mode="bilinear") + 1.5
    fb = -ff
    masks = synthetic_mask(T, H, W)[:, None].contiguous().to(dev)
    precs = {"fp16": [False], "fp32": [True], "both": [False, True]}[a.precision]
    for fp32 in precs:
        for _ in range(2):
            eng.flow_complete(ff, fb, masks, fp32=fp32)
    torch.cuda.synchronize()
    times = {p: [] for p in precs}
    for _ in range(reps):
        for fp32 in precs:
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            eng.flow_complete(ff, fb, masks, fp32=fp32)
            e.record()
            torch.cuda.synchronize()
            times[fp32].append(s.elapsed_time(e))
    card, limit = torch.cuda.get_device_name(dev), _power_limit_w()
    for fp32 in precs:
        eng.set_workspace_bytes(eng.workspace.numel())        # fresh engine arena: its peak is this precision's alone
        l0 = eng.launch_count
        eng.flow_complete(ff, fb, masks, fp32=fp32)
        torch.cuda.synchronize()
        t = sorted(times[fp32])
        print(json.dumps({"T": T, "H": H, "W": W, "precision": "fp32" if fp32 else "fp16",
                          "PP_PROG": os.environ.get("PP_PROG", "1") if not fp32 else "n/a", "ms": t[len(t) // 2],
                          "ms_min": round(t[0], 2), "ms_max": round(t[-1], 2), "ms_all": [round(x, 2) for x in times[fp32]],
                          "launches": eng.launch_count - l0, "workspace_peak_gb": round(eng.workspace_peak / 2 ** 30, 3),
                          "card": card, "power_limit_w": limit}))


if __name__ == "__main__":
    main()
