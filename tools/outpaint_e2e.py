"""End-to-end time of the Outpaint node (host IMAGE in, host IMAGE out) and of its pre-processing alone, at the inputs
users feed it: 80-frame 1280x720 and 1920x1080 clips with the default widgets (width=640, height=360, width_scale=1.2:
resized to 640x360 on a 768x360 canvas), and a 640x360 clip, which needs no resize.

Each number is a host clock around one node call that ends in a device synchronise; the median of --calls calls after
--warmup warm-up calls.  "preprocess" is the same node call with the pipeline (propainter_nodes._run) replaced by a
device synchronise: everything the node does before RAFT, uploads included.  Seeded synthetic weights and uniform random
frames (the pipeline's time does not depend on the content).  --root times the package of another checkout of this
repository, built in place (an A/B against an older build: run both alternately in one session).

Prints one JSON line per input, then one with the card's name and power limit."""
import argparse
import contextlib
import json
import os
import statistics
import subprocess
import sys
import time

INPUTS = (("1280x720", 720, 1280), ("1920x1080", 1080, 1920), ("640x360", 360, 640))
WIDGETS = dict(width=640, height=360, width_scale=1.2, height_scale=1.0, mask_dilates=5, flow_mask_dilates=8,
               ref_stride=10, neighbor_length=10, subvideo_length=80, raft_iter=20, fp16="enable")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                    help="checkout whose package is timed (default: this one)")
    ap.add_argument("--frames", type=int, default=80)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--calls", type=int, default=3)
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    import torch
    from comfyui_propainter_nodes_b200 import propainter_nodes as PN
    from comfyui_propainter_nodes_b200 import weights as Wt
    from comfyui_propainter_nodes_b200.utils import model_utils as MU

    if not torch.cuda.is_available():
        sys.exit("outpaint_e2e: needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    models = MU.build_models(dev, Wt.synthetic_raft_state_dict(), Wt.synthetic_rfc_state_dict(),
                             Wt.synthetic_generator_state_dict())       # arena sized per clip, as in the node
    MU.set_resident_models(dev, models)
    node = PN.ProPainterOutpaint()
    run = PN._run

    def preprocess_only(models, ft, fm, md, orig, cfg):
        torch.cuda.synchronize()
        return None, fm.squeeze(), None

    def median_ms(image):
        times = []
        for i in range(args.warmup + args.calls):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            with contextlib.redirect_stdout(sys.stderr):
                out = node.propainter_outpainting(image, **WIDGETS)
            torch.cuda.synchronize()
            if i >= args.warmup:
                times.append(1e3 * (time.perf_counter() - t0))
            del out
        return round(statistics.median(times), 1), [round(t, 1) for t in times]

    for name, H, W in INPUTS:
        g = torch.Generator().manual_seed(H)
        image = torch.rand(args.frames, H, W, 3, generator=g)
        PN._run = run
        e2e, e2e_all = median_ms(image)
        PN._run = preprocess_only
        pre, pre_all = median_ms(image)
        PN._run = run
        print(json.dumps({"root": os.path.abspath(args.root), "input": name, "frames": args.frames, "e2e_ms": e2e,
                          "preprocess_ms": pre, "e2e_calls_ms": e2e_all, "preprocess_calls_ms": pre_all}), flush=True)
        del image
    print(json.dumps({"card": card(), "device": torch.cuda.get_device_name(dev)}), flush=True)


if __name__ == "__main__":
    main()
