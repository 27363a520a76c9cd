"""Multi-GPU correctness check (run under torchrun, one rank per GPU):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29511 \
        tools/dist_check.py [T H W subvideo_length [fp16]]

Every rank runs the sharded clip (parallel.inpaint_clip_distributed: RAFT pairs, flow-completion teams / directions /
frames, generator windows, NCCL exchanges through pp_comm_*); rank 0 also runs the plain single-GPU path and compares
the uint8 frames and the completed flows.  fp16 is the node's switch ("enable", default; "disable" runs RAFT, flow
completion and image propagation at fp32 accuracy).  Prints one JSON line on rank 0; exit code 1 on mismatch."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.distributed as dist


def main():
    from comfyui_propainter_nodes_b200 import weights as Wt, parallel as PAR, propainter_inference as PI
    from comfyui_propainter_nodes_b200.synthetic import synthetic_clip, synthetic_mask
    from comfyui_propainter_nodes_b200.utils import image_utils as IU, model_utils as MU
    T, H, W, sub = [int(x) for x in (sys.argv[1:5] + [20, 128, 160, 80][len(sys.argv) - 1:])[:4]]
    fp16 = sys.argv[5] if len(sys.argv) > 5 else "enable"
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    rank, world = dist.get_rank(), dist.get_world_size()
    models = MU.build_models(dev, Wt.synthetic_raft_state_dict(), Wt.synthetic_rfc_state_dict(),
                             Wt.synthetic_generator_state_dict(), workspace_gb=24.0)
    eng = models.raft_model.engine
    PAR.init_engine_comm(eng)
    icfg = IU.ImageConfig(W, H, 5, 8, (W, H), T)
    ft, fm, md, orig = IU.prepare_frames_and_masks(IU.convert_image_to_frames(synthetic_clip(T, H, W, 5)),
                                                   synthetic_mask(T, H, W), icfg, dev)
    orig_dev = torch.from_numpy(np.stack(orig)).to(dev)
    cfg = PI.ProPainterConfig(4, 6, sub, 3, fp16, T, dev, icfg.process_size)
    comp = PAR.inpaint_clip_distributed(models, ft, fm, md, orig_dev, cfg)
    # flows of the distributed path, separately (collective)
    gt = PI.compute_flow(models.raft_model, ft, cfg)
    dt = torch.float16 if cfg.use_half else torch.float32       # what process_inpainting hands complete_flow
    gt = (gt[0].to(dt), gt[1].to(dt))
    pd = PAR.complete_flow_distributed(models.flow_model, gt, fm.to(dt), sub, rank, world)
    torch.cuda.synchronize()
    ok = True
    if rank == 0:
        uf, um, pf = PI.process_inpainting(models, ft, fm, md, cfg)
        ref = PI.feature_propagation_device(models.inpaint_model, uf, um, md, pf, orig_dev, cfg)
        torch.cuda.synchronize()
        rec = dict(world=world, T=T, H=H, W=W, subvideo_length=sub, fp16=fp16,
                   frames_mismatch=int((comp != ref).sum().item()),
                   flow_f_max_abs=float((pd[0].float() - pf[0].float()).abs().max()),
                   flow_b_max_abs=float((pd[1].float() - pf[1].float()).abs().max()))
        ok = rec["frames_mismatch"] == 0 and rec["flow_f_max_abs"] == 0.0 and rec["flow_b_max_abs"] == 0.0
        rec["ok"] = ok
        print(json.dumps(rec), flush=True)
    # all ranks must hold the same result
    chk = comp.to(torch.float32).sum().reshape(1)
    lst = [torch.zeros_like(chk) for _ in range(world)]
    dist.all_gather(lst, chk)
    same = all(float(x) == float(lst[0]) for x in lst)
    if rank == 0 and not same:
        print(json.dumps({"ranks_agree": False}), flush=True)
    PAR.destroy_engine_comm(eng)
    dist.destroy_process_group()
    sys.exit(0 if (ok and same) else 1)


if __name__ == "__main__":
    main()
