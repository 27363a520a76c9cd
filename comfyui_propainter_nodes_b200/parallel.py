"""Multi-GPU execution of the hot path: one process per GPU, ``torch.distributed`` (NCCL over NVLink) for the
exchange steps.  The reference has no distributed code; what shards is dictated by the algorithm (SURVEY.md 8e):

* sub-videos of a long clip are independent units up to halos  -> ``bench.py`` weak scaling: one sub-video per rank,
  no data-path collective;
* inside ONE sub-video (strong scaling, ``inpaint_clip_distributed``):
    RAFT frame pairs are independent          -> contiguous pair ranges per rank, one all-gather of the flows
    flow completion / image propagation       -> recurrent in time: chunks (when there are several) go round-robin
                                                 to ranks, a single chunk is computed redundantly by every rank
    sliding windows of the generator          -> contiguous window ranges per rank, one all-gather of the window
                                                 predictions; the order-dependent uint8 composite then runs on every
                                                 rank over the gathered predictions (identical result everywhere)

The collective payloads are small next to the compute (flows 2x[T-1,2,H,W] fp32, predictions
[sum l_t,H,W,4] fp16).  Sharding helpers are pure functions so they are covered by world-size-2 ``gloo`` tests on CPU.
"""
from __future__ import annotations

import os
import sys
from typing import List, Sequence, Tuple

import torch
import torch.distributed as dist


def init_engine_comm(engine, group=None) -> None:
    """Create the engine's own NCCL communicator (pp_comm_init): rank 0 makes the ncclUniqueId inside the C library,
    torch.distributed only carries the 128 bytes to the other ranks."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    box = [engine.comm_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(box, src=0, group=group)
    engine.comm_init(box[0], rank, world)


def destroy_engine_comm(engine) -> None:
    engine.comm_destroy()


def shard_range(n: int, world: int, rank: int) -> Tuple[int, int]:
    """Contiguous near-equal split of range(n): returns [lo, hi) of `rank` (earlier ranks get the remainder)."""
    base, rem = divmod(n, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_sizes(n: int, world: int) -> List[int]:
    return [shard_range(n, world, r)[1] - shard_range(n, world, r)[0] for r in range(world)]


def round_robin(n: int, world: int, rank: int) -> List[int]:
    return list(range(rank, n, world))


def all_gather_variable(local: torch.Tensor, sizes: Sequence[int], group=None) -> torch.Tensor:
    """All-gather of tensors whose dim-0 lengths differ per rank (``sizes[r]``); returns their concatenation.

    One collective: shards are padded to the largest length, gathered, and trimmed."""
    world = len(sizes)
    if world == 1:
        return local
    mx = max(sizes)
    pad = torch.zeros((mx,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    pad[: local.shape[0]] = local
    out = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(out, pad.contiguous(), group=group)
    return torch.cat([o[:s] for o, s in zip(out, sizes)], 0)


def window_shards(n_windows: int, world: int) -> List[Tuple[int, int]]:
    return [shard_range(n_windows, world, r) for r in range(world)]


def balanced_ranges(costs: Sequence[float], world: int) -> List[Tuple[int, int]]:
    """Contiguous partition of range(len(costs)) into `world` (possibly empty) ranges minimising the largest range sum
    (exact, dynamic programming over prefix sums).  Used for the sliding windows: they differ in length (6..11 local
    frames, 3..9 reference frames), and the rank with the heaviest share sets the time of the exchange that follows."""
    n = len(costs)
    pre = [0.0]
    for c in costs:
        pre.append(pre[-1] + float(c))
    INF = float("inf")
    # best[k][i] = minimal possible max-load when the first i items are split into k ranges
    best = [[INF] * (n + 1) for _ in range(world + 1)]
    cut = [[0] * (n + 1) for _ in range(world + 1)]
    best[0][0] = 0.0
    for k in range(1, world + 1):
        for i in range(n + 1):
            for j in range(i + 1):
                v = max(best[k - 1][j], pre[i] - pre[j])
                if v < best[k][i]:
                    best[k][i], cut[k][i] = v, j
    out, i = [], n
    for k in range(world, 0, -1):
        j = cut[k][i]
        out.append((j, i))
        i = j
    return out[::-1]


def window_cost(nb, refs) -> float:
    """Relative cost of one sliding window: the transformer / attention / SoftSplit work grows with all t frames, the
    feature propagation, decoder and encoder of new frames with the local ones."""
    return float(len(nb) + len(refs)) + 1.5 * float(len(nb))


def composite_order(schedule) -> Tuple[List[int], List[int]]:
    """Flat (frame id, first-visit flag) lists of the composite, in window order (propainter_inference.py:294-307)."""
    seen, ids, first = set(), [], []
    for nb, _ in schedule:
        for i in nb:
            ids.append(i)
            first.append(0 if i in seen else 1)
            seen.add(i)
    return ids, first


def gather_rows(eng, buf: torch.Tensor, rows: Sequence[int], first_rank: int = 0, group=None) -> torch.Tensor:
    """In-place all-gather of row blocks of `buf` (member m of the rank range owns rows[m] rows): through the engine's
    NCCL communicator (pp_comm_all_gather_rows) when it has one, else through torch.distributed (CPU/gloo tests)."""
    if len(rows) <= 1:
        return buf
    if getattr(eng, "world", 1) > 1:
        return eng.comm_all_gather_rows(buf, rows, first_rank)
    rank = dist.get_rank(group) - first_rank
    lo = sum(rows[:rank])
    buf.copy_(all_gather_variable(buf[lo:lo + rows[rank]].clone(), rows, group))
    return buf


def inpaint_clip_distributed(models, frames, flow_masks, masks_dilated, orig_u8, cfg, group=None) -> torch.Tensor:
    """Strong-scaling pass over ONE clip shared by all ranks of `group`.  Inputs are replicated on every rank
    (reference layouts, see propainter_inference.process_inpainting); returns the composited uint8 frames
    [T,H,W,3] on every rank."""
    from . import propainter_inference as PI

    eng = models.raft_model.engine
    if getattr(eng, "world", 1) > 1:
        world, rank = eng.world, eng.rank
    else:
        world = dist.get_world_size(group) if dist.is_initialized() else 1
        rank = dist.get_rank(group) if dist.is_initialized() else 0
    T = cfg.video_length
    H, W = frames.shape[-2:]
    dev = eng.device
    marks = []          # PP_DIST_TIMING=1: CUDA events between the stages, printed by rank 0

    def mark(name):
        if os.environ.get("PP_DIST_TIMING"):
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            marks.append((name, ev))

    mark("start")
    # ---- RAFT: pairs [lo, hi) need frames [lo, hi]; every rank writes its shard into the full buffers, one
    #      all-gather per direction completes them (fp32: the N-GPU flows equal the 1-GPU flows bit for bit)
    n_pairs = T - 1
    lo, hi = shard_range(n_pairs, world, rank)
    ff = torch.empty(n_pairs, 2, H, W, device=dev, dtype=torch.float32)
    fb = torch.empty_like(ff)
    if hi > lo:
        eng.raft_bidir(frames[0, lo:hi + 1], cfg.raft_iter, out=(ff[lo:hi], fb[lo:hi]), fp32=not cfg.use_half)
    mark("raft")
    sizes = shard_sizes(n_pairs, world)
    gather_rows(eng, ff, sizes, 0, group)
    gather_rows(eng, fb, sizes, 0, group)
    mark("gather_flows")
    dt = torch.float16 if cfg.use_half else torch.float32
    gt = (ff.unsqueeze(0).to(dt), fb.unsqueeze(0).to(dt))

    # ---- recurrent stages (serial in time): see complete_flow_distributed
    pred = complete_flow_distributed(models.flow_model, gt, flow_masks, cfg.subvideo_length, rank, world, group)
    mark("flow_completion")
    uf, um = PI.image_propagation(models.inpaint_model, frames, masks_dilated, pred, cfg)
    mark("image_propagation")

    # ---- generator windows: contiguous ranges; each rank encodes only the frames its windows touch and writes its
    #      predictions into the full buffer, one all-gather completes it
    sched = PI.window_schedule(cfg)
    wranges = balanced_ranges([window_cost(nb, refs) for nb, refs in sched], world)
    wlo, whi = wranges[rank]
    md = masks_dilated[0].to(device=dev, dtype=torch.float32).contiguous()
    wsizes = [sum(len(nb) for nb, _ in sched[a:b]) for a, b in wranges]
    preds = torch.empty(sum(wsizes), H, W, 4, device=dev, dtype=torch.float16)
    if whi > wlo:
        need = sorted({i for nb, refs in sched[wlo:whi] for i in list(nb) + list(refs)})
        eng.gen_begin(uf[0], md, um[0], pred[0][0], pred[1][0], frames_needed=need)
        try:
            o = sum(wsizes[:rank])
            preds[o:o + wsizes[rank]] = eng.gen_run(sched[wlo:whi])
        finally:
            eng.gen_end()
    mark("generator_windows")
    gather_rows(eng, preds, wsizes, 0, group)
    mark("gather_predictions")

    ids, first = composite_order(sched)
    ids_dev = torch.tensor(ids, dtype=torch.int32, device=dev)
    first_dev = torch.tensor(first, dtype=torch.int32, device=dev)
    orig = orig_u8.to(dev).contiguous()
    comp = torch.zeros_like(orig)
    o = 0
    for nb, _ in sched:
        n = len(nb)
        eng.composite(preds[o:o + n], md, orig, comp, ids_dev[o:o + n], first_dev[o:o + n], cfg.use_half)
        o += n
    mark("composite")
    if marks and rank == 0:
        torch.cuda.synchronize()
        print("[dist timing, rank 0, ms] " + " ".join(f"{b[0]}={a[1].elapsed_time(b[1]):.2f}" for a, b in zip(marks, marks[1:])),
              file=sys.stderr, flush=True)
    return comp


def flow_chunks(n_flows: int, subvideo_length: int, pad: int = 5):
    """The reference's chunking of complete_flow (propainter_inference.py:115-139): [(f0, f1, s, e)] = flows [f0, f1)
    are produced from the padded range [s, e) (masks [s, e])."""
    if n_flows <= subvideo_length:
        return [(0, n_flows, 0, n_flows)]
    out = []
    for f in range(0, n_flows, subvideo_length):
        f1 = min(n_flows, f + subvideo_length)
        out.append((f, f1, max(0, f - pad), min(n_flows, f1 + pad)))
    return out


def flow_teams(n_chunks: int, world: int):
    """Ranks -> teams for flow completion: as many chunks in flight as possible (the recurrence inside a chunk is
    serial, so chunk-level parallelism comes first), the ranks of a team then split directions and frames of ONE
    chunk.  Returns (n_teams, team_size); team k = ranks [k*team_size, (k+1)*team_size), left-over ranks idle."""
    n_teams = max(1, min(n_chunks, world))
    return n_teams, world // n_teams


def complete_flow_distributed(flow_model, flows_bi, flow_masks, subvideo_length, rank, world, group=None):
    """Flow completion of one clip on `world` ranks (every rank holds the full inputs, every rank gets the full
    result).  The recurrence is serial in time, so what shards is (a) the independent sub-video chunks -> teams of
    ranks, (b) inside a chunk the two direction passes and the per-frame encoder / decoder (pp_flow_complete_dist).
    Exchange: the in-team all-gathers of the C call, then one all-gather of the chunks between teams.  The precision
    follows the flows' dtype as in propainter_inference.complete_flow, so the N-GPU result equals the 1-GPU one."""
    eng = flow_model.engine
    ff, fb, fm = flows_bi[0][0], flows_bi[1][0], flow_masks[0]
    dt = flows_bi[0].dtype
    fp32 = dt == torch.float32
    L = ff.shape[0]
    if getattr(eng, "world", 1) <= 1:      # no engine communicator (CPU/gloo logic tests): every rank computes all
        from . import propainter_inference as PI
        return PI.complete_flow(flow_model, flows_bi, flow_masks, subvideo_length)
    chunks = flow_chunks(L, subvideo_length)
    n_teams, tsize = flow_teams(len(chunks), world)
    team = rank // tsize if rank < n_teams * tsize else -1
    of = torch.empty(L, 2, ff.shape[-2], ff.shape[-1], device=eng.device, dtype=torch.float32)
    ob = torch.empty_like(of)
    ff32, fb32, fm32 = eng._f32(ff), eng._f32(fb), eng._f32(fm)
    for r0 in range(0, len(chunks), n_teams):
        ci = r0 + team
        if team < 0 or ci >= len(chunks):
            continue
        f0, f1, s, e = chunks[ci]
        a, b = eng.flow_complete_dist(ff32[s:e], fb32[s:e], fm32[s:e + 1], team * tsize, tsize, fp32=fp32)
        of[f0:f1] = a[f0 - s:f1 - s]
        ob[f0:f1] = b[f0 - s:f1 - s]
    if n_teams > 1 or n_teams * tsize < world:
        # chunk ci lives on every rank of team ci % n_teams; its first rank feeds the others
        # one gather per round: in round r team k's leader owns chunk r*n_teams + k
        for r0 in range(0, len(chunks), n_teams):
            rows = [0] * world
            for k in range(n_teams):
                if r0 + k < len(chunks):
                    f0, f1, _, _ = chunks[r0 + k]
                    rows[k * tsize] = f1 - f0
            # blocks of one round are consecutive chunks: cumulative placement relative to the round's first row
            base = chunks[r0][0]
            n_rows = sum(rows)
            for t in (of, ob):
                view = t[base:base + n_rows]
                eng.comm_all_gather_rows(view, rows, 0)
    return of.unsqueeze(0).to(dt), ob.unsqueeze(0).to(dt)
