"""Backward tracking and dense mode: one pass per direction / offset against grouped passes with frame maps.

    python scripts/backward_bench.py [--reps 5] [--only NAME]

Seeded offline-model weights, seeded texture clips (cotracker_b200.synthetic) as float32 on the device.  Each workload
times whole CoTrackerPredictor calls between device synchronisations (wall clock), alternating the two variants after
one warm-up call of each.  The warm-up call starts without the model's cached update-loop workspace and gives the
variant's peak memory (torch.cuda.max_memory_allocated over the call, the device clip included):
  sequential: the previous path -- the clip encoded once, one update-loop pass for the forward queries and, for backward
              tracking, one on the pyramid reversed in place (restored afterwards); dense mode runs that per offset;
  grouped   : CoTrackerPredictor as it is -- forward and reversed queries as groups of one pass (frame maps), every
              dense offset a group, in the passes plan_dense_passes chooses for the free memory.
Workloads:
  bwd_grid10 / bwd_grid80 : 50 x 720 x 1296, grid 10 / 80 queried at frame T/2, backward_tracking=True
  dense / dense_bwd       : 8 x 160 x 224, dense mode (4 offsets of 80 x 56 tracks), without / with backward tracking
  headline_bwd            : bench.py's clip (16 x 512 x 512, grid 80) with backward_tracking=True
Prints the card's name, power limit and max SM clock, then one line per variant: median and min ms, peak MiB, and
whether the outputs are bit-identical to the sequential variant; exits non-zero if any are not.
"""
from __future__ import annotations

import argparse
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cotracker_b200.predictor import CoTrackerPredictor, _EncodedClip  # noqa: E402
from cotracker_b200.synthetic import seeded_state_dict, texture_video  # noqa: E402

DEV = "cuda:0"


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0) + " (nvidia-smi failed)"


def sequential_sparse(p, clip, video_shape, grid_size, grid_query_frame, queries=None, backward=True):
    q = p._model_queries(clip, video_shape, queries, None, grid_size, False, grid_query_frame)
    m, T = p.model, clip.T
    fwd = m._track_pyramid(clip.pyr, T, clip.H, clip.W, q, clip.ITERS, [q.shape[1]])[:2]
    bwd = None
    if backward:
        inv = q.clone()
        inv[:, :, 0] = T - inv[:, :, 0] - 1
        m._reverse_clip_pyramid_(clip.pyr, T, clip.H, clip.W)
        bwd = m._track_pyramid(clip.pyr, T, clip.H, clip.W, inv, clip.ITERS, [q.shape[1]])[:2]
        m._reverse_clip_pyramid_(clip.pyr, T, clip.H, clip.W)
    return p._finish(q, fwd, bwd, video_shape)


def sequential(p, video, grid_size=0, grid_query_frame=0, backward_tracking=False):
    clip = _EncodedClip(p.model, video, p.interp_shape)
    if grid_size > 0:
        return sequential_sparse(p, clip, video.shape, grid_size, grid_query_frame, backward=backward_tracking)
    H, W = video.shape[3:]
    step = W // 80
    gw, gh = W // step, H // step
    base_x = (torch.arange(gw, device=DEV).repeat(gh) * step).float()
    base_y = (torch.arange(gh, device=DEV).repeat_interleave(gw) * step).float()
    tracks, vis = [], []
    for offset in range(step * step):
        pts = torch.zeros(1, gw * gh, 3, device=DEV)
        pts[:, :, 0] = grid_query_frame
        pts[:, :, 1] = base_x + offset % step
        pts[:, :, 2] = base_y + offset // step
        t, v = sequential_sparse(p, clip, video.shape, 0, grid_query_frame, queries=pts, backward=backward_tracking)
        tracks.append(t)
        vis.append(v)
    return torch.cat(tracks, dim=2), torch.cat(vis, dim=2)


WORKLOADS = {
    "bwd_grid10": ((50, 720, 1296), dict(grid_size=10, grid_query_frame=25, backward_tracking=True)),
    "bwd_grid80": ((50, 720, 1296), dict(grid_size=80, grid_query_frame=25, backward_tracking=True)),
    "dense": ((8, 160, 224), dict(grid_query_frame=0, backward_tracking=False)),
    "dense_bwd": ((8, 160, 224), dict(grid_query_frame=7, backward_tracking=True)),
    "headline_bwd": ((16, 512, 512), dict(grid_size=80, grid_query_frame=0, backward_tracking=True)),
}


def timed(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t0) * 1e3, torch.cuda.max_memory_allocated() / 2 ** 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--only", action="append", default=[], choices=sorted(WORKLOADS))
    args = ap.parse_args()
    print(card(), flush=True)
    p = CoTrackerPredictor(checkpoint=None, window_len=60)
    p.model.load_state_dict(seeded_state_dict(7, offline=True, window_len=60, head_gain=10.0, vis_gain=100.0))
    p = p.to(DEV)
    ok = True
    for name, ((T, H, W), kw) in WORKLOADS.items():
        if args.only and name not in args.only:
            continue
        video = texture_video(T, H, W, seed=T).to(DEV)
        variants = {"sequential": lambda: sequential(p, video, **kw), "grouped": lambda: p(video, **kw)}
        ms = {k: [] for k in variants}
        peak = {}
        outs = {}
        with torch.no_grad():
            for k, fn in variants.items():
                # peak memory from an untimed call that starts without the model's cached update-loop workspace (it only
                # grows, so otherwise the larger variant's workspace would count against the other one too)
                p.model._ws.buf = None
                torch.cuda.empty_cache()
                outs[k], _, peak[k] = timed(fn)
            for _ in range(args.reps):
                for k, fn in variants.items():
                    ms[k].append(timed(fn)[1])
        ref = outs["sequential"]
        for k in variants:
            same = all(torch.equal(a, b) for a, b in zip(outs[k], ref))
            ok &= same
            print(f"{name:13s} {k:10s} median {statistics.median(ms[k]):9.1f} ms  min {min(ms[k]):9.1f} ms  "
                  f"peak {peak[k]:8.0f} MiB  bit-identical {same}", flush=True)
        del video, outs, ref
        torch.cuda.empty_cache()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
