"""Batched tracking: one call on B clips against B calls on one clip each.

    python scripts/batch_bench.py [--seconds 1.0] [--reps 2] [--only NAME] [--batches 1 2 4 8]

Seeded weights and seeded texture clips (cotracker_b200.synthetic), uint8 on the device, every clip of a batch from its
own seed.  Workloads:
  c1_grid10      : CoTrackerPredictor (offline model), 50 x 720 x 1296, grid 10  -- 100 tracks x 50 frames per clip
  c2_grid30      : CoTrackerPredictor (offline model), 16 x 512 x 512, grid 30
  online_grid10  : CoTrackerOnlinePredictor (window 16), 40 x 512 x 512 fed in 4 chunks of 16 frames, grid 10
  online_grid50  : the same with grid 50
For each workload and B, two variants alternate within this process after one warm-up call of each:
  batched    : one predictor call (or one sequence of online steps) on video [B,T,3,H,W];
  sequential : B calls (sequences) on video[b:b+1], one after another.
A timed window repeats the variant until `--seconds` have passed and ends in a device synchronise (wall clock); the
figure is the best window's time per call divided by B.  Peak memory is torch.cuda.max_memory_allocated over the
warm-up call, the device clips included.  Prints the card's name, power limit and max SM clock, then one line per
workload, B and variant: ms per clip, clips/s, peak MiB, and whether the batched outputs are bit-identical to the
sequential ones; exits non-zero if any are not.  Fails without a GPU.
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cotracker_b200.predictor import CoTrackerOnlinePredictor, CoTrackerPredictor  # noqa: E402
from cotracker_b200.synthetic import seeded_state_dict, texture_video  # noqa: E402

DEV = "cuda:0"

WORKLOADS = {   # name -> (online, (T, H, W), grid)
    "c1_grid10": (False, (50, 720, 1296), 10),
    "c2_grid30": (False, (16, 512, 512), 30),
    "online_grid10": (True, (40, 512, 512), 10),
    "online_grid50": (True, (40, 512, 512), 50),
}


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0) + " (nvidia-smi failed)"


def predictor(online):
    cls, S = (CoTrackerOnlinePredictor, 16) if online else (CoTrackerPredictor, 60)
    p = cls(checkpoint=None, window_len=S)
    p.model.load_state_dict(seeded_state_dict(7, offline=not online, window_len=S, head_gain=10.0, vis_gain=100.0))
    return p.to(DEV)


def track(p, online, video, grid):
    """One whole tracking job on video [b,T,3,H,W] -> (tracks, visibility) of the last call."""
    if not online:
        return p(video, grid_size=grid)
    p(video_chunk=video, is_first_step=True, grid_size=grid)
    for ind in range(0, video.shape[1] - p.step, p.step):
        out = p(video_chunk=video[:, ind:ind + 2 * p.step])
    return out


def window(fn, seconds):
    """Repeat fn for at least `seconds`, synchronise, -> seconds per call."""
    torch.cuda.synchronize()
    n, t0 = 0, time.perf_counter()
    while True:
        fn()
        n += 1
        if time.perf_counter() - t0 >= seconds:
            break
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--only", action="append", default=[], choices=sorted(WORKLOADS))
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 2, 4, 8])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("batch_bench.py needs a GPU")
    print(card(), flush=True)
    ok = True
    for name, (online, (T, H, W), grid) in WORKLOADS.items():
        if args.only and name not in args.only:
            continue
        p = predictor(online)
        for B in args.batches:
            video = torch.cat([texture_video(T, H, W, seed=1000 + b, shift=(1 + b % 3, 2)) for b in range(B)])
            video = video.to(torch.uint8).to(DEV)
            variants = {
                "batched": lambda: track(p, online, video, grid),
                "sequential": lambda: [track(p, online, video[b:b + 1], grid) for b in range(B)][-1],
            }
            peak, best = {}, {k: float("inf") for k in variants}
            with torch.no_grad():
                for k, fn in variants.items():
                    p.model._ws.buf = None          # the cached workspace only grows: each variant starts without it
                    torch.cuda.empty_cache()
                    torch.cuda.synchronize()
                    torch.cuda.reset_peak_memory_stats()
                    fn()
                    torch.cuda.synchronize()
                    peak[k] = torch.cuda.max_memory_allocated() / 2 ** 20
                got = track(p, online, video, grid)
                same = all(torch.equal(g[b:b + 1], w) for b in range(B)
                           for g, w in zip(got, track(p, online, video[b:b + 1], grid)))
                ok &= same
                for _ in range(args.reps):
                    for k, fn in variants.items():
                        best[k] = min(best[k], window(fn, args.seconds))
            for k in variants:
                per_clip = best[k] / B
                print(f"{name:14s} B {B}  {k:10s} {per_clip * 1e3:9.2f} ms/clip  {1.0 / per_clip:8.2f} clips/s  "
                      f"peak {peak[k]:8.0f} MiB  bit-identical {same}", flush=True)
            del video, got
            torch.cuda.empty_cache()
        del p
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
