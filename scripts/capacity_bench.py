"""Capacity of the offline update loop in track slabs (ct3_loop_shape.slab_tracks, DESIGN.md §4.4.5).

    python scripts/capacity_bench.py [--reps 3] [--frames 16 48 120] [--long 300] [--out DIR]

Seeded weights and seeded 512 x 512 texture clips (cotracker_b200.synthetic), CoTrackerPredictor (offline model),
grid_size = 80 (6400 tracks), 6 iterations.
  (a) at sizes that fit without slabs (--frames): the call without slabs against pass budgets that force 2, 4 and 16
      slabs (the budget is the slabbed workspace at ceil(N / k) tracks per slab).  The four variants alternate within
      this process, --reps rounds after one warm-up call of each; each call ends in a device synchronise.  Reported:
      median ms per call, points*frames/s, peak memory (torch.cuda.max_memory_allocated over the call, the model's
      cached workspace dropped before it), and whether tracks and visibility are torch.equal to the unslabbed call.
      At the middle length the per-category kernel times of one call (engine.profile_read) are recorded too.
  (b) beyond the full workspace's limit (--long frames): one call with the real pass budget; time, peak memory and
      the slab size the budget chose.
Prints the card's name, power limit and max SM clock first, then one JSON line per measurement; writes them all to
DIR/capacity.json when --out is given.  Exits non-zero if any slabbed output differs.  Fails without a GPU.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import cotracker_b200.model as M  # noqa: E402
from cotracker_b200 import engine  # noqa: E402
from cotracker_b200.predictor import CoTrackerPredictor  # noqa: E402
from cotracker_b200.synthetic import seeded_state_dict, texture_video  # noqa: E402

DEV = "cuda:0"
GRID, SIZE, ITERS = 80, 512, 6
SLAB_COUNTS = (1, 2, 4, 16)   # 1: no slabs


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    return out


class ForcedSlabs:
    """Replaces the pass budget of model._refine by the slabbed workspace at ceil(N / k) tracks per slab (k = 1: the
    real budget), and records the slab_tracks each call ran with."""

    def __init__(self):
        self.k = 1
        self.used = []
        self.real = M.slab_tracks_for
        M.slab_tracks_for = self

    def __call__(self, T, N, G, H4, W4, frames, budget):
        if self.k > 1:
            budget = engine.workspace_bytes(T, N, H4, W4, G, frames, slab_tracks=math.ceil(N / self.k))
        s = self.real(T, N, G, H4, W4, frames, budget)
        self.used.append(s)
        return s


def timed_call(p, video, forced, k):
    forced.k = k
    forced.used.clear()
    p.model._ws.buf = None
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    with torch.no_grad():
        tr, vi = p(video, grid_size=GRID)
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3
    return (tr, vi), ms, torch.cuda.max_memory_allocated() / 2 ** 20, list(forced.used)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--frames", type=int, nargs="+", default=[16, 48, 120])
    ap.add_argument("--long", type=int, default=300)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "capacity_bench needs a GPU"
    rows = [{"card": card()}]
    print(json.dumps(rows[0]), flush=True)
    p = CoTrackerPredictor(checkpoint=None, window_len=60)
    p.model.load_state_dict(seeded_state_dict(1234, offline=True, window_len=60, head_gain=1.0, vis_gain=1.0))
    p = p.to(DEV)
    forced = ForcedSlabs()
    ok = True
    N = GRID * GRID
    for T in args.frames:
        video = texture_video(T, SIZE, SIZE, seed=0).to(DEV)
        ref = {}
        times = {k: [] for k in SLAB_COUNTS}
        peaks, slabs = {}, {}
        for k in SLAB_COUNTS:                                       # warm-up, and the outputs to compare
            ref[k], _, peaks[k], slabs[k] = timed_call(p, video, forced, k)
        for _ in range(args.reps):
            for k in SLAB_COUNTS:
                out, ms, peak, _ = timed_call(p, video, forced, k)
                times[k].append(ms)
                peaks[k] = max(peaks[k], peak)
        for k in SLAB_COUNTS:
            same = torch.equal(ref[k][0], ref[1][0]) and torch.equal(ref[k][1], ref[1][1])
            ok &= same
            ms = statistics.median(times[k])
            row = {"case": "a", "T": T, "slabs": k, "slab_tracks": slabs[k][0], "ms": round(ms, 1),
                   "ms_all": [round(t, 1) for t in times[k]], "points_frames_per_s": round(N * T / ms * 1e3),
                   "peak_mib": round(peaks[k]), "equal_to_unslabbed": same}
            rows.append(row)
            print(json.dumps(row), flush=True)
        if T == args.frames[len(args.frames) // 2]:
            for k in (1, 4):
                forced.k = k
                engine.profile_enable(True)
                with torch.no_grad():
                    p(video, grid_size=GRID)
                prof = engine.profile_read()
                engine.profile_enable(False)
                row = {"case": "a_profile", "T": T, "slabs": k, "profile": prof}
                rows.append(row)
                print(json.dumps(row, default=str), flush=True)
        del video, ref
    if args.long:
        T = args.long
        video = texture_video(T, SIZE, SIZE, seed=0).to(DEV)
        need = engine.workspace_bytes(T, N, SIZE // 4, SIZE // 4)
        _, ms, peak, used = timed_call(p, video, forced, 1)
        row = {"case": "b", "T": T, "ms": round(ms, 1), "points_frames_per_s": round(N * T / ms * 1e3),
               "peak_mib": round(peak), "slab_tracks": used, "full_workspace_mib": round(need / 2 ** 20),
               "device_mib": round(torch.cuda.get_device_properties(0).total_memory / 2 ** 20)}
        rows.append(row)
        print(json.dumps(row), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "capacity.json"), "w") as f:
            json.dump(rows, f, indent=1, default=str)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
