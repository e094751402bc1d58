"""Long online streams, bounded (`history=16`) against unbounded (DESIGN.md 4.4.4).

K streams of a G x G grid on one `OnlineStreams` hub, every stream advancing each step, for `--steps` steps: 512x512
uint8 device frames, window_len 16 (8 new frames per stream and step), seeded weights.  For each (grid, K) the
bounded hub runs first, then the unbounded one (`--order unbounded-first` swaps them), after a warm-up hub has run
the shapes.  Around steps 10, 100 and `--steps` (or the checkpoints given), five consecutive steps are timed one by
one with CUDA events and the median is kept; results are dropped each step.  `memory_allocated` is read after each
checkpoint step (results dropped) and `max_memory_allocated` over the run, both relative to the allocation before the
hub opened.  Prints one JSON line per (grid, K, mode) with the card's name and power limit read in the same run.

    python scripts/long_stream_bench.py [--steps 1000] [--grids 10 50] [--ks 1 4 16] [--out long_stream_bench.json]
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SIZE, S, STEP, PERIOD = 512, 16, 8, 64


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, power = (x.strip() for x in q.split(","))
    return {"gpu": name, "power_limit": power}


def run(p, loops, K, G, history, steps, checkpoints):
    """One hub of K streams run for `steps` steps.  -> {checkpoint: (median ms, memory_allocated)}, peak."""
    from cotracker_b200.streams import OnlineStreams
    gc.collect()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    hub = OnlineStreams(p)
    ids = [hub.open(frame_size=(SIZE, SIZE), grid_size=G, history=history) for _ in range(K)]
    timed = {c: range(max(1, c - 2), c + 3) for c in checkpoints}
    want = {s for r in timed.values() for s in r}
    ms, mem = {}, {}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for i in range(1, max(want) + 1):
        o = STEP * (i - 1) % PERIOD        # the loop video repeats every PERIOD frames, so overlaps stay cached
        for k, sid in enumerate(ids):
            hub.push(sid, loops[k][:, o:o + S])
        if i in want:
            ev[0].record()
        out = hub.step()
        del out
        if i in want:
            ev[1].record()
            torch.cuda.synchronize()
            ms[i] = ev[0].elapsed_time(ev[1])
        for c in checkpoints:
            if i == c:
                torch.cuda.synchronize()
                mem[c] = torch.cuda.memory_allocated() - base
    peak = torch.cuda.max_memory_allocated() - base
    frames = hub.length(ids[0])
    for sid in ids:
        hub.close(sid)
    res = {c: (statistics.median(ms[s] for s in timed[c]), mem[c]) for c in checkpoints}
    return res, peak, frames


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--checkpoints", type=int, nargs="+", default=None)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--grids", type=int, nargs="+", default=[10, 50])
    ap.add_argument("--ks", type=int, nargs="+", default=[1, 4, 16])
    ap.add_argument("--history", type=int, default=16)
    ap.add_argument("--order", choices=["bounded-first", "unbounded-first"], default="bounded-first")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from cotracker_b200.predictor import CoTrackerOnlinePredictor
    from cotracker_b200.synthetic import seeded_state_dict, texture_video
    assert torch.cuda.is_available(), "long_stream_bench.py measures on a GPU"
    info = card()
    checkpoints = sorted(set(args.checkpoints or [10, 100, args.steps]))
    p = CoTrackerOnlinePredictor(checkpoint=None, window_len=S)
    p.model.load_state_dict(seeded_state_dict(1234, offline=False, window_len=S))
    p = p.to("cuda")
    loops = []
    for k in range(max(args.ks)):
        v = texture_video(PERIOD, SIZE, SIZE, seed=k).to(torch.uint8).cuda()
        loops.append(torch.cat([v, v[:, :S]], 1))
    rows = []
    for G in args.grids:
        for K in args.ks:
            run(p, loops, K, G, args.history, args.warmup, [args.warmup])      # warm-up: every shape of the run
            modes = (args.history, None) if args.order == "bounded-first" else (None, args.history)
            for history in modes:
                res, peak, frames = run(p, loops, K, G, history, max(checkpoints), checkpoints)
                for c, (t, m) in res.items():
                    row = dict(grid=G, K=K, history=history, step=c, frames=STEP * c + STEP, ms_per_step=round(t, 3),
                               memory_allocated_mb=round(m / 2 ** 20, 1), **info)
                    rows.append(row)
                    print(json.dumps(row), flush=True)
                row = dict(grid=G, K=K, history=history, steps=max(checkpoints), frames=frames,
                           max_memory_allocated_mb=round(peak / 2 ** 20, 1), **info)
                rows.append(row)
                print(json.dumps(row), flush=True)
                torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
