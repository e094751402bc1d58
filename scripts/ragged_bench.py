#!/usr/bin/env python
"""Clips of different lengths through CoTrackerPredictor: list calls under a sweep of padding bounds against one call
per clip, alternated in one process after a warm-up, each in windows of at least --window seconds that end in a device
synchronise.  Reports clips/s, update-loop passes and peak device memory of each way, checks that every way gives
torch.equal outputs, and reads the card's name and power limit in the same run.

    python scripts/ragged_bench.py [--rounds 3] [--window 1.0] [--out FILE.json]

A bound (f, r) lets a pass pad while its padded token rows stay within f times the real ones plus r
(`plan_ragged_passes`); (0, 0) is the list split into same-length passes, in one call with one encoder pass.
Mixes (synthetic seeded weights, 512x512 uint8 clips with lengths spread over 16-64 frames; 720x1296 clips at the
50 frames of the apple clip): 8 clips at grid 10, 32 clips at grid 10, 8 clips at grid 30, 4 clips 720x1296 at grid 10.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

MIXES = [("8x512_grid10", 8, (512, 512), 10, "spread"), ("32x512_grid10", 32, (512, 512), 10, "spread"),
         ("8x512_grid30", 8, (512, 512), 30, "spread"), ("4x720x1296_grid10", 4, (720, 1296), 10, "apple")]
BOUNDS = [(0.0, 0), (0.1, 0), (0.25, 0), (0.5, 0), (1.0, 0), (0.0, 1 << 14), (0.0, 1 << 16), (0.0, 1 << 18)]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def clips_for(n, hw, kind, seed):
    from cotracker_b200.synthetic import texture_video
    g = torch.Generator().manual_seed(seed)
    lengths = [50] * n if kind == "apple" else torch.randint(16, 65, (n,), generator=g).tolist()
    return [texture_video(T, hw[0], hw[1], seed=seed + b).to("cuda") for b, T in enumerate(lengths)]


def ways(p, clips, grid, passes):
    import cotracker_b200.predictor as P

    def per_clip():
        out = [p(c, grid_size=grid) for c in clips]
        return [o[0] for o in out], [o[1] for o in out]

    def list_call(frac, rows):
        def run():
            P.RAGGED_PAD_FRACTION, P.RAGGED_PAD_ROWS = frac, rows
            return p(clips, grid_size=grid)
        return run

    out = {"per_clip": per_clip}
    for frac, rows in BOUNDS:
        out[f"list f={frac} r={rows}"] = list_call(frac, rows)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--window", type=float, default=1.0)
    ap.add_argument("--out", default=None)
    ap.add_argument("--mix", action="append", default=None, help="run only these mixes (names as in MIXES)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ragged_bench.py measures on the GPU; none is available")
    from cotracker_b200.predictor import CoTrackerPredictor
    from cotracker_b200.synthetic import seeded_state_dict
    p = CoTrackerPredictor(checkpoint=None, window_len=60)
    p.model.load_state_dict(seeded_state_dict(1234, offline=True, window_len=60))
    p = p.cuda()
    import cotracker_b200.predictor as P
    plan = P.plan_ragged_passes
    passes = []

    def counting_plan(*args, **kw):
        out = plan(*args, **kw)
        passes.append(len(out))
        return out

    P.plan_ragged_passes = counting_plan
    result = {"card": card(), "mixes": {}}
    for name, n, hw, grid, kind in MIXES:
        if a.mix and name not in a.mix:
            continue
        clips = clips_for(n, hw, kind, seed=17)
        fns = ways(p, clips, grid, passes)
        outs, n_passes = {}, {}
        for k, f in fns.items():   # warm-up of every shape, the outputs compared, the passes of each bound
            passes.clear()
            outs[k] = f()
            n_passes[k] = passes[0] if passes else len(clips)
        ref = outs["per_clip"]
        identical = all(len(o[0]) == len(ref[0]) and all(torch.equal(x, y) for x, y in zip(o[0], ref[0]))
                        and all(torch.equal(x, y) for x, y in zip(o[1], ref[1])) for o in outs.values())
        del outs, ref
        rates = {k: [] for k in fns}
        peak = {k: 0 for k in fns}
        for _ in range(a.rounds):
            for k, f in fns.items():
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                t0, calls = time.perf_counter(), 0
                while True:
                    f()
                    calls += 1
                    torch.cuda.synchronize()
                    dt = time.perf_counter() - t0
                    if dt >= a.window:
                        break
                rates[k].append(calls * n / dt)
                peak[k] = max(peak[k], torch.cuda.max_memory_allocated())
        lengths = [c.shape[1] for c in clips]
        result["mixes"][name] = {
            "clips": n, "hw": list(hw), "grid": grid, "lengths": lengths, "identical": identical, "passes": n_passes,
            "clips_per_s": {k: sorted(v) for k, v in rates.items()},
            "peak_gib": {k: round(v / 2 ** 30, 2) for k, v in peak.items()}}
        print(name, json.dumps(result["mixes"][name]), flush=True)
        del clips
        torch.cuda.empty_cache()
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
