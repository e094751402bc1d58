"""What `return_scores=True` costs (DESIGN.md 4.11): the headline offline call (512x512x16 device clip, grid_size=80,
6400 tracks) and one step of an 8-stream hub (512x512 uint8 device chunks, window_len 16, grid_size=50 per stream),
each with and without the scores, alternating in one process so that both see the same clocks and neighbours.

Every variant is warmed up first.  Each repetition times `--calls` calls of one variant with CUDA events, the clip or
chunks already on the device, ending in a device synchronise; the variants alternate for `--reps` repetitions and the
median per call is reported.  Seeded weights.  Prints one JSON line per workload with ms per call of both variants, the
difference, and the card's name and power limit read in the same run.

    python scripts/scores_bench.py [--reps 7] [--calls 5] [--out scores_bench.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SIZE, S, STEP = 512, 16, 8


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, power = (x.strip() for x in q.split(","))
    return {"gpu": name, "power_limit": power}


def timed(fn, calls):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / calls


def alternate(variants, reps, calls):
    """{name: median ms per call} of the variants, timed in turn `reps` times."""
    for fn in variants.values():   # warm-up: every shape and code path of both variants
        fn()
        fn()
    times = {k: [] for k in variants}
    for _ in range(reps):
        for k, fn in variants.items():
            times[k].append(timed(fn, calls))
    return {k: statistics.median(v) for k, v in times.items()}


def offline(sd, reps, calls):
    from cotracker_b200.predictor import CoTrackerPredictor
    from cotracker_b200.synthetic import texture_video
    p = CoTrackerPredictor(checkpoint=None, window_len=60)
    p.model.load_state_dict(sd)
    p = p.to("cuda")
    video = texture_video(16, SIZE, SIZE, seed=0).cuda()
    return alternate({"plain": lambda: p(video, grid_size=80),
                      "scores": lambda: p(video, grid_size=80, return_scores=True)}, reps, calls)


def hub(sd, reps, calls, K=8, G=50):
    """Two hubs of K streams on one predictor, one stepped with scores and one without; each step pushes the next
    chunk of every stream (the clips are long enough for every step the run takes)."""
    from cotracker_b200.predictor import CoTrackerOnlinePredictor
    from cotracker_b200.streams import OnlineStreams
    from cotracker_b200.synthetic import texture_video
    p = CoTrackerOnlinePredictor(checkpoint=None, window_len=S)
    p.model.load_state_dict(sd)
    p = p.to("cuda")
    n_steps = 2 + reps * calls + 1     # steps of each hub: warm-up and timed
    videos = [texture_video(STEP * n_steps + S, SIZE, SIZE, seed=k).to(torch.uint8).cuda() for k in range(K)]

    def make(scores):
        h = OnlineStreams(p)
        ids = [h.open(frame_size=(SIZE, SIZE), grid_size=G, history=64) for _ in range(K)]
        pos = [0]

        def step():
            for k, i in enumerate(ids):
                h.push(i, videos[k][:, STEP * pos[0]:STEP * pos[0] + S])
            pos[0] += 1
            return h.step(return_scores=scores)
        return step
    return alternate({"plain": make(False), "scores": make(True)}, reps, calls)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from cotracker_b200.synthetic import seeded_state_dict
    assert torch.cuda.is_available(), "scores_bench.py measures on a GPU"
    info = card()
    rows = []
    for name, fn, sd in (("offline_512x16_grid80", offline, seeded_state_dict(1234, offline=True, window_len=60)),
                         ("hub_8x512_grid50_step", hub, seeded_state_dict(1234, offline=False, window_len=S))):
        ms = fn(sd, args.reps, args.calls)
        row = dict(workload=name, ms_plain=round(ms["plain"], 3), ms_scores=round(ms["scores"], 3),
                   delta_ms=round(ms["scores"] - ms["plain"], 3),
                   delta_pct=round(100 * (ms["scores"] - ms["plain"]) / ms["plain"], 2), reps=args.reps,
                   calls=args.calls, **info)
        rows.append(row)
        print(json.dumps(row), flush=True)
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
