"""K independent online streams on one GPU, three ways (DESIGN.md 4.4.4):

  (a) OnlineStreams, stream k opened k steps after stream 0 (staggered), every open stream advancing each step;
      a_aligned: the same with every stream opened at once;
  (b) K CoTrackerOnlinePredictors stepped one after another;
  (c) one CoTrackerOnlinePredictor with the K streams as a lockstep batch (possible only with aligned starts).

512x512 uint8 device frames, window_len 16 (8 new frames per stream and step), grid 10 and grid 50, K in {1, 4, 16};
seeded weights.  Every setup is warmed up on its shapes before the timed steps, which are timed with CUDA events
around `--steps` steps that end in a device synchronise.  Prints one JSON line per (setup, grid, K) with ms per step
and stream * new frames / s, plus the card's name and power limit read in the same run.

    python scripts/streams_bench.py [--steps 10] [--warmup 3] [--out streams_bench.json]
"""
from __future__ import annotations

import argparse
import gc
import json
import os
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


def make_predictor(sd):
    from cotracker_b200.predictor import CoTrackerOnlinePredictor
    p = CoTrackerOnlinePredictor(checkpoint=None, window_len=S)
    p.model.load_state_dict(sd)
    return p.to("cuda")


def timed(fn, steps):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def run(setup, K, G, videos, sd, warmup, steps):
    """ms per step of `setup` with K streams of a G x G grid, after `warmup` steps with every stream running."""
    from cotracker_b200.streams import OnlineStreams
    pos = [0] * K

    def chunk(k):
        c = videos[k][:, STEP * pos[k]:STEP * pos[k] + S]
        pos[k] += 1
        return c

    if setup in ("a", "a_aligned"):
        hub = OnlineStreams(make_predictor(sd))
        ids = []

        def step():   # staggered: one more stream opens each step until K are open
            while len(ids) < (K if setup == "a_aligned" else min(K, len(ids) + 1)):
                ids.append(hub.open(frame_size=(SIZE, SIZE), grid_size=G))
            for k, i in enumerate(ids):
                hub.push(i, chunk(k))
            return hub.step()
        for _ in range(K - 1 if setup == "a" else 0):   # the staggered opening
            step()
    elif setup == "b":
        preds = [make_predictor(sd) for _ in range(K)]
        for k, p in enumerate(preds):
            p(video_chunk=videos[k][:, :S], is_first_step=True, grid_size=G)

        def step():
            return [p(video_chunk=chunk(k)) for k, p in enumerate(preds)]
    else:
        p = make_predictor(sd)
        batch = torch.cat(videos)
        p(video_chunk=batch[:, :S], is_first_step=True, grid_size=G)

        def step():
            c = batch[:, STEP * pos[0]:STEP * pos[0] + S]
            pos[0] += 1
            return p(video_chunk=c)
    for _ in range(warmup):
        step()
    return timed(step, steps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--grids", type=int, nargs="+", default=[10, 50])
    ap.add_argument("--ks", type=int, nargs="+", default=[1, 4, 16])
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from cotracker_b200.synthetic import seeded_state_dict, texture_video
    assert torch.cuda.is_available(), "streams_bench.py measures on a GPU"
    info = card()
    sd = seeded_state_dict(1234, offline=False, window_len=S)
    n_steps = max(args.ks) + args.warmup + args.steps + 2
    videos = [texture_video(STEP * n_steps + S, SIZE, SIZE, seed=k).to(torch.uint8).cuda() for k in range(max(args.ks))]
    rows = []
    for G in args.grids:
        for K in args.ks:
            for setup in ("a", "a_aligned", "b", "c"):
                try:
                    ms = run(setup, K, G, videos[:K], sd, args.warmup, args.steps)
                    row = dict(setup=setup, grid=G, K=K, ms_per_step=round(ms, 3),
                               stream_new_frames_per_s=round(K * STEP / (ms / 1e3), 1), **info)
                except torch.OutOfMemoryError:   # K separate predictors each keep their own update-loop workspace
                    row = dict(setup=setup, grid=G, K=K, ms_per_step=None, stream_new_frames_per_s=None,
                               note="out of device memory", **info)
                gc.collect()
                rows.append(row)
                print(json.dumps(row), flush=True)
                torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
