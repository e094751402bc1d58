"""The cost of track edits in online streams (`OnlineStreams.retire_tracks` / `add_tracks`, DESIGN.md 4.4.4).

K streams of a G x G grid (default 8 x 2500 tracks) on one `OnlineStreams` hub, 512x512 uint8 device frames,
window_len 16, seeded weights, every stream bounded by `--history`.  After `--warmup` steps:

- edit: the wall time of one `retire_tracks` of 10 % of stream 0's tracks plus one `add_tracks` of as many, ending
  in a device synchronise; median of `--edits` edits made in one gap.  Each edit copies the pool's support features
  (4 x 49 x 128 fp32 = 100,352 bytes per track) once per call.
- step: the wall time of one iteration (push every stream's chunk, `step()`, synchronise) without an edit, and with
  the 10 % edit of stream 0 before it; blocks of `--block` iterations alternate between the two `--rounds` times,
  and the median of each mode is kept.

Prints one JSON line per measurement with the card's name and power limit read in the same run.

    python scripts/stream_edits_bench.py [--ks 8] [--grid 50] [--history 16] [--out stream_edits_bench.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SIZE, S, STEP, PERIOD = 512, 16, 8, 64


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, power = (x.strip() for x in q.split(","))
    return {"gpu": name, "power_limit": power}


class Churn:
    """Replaces the oldest `m` tracks of one stream with `m` new ones whose query frames lie in its next window."""

    def __init__(self, hub, sid, m, seed=0):
        self.hub, self.sid, self.m = hub, sid, m
        self.g = torch.Generator().manual_seed(seed)

    def __call__(self):
        hub, sid, m = self.hub, self.sid, self.m
        t = hub.length(sid) + torch.randint(0, STEP, (m,), generator=self.g).float()
        xy = torch.rand(m, 2, generator=self.g) * (SIZE - 1)
        hub.retire_tracks(sid, hub.track_ids(sid)[:m])
        hub.add_tracks(sid, torch.cat([t[:, None], xy], 1)[None].cuda())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", type=int, nargs="+", default=[8])
    ap.add_argument("--grid", type=int, default=50)
    ap.add_argument("--history", type=int, default=16)
    ap.add_argument("--fraction", type=float, default=0.1)
    ap.add_argument("--warmup", type=int, default=6)
    ap.add_argument("--edits", type=int, default=20)
    ap.add_argument("--block", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from cotracker_b200.predictor import CoTrackerOnlinePredictor
    from cotracker_b200.streams import OnlineStreams
    from cotracker_b200.synthetic import seeded_state_dict, texture_video
    assert torch.cuda.is_available(), "stream_edits_bench.py measures on a GPU"
    info = card()
    p = CoTrackerOnlinePredictor(checkpoint=None, window_len=S)
    p.model.load_state_dict(seeded_state_dict(1234, offline=False, window_len=S))
    p = p.to("cuda")
    loops = []
    for k in range(max(args.ks)):
        v = texture_video(PERIOD, SIZE, SIZE, seed=k).to(torch.uint8).cuda()
        loops.append(torch.cat([v, v[:, :S]], 1))
    rows = []
    for K in args.ks:
        hub = OnlineStreams(p)
        ids = [hub.open(frame_size=(SIZE, SIZE), grid_size=args.grid, history=args.history) for _ in range(K)]
        n = args.grid ** 2
        m = max(1, int(n * args.fraction))
        edit = Churn(hub, ids[0], m)
        state = {"i": 0}

        def iteration(with_edit):
            if with_edit:
                edit()
            o = STEP * state["i"] % PERIOD
            state["i"] += 1
            for k, sid in enumerate(ids):
                hub.push(sid, loops[k][:, o:o + S])
            out = hub.step()
            del out

        for i in range(args.warmup):            # every shape, with and without an edit
            iteration(i % 2 == 1)
        torch.cuda.synchronize()
        edit_ms = []
        for _ in range(args.edits):
            t0 = time.perf_counter()
            edit()
            torch.cuda.synchronize()
            edit_ms.append((time.perf_counter() - t0) * 1e3)
        step_ms = {False: [], True: []}
        for _ in range(args.rounds):
            for mode in (False, True):
                for _ in range(args.block):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    iteration(mode)
                    torch.cuda.synchronize()
                    step_ms[mode].append((time.perf_counter() - t0) * 1e3)
        pool_tracks = int(hub.pool.qframes.shape[0])
        base = dict(K=K, tracks_per_stream=n, edited=m, history=args.history, pool_tracks=pool_tracks,
                    support_mb=round(hub.pool.support.numel() * 4 / 2 ** 20, 1), **info)
        for row in (dict(base, what="edit", ms=round(statistics.median(edit_ms), 3),
                         ms_min=round(min(edit_ms), 3), count=len(edit_ms)),
                    dict(base, what="step", ms=round(statistics.median(step_ms[False]), 3),
                         ms_min=round(min(step_ms[False]), 3), count=len(step_ms[False])),
                    dict(base, what="step+edit", ms=round(statistics.median(step_ms[True]), 3),
                         ms_min=round(min(step_ms[True]), 3), count=len(step_ms[True]))):
            rows.append(row)
            print(json.dumps(row), flush=True)
        for sid in ids:
            hub.close(sid)
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
