"""The cost of stream snapshots (`OnlineStreams.snapshot` / `restore`, DESIGN.md 4.4.4).

K streams of a G x G grid (default 8 streams) on one `OnlineStreams` hub, 512x512 uint8 device frames, window_len 16,
seeded weights, every stream bounded by `--history` or unbounded (`--history 0`), advanced `--steps` steps, then stream
0 parked and restored once and every stream advanced once more, so that every shape is warm.  Then, for stream 0:

- snapshot: the wall time of `hub.snapshot(sid)`, ending in a device synchronise, median of `--reps`; and the
  snapshot's size, the bytes of its tensors.
- restore: the wall time of `hub.restore(snap)`, ending in a device synchronise, median of `--reps` (each restored copy
  is closed again, untimed).
- step / step after restore: the wall time of one iteration (push every stream's chunk, `step()`, synchronise), an
  ordinary one alternating with one right after stream 0 was parked and restored (snapshot, close, restore, untimed):
  the first step after a restore encodes stream 0's whole chunk, 16 frames instead of 8.  `--rounds` of each, medians.
- step / step after snapshot: blocks of `--block` iterations alternate between no snapshot and a snapshot of stream 0
  taken in the gap before each step (untimed), `--rounds` times; medians.

Prints one JSON line per measurement with the card's name and power limit read in the same run.

    python scripts/stream_snapshot_bench.py [--grids 10 50] [--histories 16 0] [--steps 100] [--out snap.json]
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


def snapshot_bytes(snap) -> int:
    tensors = [v for v in snap.values() if torch.is_tensor(v)] + list(snap["hist"] or [])
    return sum(t.numel() * t.element_size() for t in tensors)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def med(xs):
    return round(statistics.median(xs), 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--K", type=int, default=8)
    ap.add_argument("--grids", type=int, nargs="+", default=[10, 50])
    ap.add_argument("--histories", type=int, nargs="+", default=[16, 0], help="0: unbounded")
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--block", type=int, default=4)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from cotracker_b200.predictor import CoTrackerOnlinePredictor
    from cotracker_b200.streams import OnlineStreams
    from cotracker_b200.synthetic import seeded_state_dict, texture_video
    assert torch.cuda.is_available(), "stream_snapshot_bench.py measures on a GPU"
    info = card()
    p = CoTrackerOnlinePredictor(checkpoint=None, window_len=S)
    p.model.load_state_dict(seeded_state_dict(1234, offline=False, window_len=S))
    p = p.to("cuda")
    loops = []
    for k in range(args.K):
        v = texture_video(PERIOD, SIZE, SIZE, seed=k).to(torch.uint8).cuda()
        loops.append(torch.cat([v, v[:, :S]], 1))
    rows = []
    for grid in args.grids:
        for history in args.histories:
            hub = OnlineStreams(p)
            ids = [hub.open(frame_size=(SIZE, SIZE), grid_size=grid, history=history or None)
                   for _ in range(args.K)]
            pos = [0] * args.K

            def iteration():
                for k, sid in enumerate(ids):
                    o = STEP * pos[k] % PERIOD
                    pos[k] += 1
                    hub.push(sid, loops[k][:, o:o + S])
                out = hub.step()
                del out

            def park_restore():
                snap = hub.snapshot(ids[0])
                hub.close(ids[0])
                ids[0] = hub.restore(snap)

            for _ in range(args.steps):
                iteration()
            park_restore()                                # every shape, a restore included
            iteration()
            snap_ms, restore_ms = [], []
            for _ in range(args.reps):
                ms, snap = timed(lambda: hub.snapshot(ids[0]))
                snap_ms.append(ms)
            nbytes, length = snapshot_bytes(snap), snap["length"]
            for _ in range(args.reps):
                ms, rid = timed(lambda: hub.restore(snap))
                restore_ms.append(ms)
                hub.close(rid)
            step_ms, first_ms = [], []
            for _ in range(args.rounds):
                step_ms.append(timed(iteration)[0])
                park_restore()
                first_ms.append(timed(iteration)[0])
            plain_ms, gap_ms = [], []
            for _ in range(args.rounds):
                for _ in range(args.block):
                    plain_ms.append(timed(iteration)[0])
                for _ in range(args.block):
                    hub.snapshot(ids[0])
                    gap_ms.append(timed(iteration)[0])
            base = dict(K=args.K, grid=grid, tracks_per_stream=grid * grid, history=history or None,
                        steps_before=args.steps, snapshot_length=length, **info)
            for row in (dict(base, what="snapshot", ms=med(snap_ms), ms_min=round(min(snap_ms), 3),
                             count=len(snap_ms), bytes=nbytes),
                        dict(base, what="restore", ms=med(restore_ms), ms_min=round(min(restore_ms), 3),
                             count=len(restore_ms), bytes=nbytes),
                        dict(base, what="step", ms=med(step_ms), count=len(step_ms)),
                        dict(base, what="first step after restore", ms=med(first_ms), count=len(first_ms)),
                        dict(base, what="step, no snapshot in the gap", ms=med(plain_ms), count=len(plain_ms)),
                        dict(base, what="step, snapshot in the gap", ms=med(gap_ms), count=len(gap_ms))):
                rows.append(row)
                print(json.dumps(row), flush=True)
            for sid in ids:
                hub.close(sid)
            del hub
            torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
