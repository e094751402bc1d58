"""What results at every frame cost (DESIGN.md 4.4.4, "Previews"): a simulated 30 fps camera per stream.  K = 1, 4 and 16
streams of 512x512 uint8 device frames, window_len 16, seeded weights, grid_size 10 and 50.  At each tick every stream
gets one new frame f: it pushes the committing chunk when f completes its window (every 8th tick once running), and a
preview of frames [w, f] otherwise, then the hub steps once.

A second hub on the same predictor is fed the committing chunks only, and its commit steps alternate with the first
hub's in the same process: `commit_ms` against `commit_ms_no_previews` is what previews in between do to a commit.
`support_gather_ms` times one preview's extra device work at its stream's size, the gather of the stream's support
rows into pass scratch (CUDA events over 20 gathers).

Ticks of the first window (every stream before its first step) are the warm-up; the next `--windows` windows are
timed, each tick with a host clock around the step and a device synchronise.  Reported per workload, in one JSON line
with the card's name and power limit read in the same run: the median tick, the median preview tick and commit tick,
and the frames the encoder saw per tick and stream.

    python scripts/preview_bench.py [--windows 3] [--out preview_bench.json]
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

SIZE, S, STEP = 512, 16, 8


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, power = (x.strip() for x in q.split(","))
    return {"gpu": name, "power_limit": power}


def synced(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def gather_ms(pool, state, reps=20):
    idx = torch.arange(state.first, state.first + state.n, device=pool.support.device)
    pool.support.index_select(2, idx)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        pool.support.index_select(2, idx)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def workload(p, K, G, windows):
    from cotracker_b200.streams import OnlineStreams
    from cotracker_b200.synthetic import texture_video
    frames = S + STEP * windows
    videos = [texture_video(frames, SIZE, SIZE, seed=k).to(torch.uint8).cuda() for k in range(K)]
    encoded = []
    encode = p.model._encode
    p.model._encode = lambda video, chunk: encoded.append(video.shape[0]) or encode(video, chunk)
    try:
        live, plain = OnlineStreams(p), OnlineStreams(p)
        ids = [live.open(frame_size=(SIZE, SIZE), grid_size=G) for _ in range(K)]
        pids = [plain.open(frame_size=(SIZE, SIZE), grid_size=G) for _ in range(K)]
        ticks, previews, commits, commits_plain, enc = [], [], [], [], []
        for f in range(frames):
            w = max(0, live.length(ids[0]) - (S - STEP))
            commit = f + 1 == w + S
            for k, i in enumerate(ids):
                live.push(i, videos[k][:, w:f + 1], preview=not commit)
            n0 = sum(encoded)
            ms, _ = synced(live.step)
            n = sum(encoded) - n0
            if commit:
                for k, i in enumerate(pids):
                    plain.push(i, videos[k][:, w:f + 1])
                ms_plain, _ = synced(plain.step)
            if f < S:   # the first window: warm-up
                continue
            ticks.append(ms)
            enc.append(n / K)
            (commits if commit else previews).append(ms)
            if commit:
                commits_plain.append(ms_plain)
        state = live._streams[ids[0]]["state"]
        return dict(tick_ms=statistics.median(ticks), preview_ms=statistics.median(previews),
                    commit_ms=statistics.median(commits), commit_ms_no_previews=statistics.median(commits_plain),
                    frames_encoded_per_tick_per_stream=sum(enc) / len(enc), ticks=len(ticks), commits=len(commits),
                    support_gather_ms=gather_ms(live.pool, state), tracks_per_stream=state.n)
    finally:
        del p.model._encode


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from cotracker_b200.predictor import CoTrackerOnlinePredictor
    from cotracker_b200.synthetic import seeded_state_dict
    assert torch.cuda.is_available(), "preview_bench.py measures on a GPU"
    info = card()
    p = CoTrackerOnlinePredictor(checkpoint=None, window_len=S)
    p.model.load_state_dict(seeded_state_dict(1234, offline=False, window_len=S))
    p = p.to("cuda")
    rows = []
    for G in (10, 50):
        for K in (1, 4, 16):
            r = workload(p, K, G, args.windows)
            row = dict(workload=f"preview_{K}x512_grid{G}", K=K, grid=G,
                       **{k: round(v, 3) if isinstance(v, float) else v for k, v in r.items()},
                       fits_30fps=r["tick_ms"] <= 1000 / 30, **info)
            rows.append(row)
            print(json.dumps(row), flush=True)
            torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
