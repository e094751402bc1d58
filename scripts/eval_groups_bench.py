"""Single-point TAP-Vid evaluation: one model call per query group vs all groups through forward_groups.

    python scripts/eval_groups_bench.py [--T 50 250] [--queries 30] [--reps 3]

Workload: a TAP-Vid-like clip (256x256 input, resized to the model's 384x512 as EvaluationPredictor does), `--queries`
queries at seeded random frames and positions, seeded offline-model weights.  Each query becomes the reference's
single-point group: the query, an 8x8 local grid around it and a 5x5 global grid (90 tracks).  Two versions are timed
in one process, alternating, after a warm-up, between CUDA events:
  (a) per-query: one `model(video, group)` call per query group (the encoder and update loop run once per query);
  (b) grouped:   EvaluationPredictor(single_point=True), i.e. `forward_groups` over as few passes as fit in memory.
Prints ms per video for both, the card's name, power limit and max SM clock, and whether (a) and (b) are
bit-identical; exits non-zero if they are not.
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cotracker_b200.build import build_cotracker  # noqa: E402
from cotracker_b200.evaluation import EvaluationPredictor  # noqa: E402
from cotracker_b200.synthetic import random_queries, seeded_state_dict, texture_video  # noqa: E402


def card(dev):
    q = subprocess.run(["nvidia-smi", f"--id={dev}", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(dev) + " (nvidia-smi failed)"


def per_query(ev, video, queries):
    """What single-point evaluation did before grouped calls: one model call per query group."""
    B, T, C, H, W = video.shape
    ih, iw = ev.interp_shape
    v = F.interpolate(video.reshape(B * T, C, H, W), (ih, iw), mode="bilinear", align_corners=True)
    v = v.reshape(B, T, 3, ih, iw)
    q = queries.clone()
    q[:, :, 1] *= (iw - 1) / (W - 1)
    q[:, :, 2] *= (ih - 1) / (H - 1)
    N = q.shape[1]
    tracks, vis, conf = v.new_zeros(B, T, N, 2), v.new_zeros(B, T, N), v.new_zeros(B, T, N)
    for i in range(N):
        qi = q[:, i:i + 1]
        q_all = torch.cat([qi, ev._helpers(v, qi)], dim=1)
        tr, vi, cf, _ = ev.model(video=v, queries=q_all, iters=ev.n_iters)
        tracks[:, :, i], vis[:, :, i], conf[:, :, i] = tr[:, :, 0, :2], vi[:, :, 0], cf[:, :, 0]
    tracks[..., 0] *= (W - 1) / float(iw - 1)
    tracks[..., 1] *= (H - 1) / float(ih - 1)
    return tracks, vis * conf


def timed(fn, *args):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn(*args)
    b.record()
    b.synchronize()
    return a.elapsed_time(b), out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--T", type=int, nargs="+", default=[50, 250])
    ap.add_argument("--queries", type=int, default=30)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=6)
    args = ap.parse_args()
    dev = 0
    torch.cuda.set_device(dev)
    print(f"card: {card(dev)}")
    model = build_cotracker(None, offline=True, window_len=60).eval()
    model.load_state_dict(seeded_state_dict(1234, offline=True, window_len=60))
    model = model.to(f"cuda:{dev}")
    ev = EvaluationPredictor(model, single_point=True, grid_size=5, local_grid_size=8, n_iters=args.iters)
    identical = True
    for T in args.T:
        video = texture_video(T, 256, 256, seed=T).to(f"cuda:{dev}")
        queries = random_queries(args.queries, T, 256, 256, seed=T + 1).to(f"cuda:{dev}")
        with torch.no_grad():
            per_query(ev, video, queries)                      # warm-up (kernels, workspaces)
            ev(video, queries)
            times = {"per_query": [], "grouped": []}
            outs = {}
            for _ in range(args.reps):
                for name, fn in (("per_query", per_query), ("grouped", lambda e, v, q: e(v, q))):
                    ms, outs[name] = timed(fn, ev, video, queries)
                    times[name].append(ms)
        same = all(torch.equal(x, y) for x, y in zip(outs["per_query"], outs["grouped"]))
        identical &= same
        pq, gr = sorted(times["per_query"]), sorted(times["grouped"])
        print(f"T={T} queries={args.queries} (90 tracks each) iters={args.iters}: "
              f"per-query {pq[len(pq) // 2]:.1f} ms/video (runs {', '.join(f'{t:.1f}' for t in pq)}), "
              f"grouped {gr[len(gr) // 2]:.1f} ms/video (runs {', '.join(f'{t:.1f}' for t in gr)}), "
              f"speed-up x{pq[len(pq) // 2] / gr[len(gr) // 2]:.2f}, bit-identical: {same}", flush=True)
    if not identical:
        sys.exit("per-query and grouped outputs differ")


if __name__ == "__main__":
    main()
