"""Clip ingestion and encode-once, end to end through CoTrackerPredictor.

    python scripts/ingest_bench.py [--reps 3]

Seeded offline-model weights; seeded random uint8 clips stored channels-last [T,H,W,3] as decoders return them.  Each
workload times whole predictor calls between device synchronisations (wall clock), alternating its variants after one
warm-up call of each, and records torch.cuda.max_memory_allocated over the call (the device-resident input included):
  C1-like 50 x 720 x 1296, grid 10, and 120 x 1080 x 1920, grid 30:
    aten-dev  : a float32 clip already on the device through the sequence before this change (ATen resize and
                normalisation, then the model);
    float-dev : the same device clip through the predictor (ct3_prepare_frames on the strided tensor);
    float-host: a float32 host clip moved with .cuda() inside the timed region (what users do);
    u8-host   : the uint8 host clip passed as is (chunked pinned upload + ct3_prepare_frames).
  backward tracking (50 x 720 x 1296, 100 queries at frames >= T/2):
    before: the explicit sequence (ATen resize, the model on the clip, the model on the flipped clip);
    after : CoTrackerPredictor(backward_tracking=True) on the same float device clip (encoded once).
  dense mode (8 x 160 x 224, 4 offset passes):
    before: one ATen resize + model call per offset pass;  after: CoTrackerPredictor(video) (encoded once).
Prints the card's name, power limit and max SM clock, then one line per variant: median ms (all runs), peak MiB, and
whether the outputs are bit-identical to the first variant of the workload; exits non-zero if any are not.
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cotracker_b200.predictor import CoTrackerPredictor, get_points_on_a_grid  # noqa: E402
from cotracker_b200.synthetic import random_queries, seeded_state_dict  # noqa: E402

DEV = "cuda:0"


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0) + " (nvidia-smi failed)"


def timed(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, torch.cuda.max_memory_allocated(), out


def u8_clip(T, H, W, seed):
    """[1,T,3,H,W] uint8 view of a channels-last [T,H,W,3] buffer: a smooth random texture (bilinear-upsampled noise)
    so that tracks have something to follow."""
    g = torch.Generator().manual_seed(seed)
    base = torch.rand(T, 3, H // 16 + 2, W // 16 + 2, generator=g) * 255
    big = F.interpolate(base, (H, W), mode="bilinear", align_corners=True)
    return big.round().to(torch.uint8).permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)[None]


def old_sparse(p, video, queries, backward, grid=0, support=False):
    """The sequence a sparse predictor call ran before: ATen resize, the model on the clip and, with backward tracking,
    the model on the flipped clip.  grid > 0: a grid of queries at frame 0 instead of `queries`; support: append the
    6x6 support grid (the predictor does for explicit queries) and drop its columns at the end."""
    B, T, C, H, W = video.shape
    ih, iw = p.interp_shape
    v = F.interpolate(video[0], (ih, iw), mode="bilinear", align_corners=True)[None]
    if grid > 0:
        pts = get_points_on_a_grid(grid, p.interp_shape, device=video.device)
        q = torch.cat([torch.zeros_like(pts[:, :, :1]), pts], dim=2)
    else:
        q = queries.clone()
        q[:, :, 1:] *= q.new_tensor([(iw - 1) / (W - 1), (ih - 1) / (H - 1)])
    n = q.shape[1]
    if support:
        sup = get_points_on_a_grid(6, p.interp_shape, device=q.device)
        q = torch.cat([q, torch.cat([torch.zeros_like(sup[:, :, :1]), sup], dim=2)], dim=1)
    tracks, vis, *_ = p.model(video=v, queries=q, iters=6)
    if backward:
        iq = q.clone()
        iq[:, :, 0] = T - iq[:, :, 0] - 1
        it, ivis, *_ = p.model(video=v.flip(1).clone(), queries=iq, iters=6)
        before = torch.arange(T, device=q.device)[None, :, None] < q[:, None, :, 0]
        tracks = torch.where(before[..., None], it.flip(1), tracks)
        vis = torch.where(before, ivis.flip(1), vis)
    tracks, vis, q = tracks[:, :, :n], vis[:, :, :n], q[:, :n]
    vis = vis > 0.9
    idx = torch.arange(tracks.size(2), device=tracks.device)
    qt = q[0, :, 0].to(torch.int64)
    tracks[0, qt, idx] = q[0, :, 1:]
    vis[0, qt, idx] = True
    tracks *= tracks.new_tensor([(W - 1) / (iw - 1), (H - 1) / (ih - 1)])
    return tracks, vis


def old_dense(p, video):
    """Dense mode before: every offset pass resized and encoded the clip again."""
    *_, H, W = video.shape
    step = W // 80
    gw, gh = W // step, H // step
    base_x = (torch.arange(gw, device=DEV).repeat(gh) * step).float()
    base_y = (torch.arange(gh, device=DEV).repeat_interleave(gw) * step).float()
    outs = []
    for offset in range(step * step):
        pts = torch.zeros(1, gw * gh, 3, device=DEV)
        pts[:, :, 1] = base_x + offset % step
        pts[:, :, 2] = base_y + offset // step
        outs.append(old_sparse(p, video, pts, backward=False))
    return torch.cat([t for t, _ in outs], dim=2), torch.cat([v for _, v in outs], dim=2)


def run(name, variants, reps):
    """variants: [(label, fn)]; fn() -> tuple of output tensors.  Alternates the variants, reps rounds after a warm-up."""
    outs, times, peaks = {}, {lab: [] for lab, _ in variants}, {}
    with torch.no_grad():
        for lab, fn in variants:
            _, peaks[lab], outs[lab] = timed(fn)
        for _ in range(reps):
            for lab, fn in variants:
                ms, pk, outs[lab] = timed(fn)
                times[lab].append(ms)
                peaks[lab] = max(peaks[lab], pk)
    first = variants[0][0]
    ok = True
    for lab, _ in variants:
        same = all(torch.equal(a, b) for a, b in zip(outs[lab], outs[first]))
        ok &= same
        ts = sorted(times[lab])
        print(f"{name:<26} {lab:<10} {ts[len(ts) // 2]:9.1f} ms  (runs {', '.join(f'{t:.1f}' for t in ts)})  "
              f"peak {peaks[lab] / 2**20:8.0f} MiB  bit-identical to {first}: {same}", flush=True)
    return ok


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    print(f"card: {card()}")
    p = CoTrackerPredictor(checkpoint=None, window_len=60)
    p.model.load_state_dict(seeded_state_dict(1234, offline=True, window_len=60))
    p = p.to(DEV)
    ok = True
    for T, H, W, grid in ((50, 720, 1296, 10), (120, 1080, 1920, 30)):
        u8 = u8_clip(T, H, W, seed=T)
        fl_host = u8.float()                          # channels-last float host clip, as .float() leaves it
        fl_dev = fl_host.to(DEV)
        ok &= run(f"{T}x{H}x{W} grid {grid}", [
            ("aten-dev", lambda: old_sparse(p, fl_dev, None, backward=False, grid=grid)),
            ("float-dev", lambda: p(fl_dev, grid_size=grid)),
            ("float-host", lambda: p(fl_host.cuda(), grid_size=grid)),
            ("u8-host", lambda: p(u8, grid_size=grid)),
        ], args.reps)
        del fl_dev, fl_host, u8
        torch.cuda.empty_cache()

    T, H, W = 50, 720, 1296
    video = u8_clip(T, H, W, seed=7).float().to(DEV)
    queries = random_queries(100, T, H, W, seed=8).to(DEV)
    queries[0, :, 0] = queries[0, :, 0] % (T // 2) + T // 2  # every query at a later frame
    ok &= run(f"backward {T}x{H}x{W} N=100", [
        ("before", lambda: old_sparse(p, video, queries, backward=True, support=True)),
        ("after", lambda: p(video, queries=queries, backward_tracking=True)),
    ], args.reps)
    del video

    dense = u8_clip(8, 160, 224, seed=9).float().to(DEV)
    ok &= run("dense 8x160x224", [
        ("before", lambda: old_dense(p, dense)),
        ("after", lambda: p(dense)),
    ], args.reps)
    if not ok:
        sys.exit("variants of a workload differ")


if __name__ == "__main__":
    main()
