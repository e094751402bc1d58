"""What encoding a clip once saves: direct predictor calls against `encode` once and calls on the EncodedClip, and
what parking a clip on the host costs.

    python scripts/encoded_clip_bench.py [--reps 5] [--out result.json]

Reports, with the GPU's name and power limit:
  - calls: for host uint8 clips of 720p and 1080p, T = 24 and 60, the offline predictor (seeded weights) with 1, 16 and
    256 query points (the support grid is appended to each) and with grid_size=30: ms per direct call
    `predictor(video, queries=...)`, ms of one `encode(video)`, and ms per call `predictor(clip, queries=...)` on the
    encoded clip, which includes the clip's checks (the weights' fingerprint among them).  The two kinds of call
    alternate, each is timed by a host clock around work that ends in a device synchronise, after one warm-up of
    each, and the median of --reps is reported.  `equal` records that the two results were torch.equal.
  - park: for the 720p clips, ms of clip.to("cpu") (the copy of level 0 into pinned host memory, ending in a
    synchronise) and of clip.to("cuda:0") (upload plus ct3_pyramid_pools, synchronised), the device bytes the clip
    held, the bytes moved each way and the rate.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from cotracker_b200.predictor import CoTrackerPredictor  # noqa: E402
from cotracker_b200.synthetic import random_queries, seeded_state_dict  # noqa: E402

DEV = "cuda:0"
SIZES = {"720p": (720, 1280), "1080p": (1080, 1920)}


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name(0) + ", power limit unknown"
    return q


def _ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def host_clip(T, H, W, seed):
    """[1,T,3,H,W] uint8 on the host, laid out as a decoder hands it over ([T,H,W,3] storage): a random texture
    moving by a few pixels per frame."""
    g = torch.Generator().manual_seed(seed)
    tex = torch.randint(0, 256, (3, H // 8 + 8, W // 8 + 8), generator=g, dtype=torch.uint8)
    tex = tex.repeat_interleave(8, 1).repeat_interleave(8, 2)
    frames = torch.stack([tex[:, t % 32:t % 32 + H, 2 * (t % 32):2 * (t % 32) + W] for t in range(T)])
    return frames.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)[None]


def bench_calls(p, name, T, reps):
    H, W = SIZES[name]
    video = host_clip(T, H, W, seed=T)
    p.encode(video)   # warm-up: the first call at a size also sets up the encoder's workspace
    enc_ms, clip = _ms(lambda: p.encode(video))
    rows = []
    modes = [(f"{n} queries", dict(queries=random_queries(n, T, H, W, seed=n).to(DEV))) for n in (1, 16, 256)]
    for kw_name, kw in modes + [("grid 30", dict(grid_size=30))]:
        direct, cached = [], []
        want, got = p(video, **kw), p(clip, **kw)   # warm-up of both
        equal = all(torch.equal(a, b) for a, b in zip(want, got))
        for _ in range(reps):
            direct.append(_ms(lambda: p(video, **kw))[0])
            cached.append(_ms(lambda: p(clip, **kw))[0])
        d, c = statistics.median(direct), statistics.median(cached)
        rows.append(dict(clip=f"{name} T={T}", tracks=kw_name, direct_ms=round(d, 2), encoded_ms=round(c, 2),
                         saved_ms=round(d - c, 2), speedup=round(d / c, 2), encode_ms=round(enc_ms, 2), equal=equal))
        print(json.dumps(rows[-1]), flush=True)
    return rows, clip


def bench_park(clip, name, reps):
    held = clip.nbytes
    downs, ups, moved = [], [], 0
    for _ in range(reps + 1):
        down, _ = _ms(lambda: clip.to("cpu"))
        moved = clip.host.numel() * clip.host.element_size()
        up, _ = _ms(lambda: clip.to(DEV))
        downs.append(down)
        ups.append(up)
    d, u = statistics.median(downs[1:]), statistics.median(ups[1:])
    row = dict(clip=name, device_bytes=held, parked_bytes=moved, parked_share=round(moved / held, 3),
               park_ms=round(d, 2), return_ms=round(u, 2), park_GBps=round(moved / d / 1e6, 1),
               return_GBps=round(moved / u / 1e6, 1))
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("encoded_clip_bench.py needs a GPU")
    res = dict(gpu=gpu_info(), calls=[], park=[])
    print(res["gpu"], flush=True)
    p = CoTrackerPredictor(checkpoint=None, window_len=60)
    p.model.load_state_dict(seeded_state_dict(1234, offline=True, window_len=60))
    p = p.to(DEV)
    with torch.no_grad():
        for name in SIZES:
            for T in (24, 60):
                rows, clip = bench_calls(p, name, T, a.reps)
                res["calls"] += rows
                if name == "720p":
                    res["park"].append(bench_park(clip, f"{name} T={T}", a.reps))
                del clip
    res["never_slower"] = all(r["encoded_ms"] <= r["direct_ms"] for r in res["calls"])
    res["all_equal"] = all(r["equal"] for r in res["calls"])
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
