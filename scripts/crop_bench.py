"""What tracking inside a window of the frame costs: a 3840 x 2160 clip at full frame against a 1024 x 768 window that
moves from frame to frame (`Crop`).

    python scripts/crop_bench.py [--reps 5] [--T 48] [--out result.json]

Reports, with the GPU's name and power limit, for a host uint8 clip (laid out as a decoder hands it over, [T,H,W,3])
and a device NV12 clip, each at full frame and in the moving window:
  - ingest_ms: one `prepare_video` to the model resolution (the ingest step of every call);
  - call_ms: one offline predictor call with grid_size=30 (seeded weights), ingest, encoder and update loop;
  - staged_bytes: the bytes a host clip stages through the pinned slots and uploads (0 for a device clip, which the
    kernels read in place).
Each time is a host clock around work that ends in a device synchronise, after one warm-up, median of --reps.
`equal` records that the Crop call was torch.equal to the call on the materialised window.
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

from cotracker_b200 import Crop, YUVClip, ingest  # noqa: E402
from cotracker_b200.predictor import CoTrackerPredictor  # noqa: E402
from cotracker_b200.synthetic import seeded_state_dict  # noqa: E402

DEV = "cuda:0"
H, W = 2160, 3840
WINDOW = (768, 1024)


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


def _median(fn, reps):
    fn()
    return statistics.median(_ms(fn)[0] for _ in range(reps))


def host_rgb(T, seed=1):
    """[1,T,3,H,W] uint8 on the host in [T,H,W,3] storage: a coarse random texture moving a few pixels a frame."""
    g = torch.Generator().manual_seed(seed)
    tex = torch.randint(0, 256, (H // 16 + 8, W // 16 + 8, 3), generator=g, dtype=torch.uint8)
    tex = tex.repeat_interleave(16, 0).repeat_interleave(16, 1)
    frames = torch.stack([tex[t % 64:t % 64 + H, 2 * (t % 64):2 * (t % 64) + W] for t in range(T)])
    return frames.permute(0, 3, 1, 2)[None]


def device_nv12(T, seed=2):
    """[1,T,H*3/2,W] NV12 on the device: the luma of host_rgb's texture, flat chroma."""
    y = host_rgb(T, seed)[0, :, 1].to(DEV)
    uv = torch.full((T, H // 2, W), 128, dtype=torch.uint8, device=DEV)
    return YUVClip(torch.cat([y, uv], 1)[None].contiguous(), "nv12")


def moving_window(T):
    """A 1024 x 768 window sweeping across the frame, [T,2] (top, left)."""
    t = torch.arange(T)
    return torch.stack([(23 * t) % (H - WINDOW[0] + 1), (61 * t) % (W - WINDOW[1] + 1)], -1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--T", type=int, default=48)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("crop_bench.py needs a GPU")
    res = dict(gpu=gpu_info(), T=a.T, frame=[H, W], window=list(WINDOW), rows=[])
    print(res["gpu"], flush=True)
    p = CoTrackerPredictor(checkpoint=None, window_len=60)
    p.model.load_state_dict(seeded_state_dict(1234, offline=True, window_len=60))
    p = p.to(DEV)
    off = moving_window(a.T)
    with torch.no_grad():
        for source, video in (("host uint8", host_rgb(a.T)), ("device nv12", device_nv12(a.T))):
            host = not video.is_cuda
            for name, clip, hw in (("full frame", video, (H, W)), ("1024x768 moving", Crop(video, WINDOW, off),
                                                                    WINDOW)):
                ingest_ms = _median(lambda: ingest.prepare_video(clip, p.interp_shape, DEV), a.reps)
                call_ms = _median(lambda: p(clip, grid_size=30), a.reps)
                row = dict(source=source, window=name, ingest_ms=round(ingest_ms, 2), call_ms=round(call_ms, 2),
                           staged_bytes=a.T * 3 * hw[0] * hw[1] if host else 0)
                if isinstance(clip, Crop):   # the same call on the materialised window
                    rgb = video if not isinstance(video, YUVClip) else None
                    if rgb is not None:
                        mat = torch.stack([rgb[0, t, :, r:r + WINDOW[0], c:c + WINDOW[1]]
                                           for t, (r, c) in enumerate(off.tolist())])[None]
                        row["equal"] = all(torch.equal(x, y) for x, y in zip(p(clip, grid_size=30),
                                                                               p(mat, grid_size=30)))
                res["rows"].append(row)
                print(json.dumps(row), flush=True)
            del video
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
