"""YUV input, measured: the conversion kernel, a host 1080p clip through CoTrackerPredictor, and host 720p streams.

    python scripts/yuv_bench.py [--reps 3] [--steps 10]

Seeded weights (cotracker_b200.synthetic) and seeded smooth random clips.  Prints the card's name, power limit and max
SM clock, then:
  1. kernel: ct3_prepare_frames_yuv for nv12, i420 and yuyv, and ct3_prepare_frames on the uint8 RGB clip [T,3,H,W],
     1080 x 1920 -> 384 x 512, 8 frames a launch, CUDA events over >= 1 s of launches: us per frame.
  2. clip: a host 1080p clip of 50 frames through CoTrackerPredictor(grid_size=10), the arms alternating after one
     warm-up call each: wall ms (ending in a synchronise) and host CPU ms (time.process_time) per call, median.
       yuv-i420 : the decoder's I420 frames as a YUVClip;
       cv2-rgb  : cv2.cvtColor(COLOR_YUV2RGB_I420) per frame on the host, then the RGB clip (skipped without cv2);
       rgb      : the RGB clip already converted (conversion not counted), for the upload alone.
  3. streams: OnlineStreams with four host 720p streams (window 16, grid 10), one 16-frame chunk (8 new frames) per
     stream and step, the same three arms: ms per step (push + step, ending in a synchronise), median over --steps
     steps.
Every arm's results are compared with torch.equal against the yuv-i420 arm's; the script exits non-zero if any differ.
"""
from __future__ import annotations

import argparse
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from cotracker_b200 import OnlineStreams, YUVClip, engine  # noqa: E402
from cotracker_b200.predictor import CoTrackerOnlinePredictor, CoTrackerPredictor  # noqa: E402
from cotracker_b200.synthetic import seeded_state_dict  # noqa: E402
from yuv_cases import pack, yuv_to_rgb  # noqa: E402

DEV = "cuda:0"
try:
    import cv2
except ImportError:   # the cv2 arms are skipped, and say so
    cv2 = None


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0) + " (nvidia-smi failed)"


def i420_clip(T, H, W, seed):
    """uint8 I420 frames [1,T,H*3/2,W] of a smooth random texture drifting 2 px a frame (something to track)."""
    g = torch.Generator().manual_seed(seed)
    base = torch.rand(1, 3, H // 16 + 2, W // 16 + 2, generator=g) * 255
    big = F.interpolate(base, (H + 2 * T, W + 2 * T), mode="bilinear", align_corners=True)[0].round().to(torch.uint8)
    f = torch.stack([big[:, 2 * t:2 * t + H, 2 * t:2 * t + W] for t in range(T)])         # [T,3,H,W]
    return pack("i420", f[:, 0], f[:, 1, 0::2, 0::2].contiguous(), f[:, 2, 1::2, 1::2].contiguous())[None].contiguous()


def cv2_rgb(i420):
    """[1,T,H*3/2,W] I420 -> [1,T,3,H,W] uint8 view of cv2's channels-last RGB frames."""
    frames = [cv2.cvtColor(f.numpy(), cv2.COLOR_YUV2RGB_I420) for f in i420[0]]
    return torch.from_numpy(np.stack(frames)).permute(0, 3, 1, 2)[None]


def kernel_bench():
    H, W, T, oh, ow = 1080, 1920, 8, 384, 512
    g = torch.Generator().manual_seed(1)
    srcs = {"nv12": torch.randint(0, 256, (T, H * 3 // 2, W), generator=g, dtype=torch.uint8),
            "i420": torch.randint(0, 256, (T, H * 3 // 2, W), generator=g, dtype=torch.uint8),
            "yuyv": torch.randint(0, 256, (T, H, W, 2), generator=g, dtype=torch.uint8),
            "rgb-u8": torch.randint(0, 256, (T, 3, H, W), generator=g, dtype=torch.uint8)}
    out = torch.empty(T, 3, oh, ow, device=DEV)
    for name, src in srcs.items():
        src = src.to(DEV)
        fn = ((lambda: engine.prepare_frames(src, (oh, ow), out=out)) if name == "rgb-u8" else
              (lambda: engine.prepare_frames_yuv(src, name, (oh, ow), out=out)))
        for _ in range(20):
            fn()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n, ms = 0, 0.0
        while ms < 1000.0:
            a.record()
            for _ in range(200):
                fn()
            b.record()
            b.synchronize()
            ms += a.elapsed_time(b)
            n += 200
        in_bytes = src.numel()
        print(f"kernel {name:7s}: {ms * 1e3 / (n * T):7.2f} us/frame over {ms / 1e3:.2f} s  "
              f"({in_bytes // T} source bytes a frame)", flush=True)


def run_arms(arms, reps):
    """arms: name -> fn() returning results; alternate them reps times after one warm-up each.  -> name -> (wall ms
    list, cpu ms list, results of the last call)"""
    res = {k: ([], [], None) for k in arms}
    for k, fn in arms.items():
        fn()
    for _ in range(reps):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            c0, t0 = time.process_time(), time.perf_counter()
            out = fn()
            torch.cuda.synchronize()
            res[k][0].append((time.perf_counter() - t0) * 1e3)
            res[k][1].append((time.process_time() - c0) * 1e3)
            res[k] = (res[k][0], res[k][1], out)
    return res


def equal(a, b):
    if isinstance(a, (list, tuple, dict)):
        a, b = (list(a.values()), list(b.values())) if isinstance(a, dict) else (a, b)
        return len(a) == len(b) and all(equal(x, y) for x, y in zip(a, b))
    return torch.equal(a, b)


def report(title, res, unit="call"):
    ok = True
    first = next(iter(res.values()))[2]
    for k, (wall, cpu, out) in res.items():
        same = equal(out, first)
        ok &= same
        print(f"{title} {k:8s}: wall {statistics.median(wall):8.1f} ms/{unit}  host cpu {statistics.median(cpu):8.1f} "
              f"ms/{unit}  (runs {len(wall)}; results equal to yuv-i420: {same})", flush=True)
    return ok


def clip_bench(reps):
    p = CoTrackerPredictor(checkpoint=None, window_len=60)
    p.model.load_state_dict(seeded_state_dict(43, offline=True, window_len=60, head_gain=10.0, vis_gain=100.0))
    p = p.to(DEV)
    i420 = i420_clip(50, 1080, 1920, seed=2)
    rgb = yuv_to_rgb("i420", i420.to(DEV)).cpu()
    arms = {"yuv-i420": lambda: p(YUVClip(i420, "i420"), grid_size=10)}
    if cv2 is not None:
        arms["cv2-rgb"] = lambda: p(cv2_rgb(i420), grid_size=10)
    else:
        print("clip cv2-rgb : skipped (cv2 is not importable here)", flush=True)
    arms["rgb"] = lambda: p(rgb, grid_size=10)
    return report("clip", run_arms(arms, reps))


def streams_bench(steps):
    S, K, H, W = 16, 4, 720, 1280
    T = S + (steps + 1) * (S // 2)
    clips = [i420_clip(T, H, W, seed=10 + k) for k in range(K)]
    rgbs = [yuv_to_rgb("i420", c.to(DEV)).cpu() for c in clips]

    def predictor():
        p = CoTrackerOnlinePredictor(checkpoint=None, window_len=S)
        p.model.load_state_dict(seeded_state_dict(47, offline=False, window_len=S, head_gain=10.0, vis_gain=100.0))
        return p.to(DEV)

    def arm(chunk):
        hub = OnlineStreams(predictor())
        ids = [hub.open(frame_size=(H, W), grid_size=10) for _ in range(K)]
        state = {"t": 0}

        def step():
            t0 = state["t"]
            for k, sid in enumerate(ids):
                hub.push(sid, chunk(k, t0, t0 + S))
            state["t"] = t0 + S // 2
            return hub.step()
        return step

    makers = {"yuv-i420": lambda k, a, b: YUVClip(clips[k][:, a:b], "i420")}
    if cv2 is not None:
        makers["cv2-rgb"] = lambda k, a, b: cv2_rgb(clips[k][:, a:b])
    else:
        print("streams cv2-rgb : skipped (cv2 is not importable here)", flush=True)
    makers["rgb"] = lambda k, a, b: rgbs[k][:, a:b]
    fns = {k: arm(m) for k, m in makers.items()}
    return report("streams", run_arms(fns, steps), unit="step")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    print(f"card: {card()}", flush=True)
    print("computed: a 4:2:0 frame is 1.5 bytes a pixel to upload, against 3 for RGB", flush=True)
    torch.backends.cudnn.benchmark = False
    with torch.no_grad():
        kernel_bench()
        ok = clip_bench(args.reps)
        ok &= streams_bench(args.steps)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
