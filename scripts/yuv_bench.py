"""YUV input, measured: the conversion kernel, a host 1080p clip through CoTrackerPredictor, and host 720p streams.

    python scripts/yuv_bench.py [--reps 3] [--steps 10] [--compare-lib PATH] [--parts kernel,clip,streams]

Seeded weights (cotracker_b200.synthetic) and seeded smooth random clips.  Prints the card's name, power limit and max
SM clock, then:
  1. kernel: 1080 x 1920 -> 384 x 512, 8 frames a launch, CUDA events over >= 1 s of launches: us per frame, for
     ct3_prepare_frames_yuv on nv12, i420 and yuyv (default colour), ct3_prepare_frames_yuv_fmt on every other layout
     (BT.601 limited, and BT.709 limited for the runtime-coefficient path of 8-bit layouts), and ct3_prepare_frames on
     the uint8 RGB clip [T,3,H,W], each called straight through ctypes (class Build).
     --compare-lib PATH: another build of libct3_b200.so (e.g. the parent commit's).  Its ct3_prepare_frames_yuv on
     nv12, i420 and yuyv is timed in rounds alternating with this build's, and both builds' outputs must be
     torch.equal.
  2. clip: a host 1080p clip of 50 frames through CoTrackerPredictor(grid_size=10), the arms alternating after one
     warm-up call each: wall ms (ending in a synchronise) and host CPU ms (time.process_time) per call, median.
       yuv-i420  : the decoder's I420 frames as a YUVClip;
       cv2-rgb   : cv2.cvtColor(COLOR_YUV2RGB_I420) per frame on the host, then the RGB clip (skipped without cv2);
       rgb       : the RGB clip already converted (conversion not counted), for the upload alone.
     and, as a second group on the same clip at 10 bits (yuv420p10, BT.709 limited range):
       yuv-p10   : the frames as a YUVClip;
       host-p10  : converted to uint8 RGB on the host by the integer formula (tests/yuv_color_cases.py's, in torch
                   int64 frame by frame with the chroma terms at chroma resolution; counted), then the RGB clip.
     A 16-bit 4:2:0 frame is 3 bytes a pixel, as uint8 RGB is, so the two upload the same bytes: the difference is
     the host conversion.  Neither arm counts decoding.
  3. streams: OnlineStreams with four host 720p streams (window 16, grid 10), one 16-frame chunk (8 new frames) per
     stream and step, the first three arms: ms per step (push + step, ending in a synchronise), median over --steps
     steps.
Every arm's results are compared with torch.equal against its group's first arm; the script exits non-zero if any
differ.
"""
from __future__ import annotations

import argparse
import ctypes
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
import yuv_color_cases  # noqa: E402
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


def timed(fn, T, seconds=1.0):
    """us per frame of fn() (T frames a launch), CUDA events over >= `seconds` of launches after 20 warm-up calls."""
    for _ in range(20):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n, ms = 0, 0.0
    while ms < seconds * 1e3:
        a.record()
        for _ in range(200):
            fn()
        b.record()
        b.synchronize()
        ms += a.elapsed_time(b)
        n += 200
    return ms * 1e3 / (n * T), ms / 1e3


class Build:
    """One build of libct3_b200.so, its frame entry points called straight through ctypes with their arguments packed
    once: an 8-frame launch takes ~20 us of GPU time, less than engine.prepare_frames_yuv's argument checks take on
    the host, so timing through the Python wrappers would time the host."""

    def __init__(self, path):
        self.path = os.path.abspath(path)
        self.lib = ctypes.CDLL(self.path)
        i, i64, p = ctypes.c_int, ctypes.c_int64, ctypes.c_void_p
        for name, args in (("ct3_prepare_frames", [p, i, i, i, i, i64, i64, i64, i64, i, i, p, p]),
                           ("ct3_prepare_frames_yuv", [p, i, i, i, i, i64, i64, i, i, p, p]),
                           ("ct3_prepare_frames_yuv_fmt", [p, i, i, i, i, i, i, i64, i64, i, i, p, p])):
            fn = getattr(self.lib, name, None)
            if fn is not None:
                fn.restype, fn.argtypes = i, args

    def yuv(self, src, layout, out, matrix="bt601"):
        """A call of ct3_prepare_frames_yuv (the three original layouts in BT.601 limited range) or of
        ct3_prepare_frames_yuv_fmt on src -> out, ready to repeat: () -> None."""
        H, W = engine.yuv_frame_hw(layout, src.shape)
        es, stream = src.element_size(), torch.cuda.current_stream().cuda_stream
        tail = (src.shape[0], H, W, src.stride(0) * es, src.stride(1) * es, out.shape[2], out.shape[3], out.data_ptr(),
                stream)
        if layout in engine.YUV_LAYOUTS and matrix == "bt601":
            fn, args = self.lib.ct3_prepare_frames_yuv, (src.data_ptr(), engine.YUV_LAYOUTS[layout]) + tail
        else:
            fn = self.lib.ct3_prepare_frames_yuv_fmt
            args = (src.data_ptr(), engine.YUV_FORMATS[layout], engine.YUV_MATRICES[matrix], 0) + tail
        return self._checked(fn, args)

    def rgb(self, src, out):
        T, _, H, W = src.shape
        args = (src.data_ptr(), engine.FRAME_DTYPES[src.dtype], T, H, W, *src.stride(), out.shape[2], out.shape[3],
                out.data_ptr(), torch.cuda.current_stream().cuda_stream)
        return self._checked(self.lib.ct3_prepare_frames, args)

    def _checked(self, fn, args):
        if fn(*args) != 0:
            raise RuntimeError(f"{self.path}: {self.lib.ct3_last_error()}")
        return lambda: fn(*args)


def kernel_bench(compare_lib=None):
    H, W, T, oh, ow = 1080, 1920, 8, 384, 512
    srcs = {name: yuv_color_cases.random_frames(name, (T,), H, W, seed=1 + i).to(DEV)
            for i, name in enumerate(yuv_color_cases.FORMATS)}
    g = torch.Generator().manual_seed(1)
    rgb = torch.randint(0, 256, (T, 3, H, W), generator=g, dtype=torch.uint8).to(DEV)
    out = torch.empty(T, 3, oh, ow, device=DEV)
    this = Build(engine.LIB_PATH)
    arms = [("rgb-u8", "", this.rgb(rgb, out), rgb)]
    for name, src in srcs.items():
        for m in ["bt601"] + (["bt709"] if src.dtype == torch.uint8 else []):
            arms.append((name, m, this.yuv(src, name, out, m), src))
    for name, m, fn, src in arms:
        us, s = timed(fn, T)
        entry = "ct3_prepare_frames" if name == "rgb-u8" else \
            "ct3_prepare_frames_yuv" if name in engine.YUV_LAYOUTS and m == "bt601" else "ct3_prepare_frames_yuv_fmt"
        print(f"kernel {name:9s} {m:6s}: {us:7.2f} us/frame over {s:.2f} s  ({src[0].numel() * src.element_size()} "
              f"source bytes a frame; {entry})", flush=True)
    if compare_lib is None:
        return True
    other = Build(compare_lib)
    ok = True
    for name in engine.YUV_LAYOUTS:
        src = srcs[name]
        mine, theirs = torch.empty_like(out), torch.empty_like(out)
        this.yuv(src, name, mine)
        other.yuv(src, name, theirs)
        torch.cuda.synchronize()
        same = torch.equal(mine, theirs)
        ok &= same
        t_mine, t_theirs = [], []
        for _ in range(5):                     # alternating rounds of >= 0.5 s each
            t_mine.append(timed(this.yuv(src, name, out), T, 0.5)[0])
            t_theirs.append(timed(other.yuv(src, name, out), T, 0.5)[0])
        print(f"kernel {name:9s} this build {statistics.median(t_mine):7.3f} us/frame, other build "
              f"{statistics.median(t_theirs):7.3f} us/frame (median of 5 alternating rounds: "
              f"{' '.join(f'{x:.3f}' for x in t_mine)} | {' '.join(f'{x:.3f}' for x in t_theirs)}); outputs equal: "
              f"{same}", flush=True)
    return ok


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
    first_arm = next(iter(res))
    first = res[first_arm][2]
    for k, (wall, cpu, out) in res.items():
        same = equal(out, first)
        ok &= same
        print(f"{title} {k:8s}: wall {statistics.median(wall):8.1f} ms/{unit}  host cpu {statistics.median(cpu):8.1f} "
              f"ms/{unit}  (runs {len(wall)}; results equal to {first_arm}: {same})", flush=True)
    return ok


def host_yuv420p10_bt709(frame):
    """One yuv420p10 frame [H*3/2,W] -> uint8 RGB [3,H,W] on the host: the integer formula of yuv_color_cases in torch
    int64, with the chroma terms at chroma resolution and broadcast over their 2x2 blocks (the restatement itself
    repeats the chroma planes first and is ~50x slower)."""
    k = yuv_color_cases.coeffs("bt709", False, 10)
    cy, crv, cgv, cgu, cbu = k["c"]
    H, W = frame.shape[0] // 3 * 2, frame.shape[1]
    flat = frame.long().reshape(-1) & 1023
    q = H * W // 4
    y = (flat[:H * W].reshape(H // 2, 2, W // 2, 2) - k["yoff"]).clamp_(min=k["ylo"]).mul_(cy)
    u = flat[H * W:H * W + q].view(H // 2, 1, W // 2, 1) - k["coff"]
    v = flat[H * W + q:].view(H // 2, 1, W // 2, 1) - k["coff"]
    h = 1 << (k["shift"] - 1)
    out = torch.empty(3, H // 2, 2, W // 2, 2, dtype=torch.uint8)
    for c, chroma in enumerate((crv * v + h, h - cgv * v - cgu * u, cbu * u + h)):
        out[c] = ((y + chroma) >> k["shift"]).clamp_(0, 255)
    return out.view(3, H, W)


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
    ok = report("clip", run_arms(arms, reps))

    # the same clip at 10 bits: each sample v becomes v << 2 | v >> 6, in the same planar 4:2:0 layout
    p10 = ((i420.long() << 2) | (i420.long() >> 6)).to(torch.uint16)

    first = p10[0, 0]
    assert torch.equal(host_yuv420p10_bt709(first), yuv_color_cases.yuv_to_rgb("yuv420p10", first, "bt709"))

    def host_p10():
        out = torch.empty(p10.shape[:2] + (3, 1080, 1920), dtype=torch.uint8)
        for t in range(p10.shape[1]):
            out[0, t] = host_yuv420p10_bt709(p10[0, t])
        return p(out, grid_size=10)

    arms = {"yuv-p10": lambda: p(YUVClip(p10, "yuv420p10", matrix="bt709"), grid_size=10), "host-p10": host_p10}
    return ok & report("clip10", run_arms(arms, reps))


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
    ap.add_argument("--compare-lib", default=None, help="another build of libct3_b200.so to time the old entry against")
    ap.add_argument("--parts", default="kernel,clip,streams")
    args = ap.parse_args()
    parts = set(args.parts.split(","))
    print(f"card: {card()}", flush=True)
    print("computed: an 8-bit 4:2:0 frame is 1.5 bytes a pixel to upload, a 16-bit one 3, against 3 for uint8 RGB",
          flush=True)
    torch.backends.cudnn.benchmark = False
    ok = True
    with torch.no_grad():
        if "kernel" in parts:
            ok &= kernel_bench(args.compare_lib)
        if "clip" in parts:
            ok &= clip_bench(args.reps)
        if "streams" in parts:
            ok &= streams_bench(args.steps)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
