"""Time the track visualiser on the demo workloads (50 x 720 x 1296 clip, pad_value 120, linewidth 3):
grid 10 and grid 80 without trails, grid 80 with tracks_leave_trace = 8 and = -1.

    python scripts/render_bench.py                 # GPU: visualize(save_video=False) and the kernels alone
    python scripts/render_bench.py --reference     # CPU: the reference's draw_tracks_on_video (needs its checkout)

GPU times are CUDA-event times over --iters calls after one warm-up, printed with the card's name, power limit and
max SM clock.  visualize() includes the upload of host-side colours, the gather of the show_first_frame copies and
the copy of the finished frames to the host; "kernels" is ct3_render_prepare + ct3_render_tracks on device inputs.
The reference mode stubs imageio and matplotlib (oracle/make_visualizer_golden.py) and times one call per workload
on this host's CPU; --frames shortens the clip there.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = [("grid10", 10, 0), ("grid80", 80, 0), ("grid80_trace8", 80, 8), ("grid80_trace-1", 80, -1)]


def inputs(T, H, W, G, device, seed=0):
    g = torch.Generator().manual_seed(seed)
    video = torch.randint(0, 256, (1, T, 3, H, W), dtype=torch.uint8, generator=g)
    ys, xs = torch.meshgrid(torch.linspace(8, H - 8, G), torch.linspace(8, W - 8, G), indexing="ij")
    start = torch.stack([xs.flatten(), ys.flatten()], dim=1)
    tracks = (start[None] + torch.cumsum(torch.randn(T, G * G, 2, generator=g) * 3, dim=0))[None]
    vis = torch.rand(1, T, G * G, generator=g) > 0.2
    return video.to(device), tracks.to(device), vis.to(device)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})"


def gpu(args):
    from cotracker_b200 import engine
    from cotracker_b200.visualizer import Visualizer
    from oracle.make_visualizer_golden import StubColormap
    assert torch.cuda.is_available(), "the GPU mode needs a CUDA device"
    print(json.dumps({"card": card(), "torch": torch.__version__}))
    for name, G, trace in WORKLOADS:
        video, tracks, vis = inputs(args.frames, 720, 1296, G, "cuda")
        v = Visualizer(pad_value=120, linewidth=3, tracks_leave_trace=trace)
        v.color_map = StubColormap("gist_rainbow")   # matplotlib's colour maps cost the same host time per track
        out = v.visualize(video, tracks, vis, save_video=False)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.iters):
            out = v.visualize(video, tracks, vis, save_video=False)
        b.record()
        torch.cuda.synchronize()
        ms_vis = a.elapsed_time(b) / args.iters
        # kernels alone, on the same device inputs
        T, N = args.frames, G * G
        pts = (tracks[0] + 120).contiguous()
        colors = torch.randint(0, 256, (T, N, 3), dtype=torch.uint8, device="cuda")
        visu8 = vis[0].to(torch.uint8).contiguous()
        S = min(trace, T - 1) if trace > 0 else T - 1
        alphas = torch.rand(T, max(S, 1), 2, dtype=torch.float64, device="cuda") if trace > 0 else None
        Hp, Wp = 720 + 240, 1296 + 240
        ws = torch.empty(engine.render_workspace_bytes(T, Hp, Wp, N, trace), dtype=torch.uint8, device="cuda")

        def kernels():
            f = engine.render_prepare(video[0], 120, False)
            engine.render_tracks(f, pts, colors, 6, 3, trail=trace, visible=visu8, alphas=alphas, workspace=ws)
        kernels()
        torch.cuda.synchronize()
        a.record()
        for _ in range(args.iters):
            kernels()
        b.record()
        torch.cuda.synchronize()
        ms_k = a.elapsed_time(b) / args.iters
        print(json.dumps({"workload": name, "T": T, "HxW": "720x1296", "pad": 120, "N": N, "trace": trace,
                          "visualize_ms": round(ms_vis, 2), "kernels_ms": round(ms_k, 2), "out": list(out.shape)}))


def reference(args):
    ref = os.environ.get("COTRACKER_REFERENCE", "/root/reference")
    sys.path.insert(0, ref)
    from oracle.make_visualizer_golden import StubColormap, install_stubs
    install_stubs()
    import torch.nn.functional as F
    from cotracker.utils.visualizer import Visualizer
    print(json.dumps({"host": "reference on CPU", "cpus": len(os.sched_getaffinity(0))}))
    for name, G, trace in WORKLOADS:
        if args.only and name not in args.only:
            continue
        video, tracks, vis = inputs(args.frames, 720, 1296, G, "cpu")
        v = Visualizer(pad_value=120, linewidth=3, tracks_leave_trace=trace)
        v.color_map = StubColormap("gist_rainbow")
        vp = F.pad(video, (120,) * 4, "constant", 255)
        t0 = time.perf_counter()
        v.draw_tracks_on_video(vp, tracks + 120, vis)
        s = time.perf_counter() - t0
        print(json.dumps({"workload": name, "T": args.frames, "N": G * G, "trace": trace,
                          "reference_cpu_s": round(s, 2)}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", action="store_true")
    ap.add_argument("--frames", type=int, default=50)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--only", nargs="*")
    args = ap.parse_args()
    reference(args) if args.reference else gpu(args)


if __name__ == "__main__":
    main()
