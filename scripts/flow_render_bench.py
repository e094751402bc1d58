"""Time the visualiser's optical_flow mode on the reference notebook's dense cell at its real size: a 50 x 200 x 360
clip, one track per pixel (N = 72 000), pad_value 20, linewidth 1.

    python scripts/flow_render_bench.py                       # GPU: kernels, visualize(save_video=False), peak memory
    python scripts/flow_render_bench.py --reference --frames 5   # CPU: the reference's draw_tracks_on_video

GPU times are CUDA-event times over --iters calls after one warm-up, printed with the card's name, power limit and max
SM clock:
  - colors_ms: ct3_render_flow_colors alone;
  - kernels_ms: ct3_render_prepare + ct3_render_flow_colors + ct3_render_tracks on device inputs;
  - visualize_ms: the whole visualize(save_video=False) call on device inputs, including the show_first_frame gather
    and the copy of the finished frames to the host;
  - peak_mib: the device memory visualize() allocates above what its inputs hold.
The reference mode stubs imageio and matplotlib (oracle/make_visualizer_golden.py) and flow_vis (its numpy restatement,
oracle/flow_vis_oracle.py), and times one draw_tracks_on_video call on the first --frames frames on this host's CPU.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

T, H, W, PAD, LW = 50, 200, 360, 20, 1


def inputs(T, device, seed=0):
    g = torch.Generator().manual_seed(seed)
    video = torch.randint(0, 256, (1, T, 3, H, W), dtype=torch.uint8, generator=g).float()
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    start = torch.stack([xs.flatten(), ys.flatten()], dim=1)
    tracks = (start[None] + torch.cumsum(torch.randn(T, H * W, 2, generator=g) * 1.5, dim=0))[None]
    vis = torch.rand(1, T, H * W, generator=g) > 0.2
    return video.to(device), tracks.to(device), vis.to(device)


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def gpu(args):
    from cotracker_b200 import engine
    from cotracker_b200.visualizer import Visualizer
    from scripts.render_bench import card
    assert torch.cuda.is_available(), "the GPU mode needs a CUDA device"
    print(json.dumps({"card": card(), "torch": torch.__version__}))
    video, tracks, vis = inputs(args.frames, "cuda")
    Tn, N = args.frames, H * W
    v = Visualizer(save_dir="./videos", pad_value=PAD, linewidth=LW, mode="optical_flow")
    pts = (tracks[0] + PAD).contiguous()
    visu8 = vis[0].to(torch.uint8).contiguous()
    ws = torch.empty(engine.render_workspace_bytes(Tn, H + 2 * PAD, W + 2 * PAD, N, 0), dtype=torch.uint8,
                     device="cuda")

    def kernels():
        f = engine.render_prepare(video[0], PAD, False)
        engine.render_tracks(f, pts, engine.render_flow_colors(pts, 0), 2 * LW, LW, visible=visu8, workspace=ws)
    ms_colors = timed(lambda: engine.render_flow_colors(pts, 0), args.iters)
    ms_k = timed(kernels, args.iters)
    ms_vis = timed(lambda: v.visualize(video, tracks, vis, save_video=False), args.iters)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = v.visualize(video, tracks, vis, save_video=False)
    torch.cuda.synchronize()
    peak = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    print(json.dumps({"workload": "notebook_dense_optical_flow", "T": Tn, "HxW": f"{H}x{W}", "pad": PAD, "N": N,
                      "linewidth": LW, "colors_ms": round(ms_colors, 3), "kernels_ms": round(ms_k, 3),
                      "visualize_ms": round(ms_vis, 2), "peak_mib": round(peak, 1), "out": list(out.shape)}))


def reference(args):
    ref = os.environ.get("COTRACKER_REFERENCE", "/root/reference")
    sys.path.insert(0, ref)
    from oracle import flow_vis_oracle
    from oracle.make_visualizer_golden import install_stubs
    install_stubs()
    sys.modules["flow_vis"] = flow_vis_oracle
    import torch.nn.functional as F
    from cotracker.utils.visualizer import Visualizer
    video, tracks, vis = inputs(T, "cpu")
    video, tracks, vis = video[:, : args.frames], tracks[:, : args.frames], vis[:, : args.frames]
    v = Visualizer(pad_value=PAD, linewidth=LW, mode="optical_flow")
    vp = F.pad(video, (PAD,) * 4, "constant", 255)
    t0 = time.perf_counter()
    v.draw_tracks_on_video(vp, tracks + PAD, vis)
    s = time.perf_counter() - t0
    print(json.dumps({"host": "reference on CPU", "cpus": len(os.sched_getaffinity(0)), "T": args.frames,
                      "N": H * W, "reference_cpu_s": round(s, 2), "per_frame_s": round(s / args.frames, 3)}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", action="store_true")
    ap.add_argument("--frames", type=int, default=None, help="clip length (GPU default 50, reference default 5)")
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if args.frames is None:
        args.frames = 5 if args.reference else T
    reference(args) if args.reference else gpu(args)


if __name__ == "__main__":
    main()
