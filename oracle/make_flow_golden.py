"""Generate tests/golden/flowvis_*.npz: the UNMODIFIED reference visualiser (cotracker/utils/visualizer.py,
Visualizer.visualize with save_video=False) in mode="optical_flow" on small seeded clips and tracks.  Run in the build
container only (the GPU box has no reference checkout):

    python oracle/make_flow_golden.py

imageio and matplotlib are stubbed as for make_visualizer_golden.py, and flow_vis by its numpy restatement
(oracle/flow_vis_oracle.py).  Each file holds the inputs (video, tracks, visibility, segm_mask), the parameters as
JSON, the uint8 output [1,T',3,H',W'], the [T,N,3] colours flow_to_color returned to the reference (vector_colors) and
their attainable range lo / hi under +-4-ulp arctan2 (flow_vis_oracle.attainable).  The files are named flowvis_* so
that the visualizer_* goldens, which other tests enumerate, stay exactly the set make_visualizer_golden.py writes.
"""
from __future__ import annotations

import json
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import flow_vis_oracle  # noqa: E402
from oracle.make_visualizer_golden import GOLDEN_DIR, REF, install_stubs  # noqa: E402

H, W = 96, 128

# name -> (constructor kwargs, visualize kwargs, input options)
CASES = {
    "notebook": (dict(pad_value=20, linewidth=1), {}, dict(dtype="uint8")),
    "query_frame": (dict(pad_value=4, linewidth=2, show_first_frame=0), dict(query_frame=3), dict(dtype="float32")),
    "trace3": (dict(pad_value=6, linewidth=2, show_first_frame=0, tracks_leave_trace=3), dict(query_frame=2),
               dict(dtype="uint8", jumps=True)),
    "trace_inf": (dict(pad_value=0, linewidth=1, show_first_frame=2, tracks_leave_trace=-1), dict(query_frame=2),
                  dict(dtype="float32", vis4=True)),
    "compensate": (dict(pad_value=10, linewidth=2, show_first_frame=0, tracks_leave_trace=4),
                   dict(compensate_for_camera_motion=True), dict(dtype="uint8", segm=True)),
    "gray_opacity": (dict(pad_value=6, linewidth=3, grayscale=True, show_first_frame=1), dict(opacity=0.5),
                     dict(dtype="float32")),
    "offframe": (dict(pad_value=3, linewidth=2, show_first_frame=0), {}, dict(dtype="uint8", edges=True)),
    "motionless": (dict(pad_value=5, linewidth=2, show_first_frame=0, tracks_leave_trace=-1), {},
                   dict(dtype="uint8", still=True)),
    "t1": (dict(pad_value=2, linewidth=2), {}, dict(dtype="uint8", T=1)),
}


def case_inputs(name: str):
    """Seeded inputs of one case: video [1,T,3,H,W], tracks [1,T,N,2] fp32, visibility, segm_mask [1,1,H,W] or None."""
    _, _, opt = CASES[name]
    T, N = opt.get("T", 8), 24
    rng = np.random.default_rng(sum(map(ord, name)) * 104729)
    t, c, y, x = np.meshgrid(np.arange(T), np.arange(3), np.arange(H), np.arange(W), indexing="ij")
    base = (x * (2 + c) + y * (3 - c) + 9 * t + 40 * c + 8 * rng.integers(0, 4, size=(T, 3, H // 8, W // 8)).repeat(
        8, axis=2).repeat(8, axis=3)) % 256
    base = base[None]
    video = base.astype(np.uint8) if opt["dtype"] == "uint8" else (base + 0.25 * (x % 4)[None]).astype(np.float32)
    start = np.stack([rng.uniform(2, W - 3, N), rng.uniform(2, H - 3, N)], axis=1)
    step = rng.normal(0, 6 if opt.get("jumps") else 2.5, size=(T, N, 2))
    step[0] = 0
    if opt.get("still"):
        step[:] = 0
    tr = start[None] + np.cumsum(step, axis=0)
    if opt.get("edges"):
        # zero x, zero y, off-frame, negative, straddling every border, and one far outlier that sets rad_max
        tr[2, 0, 0] = 0.4;   tr[3, 1, 1] = -0.6;   tr[4, 2] = (-40.0, 30.0)
        tr[1, 3] = (-2.5, 50.0);  tr[5, 4] = (W + 1.2, 40.0);  tr[2, 5] = (60.0, -3.3);  tr[6, 6] = (70.0, H + 2.7)
        tr[3, 7] = (-1.5, -2.5);  tr[4, 8] = (W + 3.0, H + 1.0);  tr[5, 9] = (1e4, -1e4)
        tr[1:, 10] = tr[1:, 10] * 0 + (W - 1.0, H - 1.0)
    tracks = tr[None].astype(np.float32)
    vis = rng.random((1, T, N)) > 0.35
    if opt.get("vis4"):
        vis = vis[..., None].astype(np.float32)
    segm = None
    if opt.get("segm"):
        segm = (rng.random((1, 1, H, W)) > 0.5).astype(np.float32)
        c = tracks[0, 0].round().astype(int)
        bg = segm[0, 0, c[:, 1], c[:, 0]] <= 0
        cam = np.cumsum(rng.normal(0, 2, size=(T, 2)), axis=0).astype(np.float32)
        tr0 = tracks[0]
        tr0[:, bg] = tr0[0, bg][None] + cam[:, None]
    return video, tracks, vis, segm


def main():
    sys.path.insert(0, REF)
    install_stubs()
    recorded = []
    stub = types.ModuleType("flow_vis")

    def flow_to_color(flow_uv, clip_flow=None, convert_to_bgr=False):
        out = flow_vis_oracle.flow_to_color(flow_uv, clip_flow, convert_to_bgr)
        recorded.append(out.copy())
        return out
    stub.flow_to_color = flow_to_color
    sys.modules["flow_vis"] = stub
    import torch
    from cotracker.utils.visualizer import Visualizer
    for name, (ctor, kw, _) in CASES.items():
        video, tracks, vis, segm = case_inputs(name)
        recorded.clear()
        v = Visualizer(save_dir="/nonexistent", mode="optical_flow", **ctor)
        out = v.visualize(torch.from_numpy(video), torch.from_numpy(tracks), torch.from_numpy(vis),
                          segm_mask=None if segm is None else torch.from_numpy(segm), save_video=False, **kw)
        assert len(recorded) == 1
        colors = recorded[0]
        lo, hi = flow_vis_oracle.attainable((torch.from_numpy(tracks) + v.pad_value)[0].long().numpy(),
                                            kw.get("query_frame", 0))
        assert (lo <= colors).all() and (colors <= hi).all()
        path = os.path.join(GOLDEN_DIR, f"flowvis_{name}.npz")
        np.savez_compressed(path, video=video, tracks=tracks, visibility=vis,
                            segm_mask=np.zeros(0) if segm is None else segm, out=out.numpy(),
                            vector_colors=colors, lo=lo, hi=hi,
                            params=np.array(json.dumps(dict(ctor=dict(ctor, mode="optical_flow"), kw=kw))))
        print(name, out.shape, "sensitive entries:", int((lo != hi).any(-1).sum()), "of", lo.shape[0] * lo.shape[1],
              os.path.getsize(path))


if __name__ == "__main__":
    main()
