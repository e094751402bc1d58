"""Generate tests/golden/visualizer_*.npz by running the UNMODIFIED reference visualiser
(cotracker/utils/visualizer.py, Visualizer.visualize with save_video=False) on small seeded clips and tracks.  Run in
the build container only (the GPU box has no reference checkout):

    python oracle/make_visualizer_golden.py

imageio and matplotlib are not needed: stub modules are placed in sys.modules before the reference is imported.  The
stub colour map (StubColormap, a fixed piecewise-linear RGBA table) and Normalize ((v - vmin) / (vmax - vmin) in
float64) are what tests/test_gpu_visualizer.py sets on cotracker_b200's Visualizer as well, so both draw with the same
colours.  Each file holds the inputs (video, tracks, visibility, segm_mask), the parameters as JSON and the uint8
output [1,T',3,H',W'].
"""
from __future__ import annotations

import json
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("COTRACKER_REFERENCE", "/root/reference")
GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")

# piecewise-linear RGBA table: (position, r, g, b, a)
_TABLE = np.array([
    (0.00, 0.90, 0.10, 0.20, 1.0),
    (0.20, 0.95, 0.60, 0.05, 1.0),
    (0.45, 0.30, 0.85, 0.15, 1.0),
    (0.70, 0.10, 0.55, 0.95, 1.0),
    (1.00, 0.65, 0.20, 0.80, 1.0),
])


class StubColormap:
    """Callable like a matplotlib colour map: a float in [0, 1] -> RGBA tuple, an array -> [n, 4] float64."""

    def __init__(self, name: str):
        self.name = name
        self.shift = 0.0 if name == "gist_rainbow" else 0.25   # "cool" gets a different table

    def _rgba(self, x):
        x = np.clip(np.asarray(x, dtype=np.float64), 0.0, 1.0)
        x = np.where(x + self.shift > 1.0, x + self.shift - 1.0, x + self.shift) if self.shift else x
        return np.stack([np.interp(x, _TABLE[:, 0], _TABLE[:, c]) for c in range(1, 5)], axis=-1)

    def __call__(self, x):
        out = self._rgba(x)
        return tuple(float(v) for v in out) if out.ndim == 1 else out


def stub_normalize(vmin, vmax):
    def norm(v):
        return 0.0 if float(vmin) == float(vmax) else (np.float64(v) - np.float64(vmin)) / (np.float64(vmax) - np.float64(vmin))
    return norm


def install_stubs():
    """Stub imageio / matplotlib modules for the reference's module-level imports."""
    mpl = types.ModuleType("matplotlib")
    cm = types.ModuleType("matplotlib.cm")
    cm.get_cmap = StubColormap
    plt = types.ModuleType("matplotlib.pyplot")
    plt.Normalize = stub_normalize
    mpl.cm, mpl.pyplot = cm, plt
    io = types.ModuleType("imageio")

    def _missing(*a, **k):
        raise RuntimeError("imageio stub")
    io.get_reader = io.get_writer = _missing
    sys.modules.update({"matplotlib": mpl, "matplotlib.cm": cm, "matplotlib.pyplot": plt, "imageio": io})


H, W, T, N = 96, 128, 8, 24

# name -> (constructor kwargs, visualize kwargs, input options)
CASES = {
    "demo": (dict(pad_value=12, linewidth=3, show_first_frame=10), {}, dict(dtype="uint8")),
    "lw1_trace3": (dict(pad_value=0, linewidth=1, show_first_frame=0, tracks_leave_trace=3), {}, dict(dtype="float32")),
    "lw2_trace_inf": (dict(pad_value=5, linewidth=2, show_first_frame=2, tracks_leave_trace=-1), {},
                      dict(dtype="uint8", vis4=True)),
    "opacity": (dict(pad_value=4, linewidth=3, show_first_frame=1), dict(opacity=0.5), dict(dtype="uint8")),
    "gray_float": (dict(pad_value=6, linewidth=2, grayscale=True, show_first_frame=0), {}, dict(dtype="float32")),
    "gray_uint8": (dict(pad_value=6, linewidth=2, grayscale=True, show_first_frame=3), {}, dict(dtype="uint8")),
    "cool": (dict(pad_value=3, linewidth=3, mode="cool", show_first_frame=0), {}, dict(dtype="uint8")),
    "segm_rainbow": (dict(pad_value=8, linewidth=2, show_first_frame=0), {}, dict(dtype="uint8", segm=True)),
    "segm_cool": (dict(pad_value=8, linewidth=2, mode="cool", show_first_frame=0), {}, dict(dtype="uint8", segm=True)),
    "trace3": (dict(pad_value=12, linewidth=3, show_first_frame=0, tracks_leave_trace=3), {},
               dict(dtype="uint8", jumps=True)),
    "trace_inf_lw3": (dict(pad_value=0, linewidth=3, show_first_frame=0, tracks_leave_trace=-1), {},
                      dict(dtype="float32", jumps=True)),
    "compensate": (dict(pad_value=10, linewidth=2, show_first_frame=0, tracks_leave_trace=4),
                   dict(compensate_for_camera_motion=True), dict(dtype="uint8", segm=True)),
}


def case_inputs(name: str):
    """Seeded inputs of one case: video [1,T,3,H,W], tracks [1,T,N,2] fp32, visibility, segm_mask [1,1,H,W] or None."""
    _, _, opt = CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)) * 7919)
    # a smooth moving pattern (compresses well) with coarse noise; float clips get fractional parts in quarters
    t, c, y, x = np.meshgrid(np.arange(T), np.arange(3), np.arange(H), np.arange(W), indexing="ij")
    base = (x * (2 + c) + y * (3 - c) + 9 * t + 40 * c + 8 * rng.integers(0, 4, size=(T, 3, H // 8, W // 8)).repeat(
        8, axis=2).repeat(8, axis=3)) % 256
    base = base[None]
    video = base.astype(np.uint8) if opt["dtype"] == "uint8" else (base + 0.25 * (x % 4)[None]).astype(np.float32)
    # tracks: a seeded walk; frame 0 inside the frame (segm lookups need it), later frames free to leave it
    start = np.stack([rng.uniform(2, W - 3, N), rng.uniform(2, H - 3, N)], axis=1)
    step = rng.normal(0, 6 if opt.get("jumps") else 2.5, size=(T, N, 2))
    step[0] = 0
    tr = start[None] + np.cumsum(step, axis=0)
    if not opt.get("segm"):
        # edge cases at later frames: zero x, zero y, off-frame, negative, straddling every border
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
        # background tracks move together (the camera), foreground ones on their own
        c = tracks[0, 0].round().astype(int)
        bg = segm[0, 0, c[:, 1], c[:, 0]] <= 0
        cam = np.cumsum(rng.normal(0, 2, size=(T, 2)), axis=0).astype(np.float32)
        tr0 = tracks[0]
        tr0[:, bg] = tr0[0, bg][None] + cam[:, None]
    return video, tracks, vis, segm


def main():
    sys.path.insert(0, REF)
    install_stubs()
    import torch
    import cotracker.utils.visualizer as refvis
    from cotracker.utils.visualizer import Visualizer
    draw_circle = refvis.draw_circle
    for name, (ctor, kw, _) in CASES.items():
        video, tracks, vis, segm = case_inputs(name)
        # the colour of every point the reference draws, in draw order: (x, y, r, g, b) per call
        calls = []

        def recording_circle(rgb, coord, radius, color=(255, 0, 0), visible=True, color_alpha=None):
            calls.append((int(coord[0]), int(coord[1])) + tuple(int(c) for c in color))
            return draw_circle(rgb, coord, radius, color, visible, color_alpha)
        refvis.draw_circle = recording_circle
        v = Visualizer(save_dir="/nonexistent", **ctor)
        v.color_map = StubColormap("gist_rainbow" if ctor.get("mode", "rainbow") == "rainbow" else "cool")
        out = v.visualize(torch.from_numpy(video), torch.from_numpy(tracks), torch.from_numpy(vis),
                          segm_mask=None if segm is None else torch.from_numpy(segm), save_video=False, **kw)
        out = out.numpy()
        path = os.path.join(GOLDEN_DIR, f"visualizer_{name}.npz")
        np.savez_compressed(path, video=video, tracks=tracks, visibility=vis,
                            segm_mask=np.zeros(0) if segm is None else segm, out=out,
                            point_colors=np.array(calls, dtype=np.int64).reshape(-1, 5),
                            params=np.array(json.dumps(dict(ctor=ctor, kw=kw))))
        print(name, out.shape, os.path.getsize(path))


if __name__ == "__main__":
    main()
