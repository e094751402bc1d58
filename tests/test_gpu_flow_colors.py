"""GPU tests of the visualiser's optical_flow mode (ct3_render_flow_colors).

Against every flowvis_* golden of the unmodified reference (oracle/make_flow_golden.py), from host and device inputs,
uint8 and float:
  (a) the kernel's colours lie in the fixture's attainable range lo..hi and equal the reference's where lo == hi;
  (b) the drawing fed the fixture's colours reproduces the reference's frames bit for bit;
  (c) the public visualize() equals the drawing fed the kernel's own colours.
Then a dense-scale random field against this host's attainable range, and the notebook's dense cell end to end."""
import glob
import json
import os

import numpy as np
import pytest
import torch

from cotracker_b200 import engine
from cotracker_b200.visualizer import Visualizer
from oracle import flow_vis_oracle as fv

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDENS = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "flowvis_*.npz")))


def _check_in_range(got: np.ndarray, lo: np.ndarray, hi: np.ndarray, want: np.ndarray = None):
    outside = ((got < lo) | (got > hi)).any(-1)
    assert not outside.any(), f"{int(outside.sum())} colours outside the attainable set, first at {np.argwhere(outside)[0]}"
    if want is not None:
        fixed = (lo == hi).all(-1)
        bad = fixed & (got != want).any(-1)
        assert not bad.any(), f"{int(bad.sum())} exact colours differ, first at {np.argwhere(bad)[0]}"


def test_goldens_cover_the_cases():
    from oracle.make_flow_golden import CASES
    assert {os.path.basename(p)[8:-4] for p in GOLDENS} == set(CASES)


@pytest.mark.parametrize("where", ["host", "device"])
@pytest.mark.parametrize("path", GOLDENS, ids=lambda p: os.path.basename(p)[8:-4])
def test_golden(path, where, monkeypatch):
    z = np.load(path)
    params = json.loads(str(z["params"]))
    ctor, kw = params["ctor"], params["kw"]
    dev = "cuda" if where == "device" else "cpu"
    q = kw.get("query_frame", 0)
    tracks = torch.from_numpy(z["tracks"])

    # (a) the kernel's colours
    pts = (tracks[0] + ctor["pad_value"]).cuda().contiguous()
    got = engine.render_flow_colors(pts, q).cpu().numpy()
    _check_in_range(got, z["lo"], z["hi"], z["vector_colors"])

    video = torch.from_numpy(z["video"])
    videos = [video, video.float() if video.dtype == torch.uint8 else
              video.permute(0, 1, 3, 4, 2).contiguous().permute(0, 1, 4, 2, 3)]
    segm = torch.from_numpy(z["segm_mask"]).to(dev) if z["segm_mask"].size else None
    want = torch.from_numpy(z["out"])
    real = engine.render_flow_colors
    for vid in videos:
        def run(colors=None):
            if colors is not None:
                monkeypatch.setattr(engine, "render_flow_colors", lambda p, qf: torch.from_numpy(colors).to(p.device))
            try:
                return Visualizer(save_dir="/nonexistent", **ctor).visualize(
                    vid.to(dev), tracks.to(dev), torch.from_numpy(z["visibility"]).to(dev), segm_mask=segm,
                    save_video=False, **kw)
            finally:
                monkeypatch.setattr(engine, "render_flow_colors", real)

        # (b) the reference's colours drawn by render_tracks give the reference's frames
        drawn = run(z["vector_colors"])
        assert drawn.dtype == torch.uint8 and drawn.shape == want.shape
        bad = (drawn != want).any(dim=2)
        assert not bad.any(), f"{int(bad.sum())} pixels differ, first at {bad.nonzero()[0].tolist()}"
        # (c) visualize() draws the kernel's colours
        out = run()
        assert out.device.type == "cpu" and torch.equal(out, run(got))
        if np.array_equal(got, z["vector_colors"]):
            assert torch.equal(out, want)


def test_motionless_is_white_and_plus_x_is_red():
    T, N = 5, 300
    pts = torch.rand(1, N, 2, device="cuda").mul(200).expand(T, N, 2).contiguous()
    assert (engine.render_flow_colors(pts, 2) == 255).all()
    pts = pts.clone()
    pts[:, :, 0] += torch.arange(T, device="cuda", dtype=torch.float32)[:, None] * 7   # pure +x motion from frame 0
    c = engine.render_flow_colors(pts, 0)
    assert (c[0] == 255).all() and (c[-1] == torch.tensor([255, 0, 0], dtype=torch.uint8, device="cuda")).all()


def _dense_field(T=50, N=72000, r=600, seed=0):
    rng = np.random.default_rng(seed)
    base = rng.uniform(-50, 1000, size=(1, N, 2))
    disp = rng.integers(-r, r + 1, size=(T, N, 2)).astype(np.float64)
    rows = np.array([(1, 0), (-1, 0), (0, 1), (0, -1), (1, 1), (-1, 1), (1, -1), (-1, -1), (0, 0)], np.float64)
    for k, d in enumerate(rows):           # pure +-x, +-y, diagonals and zeros at several speeds
        for s in range(40):
            disp[:, 9 * s + k] = d[None] * np.arange(T)[:, None] * (s + 1)
    frac = rng.uniform(0, 0.999, size=(T, N, 2))
    return (base + disp + frac).astype(np.float32)


def test_dense_random_field_within_attainable_set():
    T, N, q = 50, 72000, 20
    pts = torch.from_numpy(_dense_field(T, N))
    tracks = pts.long().numpy()                                     # the reference's .long()
    lo, hi = fv.attainable(tracks, q)
    got = engine.render_flow_colors(pts.cuda(), q).cpu().numpy()
    host = fv.flow_to_color(tracks - tracks[q][None])
    print(f"{int((got != host).any(-1).sum())} of {T * N} entries differ from this host's numpy; "
          f"{int((lo != hi).any(-1).sum())} have more than one attainable colour")
    _check_in_range(got, lo, hi, host)
    again = engine.render_flow_colors(pts.cuda(), q).cpu().numpy()
    assert np.array_equal(got, again)


def test_dropin_draws_optical_flow_without_flow_vis():
    """The reference's import path, with imageio, matplotlib and flow_vis unavailable, draws the mode."""
    import subprocess
    import sys
    code = ("import sys\n"
            "for m in ('imageio', 'matplotlib', 'flow_vis'):\n"
            "    sys.modules[m] = None   # import of any of them now fails\n"
            "import torch\n"
            "from cotracker.utils.visualizer import Visualizer\n"
            "v = Visualizer(save_dir='./videos', pad_value=20, linewidth=1, mode='optical_flow')\n"
            "assert v.color_map is None\n"
            "video = torch.zeros(1, 4, 3, 32, 48, device='cuda')\n"
            "tracks = torch.tensor([[5.0, 6.0], [20.0, 9.0]], device='cuda')[None, None].repeat(1, 4, 1, 1)\n"
            "tracks[0, :, 1, 0] += torch.arange(4, device='cuda') * 3   # track 1 moves in +x: red\n"
            "out = v.visualize(video, tracks, save_video=False)\n"
            "assert out.shape == (1, 13, 3, 72, 88), out.shape\n"
            "assert out[0, -1, :, 29, 20 + 9 + 20].tolist() == [255, 0, 0], out[0, -1, :, 29, 49]\n"
            "print('ok')\n")
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.join(ROOT, "dropin"), ROOT]))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0 and r.stdout.strip() == "ok", r.stderr


def test_notebook_dense_cell_end_to_end():
    """The notebook's last cell with random weights: dense tracking with backward tracking on a 50 x 200 x 360 clip
    (72 000 tracks), then Visualizer(mode="optical_flow", pad_value=20, linewidth=1).visualize(save_video=False)."""
    from cotracker_b200.synthetic import texture_video
    torch.manual_seed(0)
    model = torch.hub.load(ROOT, "cotracker3_offline", source="local", pretrained=False).to("cuda")
    T, H, W, pad = 50, 200, 360, 20
    video = texture_video(T, H, W, seed=3).cuda()
    with torch.no_grad():
        tracks, vis = model(video, grid_query_frame=20, backward_tracking=True)
    N = tracks.shape[2]
    assert tracks.shape == (1, T, 72000, 2) and N == 72000 and torch.isfinite(tracks).all()
    v = Visualizer(save_dir="./videos", pad_value=pad, linewidth=1, mode="optical_flow")
    v.visualize(video, tracks, vis, save_video=False)                # warm-up (module load, allocator)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    a = v.visualize(video, tracks, vis, save_video=False)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    Hp, Wp = H + 2 * pad, W + 2 * pad
    frame = Hp * Wp * 3
    # the padded clip, its show_first_frame gather, one int32 key per pixel, the padded tracks, the colours and the
    # visibility mask, plus 64 MiB
    bound = T * frame + (T - 1 + 10) * frame + T * Hp * Wp * 4 + T * N * 2 * 4 + T * N * 3 + 2 * T * N + (64 << 20)
    print(f"visualize peak {peak / 2**20:.1f} MiB, bound {bound / 2**20:.1f} MiB")
    assert peak < bound, (peak, bound)
    assert a.shape == (1, T - 1 + 10, 3, Hp, Wp) and a.dtype == torch.uint8
    b = v.visualize(video, tracks, vis, save_video=False)
    assert torch.equal(a, b)
    tl = (tracks[0] + pad).long().cpu().numpy()
    lo, hi = fv.attainable(tl, 0)
    got = engine.render_flow_colors((tracks[0] + pad).contiguous(), 0).cpu().numpy()
    _check_in_range(got, lo, hi, fv.flow_to_color(tl - tl[0][None]))
