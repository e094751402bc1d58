"""GPU tests of the track visualiser: every golden of the unmodified reference (oracle/make_visualizer_golden.py)
reproduced bitwise from host and device inputs, uint8 and float, and a grid-80 x 50-frame run with trails that stays
under a memory bound computed from shapes and repeats exactly."""
import glob
import json
import os

import numpy as np
import pytest
import torch

from cotracker_b200.visualizer import Visualizer
from oracle.make_visualizer_golden import StubColormap

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDENS = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "visualizer_*.npz")))


def _visualizer(ctor):
    v = Visualizer(save_dir="/nonexistent", **ctor)
    v.color_map = StubColormap("gist_rainbow" if v.mode == "rainbow" else "cool")
    return v


@pytest.mark.parametrize("where", ["host", "device"])
@pytest.mark.parametrize("path", GOLDENS, ids=lambda p: os.path.basename(p)[11:-4])
def test_golden_bitwise(path, where):
    z = np.load(path)
    params = json.loads(str(z["params"]))
    dev = "cuda" if where == "device" else "cpu"
    video = torch.from_numpy(z["video"])
    videos = [video]
    if video.dtype == torch.uint8:
        videos.append(video.float())                                   # the same pixels as float: the same frames
    else:
        videos.append(video.permute(0, 1, 3, 4, 2).contiguous().permute(0, 1, 4, 2, 3))   # channels-last strides
    segm = torch.from_numpy(z["segm_mask"]).to(dev) if z["segm_mask"].size else None
    want = torch.from_numpy(z["out"])
    for vid in videos:
        out = _visualizer(params["ctor"]).visualize(vid.to(dev), torch.from_numpy(z["tracks"]).to(dev),
                                                    torch.from_numpy(z["visibility"]).to(dev), segm_mask=segm,
                                                    save_video=False, **params["kw"])
        assert out.device.type == "cpu" and out.dtype == torch.uint8 and out.shape == want.shape
        bad = (out != want).any(dim=2)
        assert not bad.any(), f"{int(bad.sum())} pixels differ, first at {bad.nonzero()[0].tolist()}"


def test_draw_tracks_on_video_matches_visualize():
    """draw_tracks_on_video on an already padded clip gives what visualize gives on the unpadded one."""
    z = np.load(os.path.join(ROOT, "tests", "golden", "visualizer_demo.npz"))
    params = json.loads(str(z["params"]))
    v = _visualizer(params["ctor"])
    p = v.pad_value
    video = torch.nn.functional.pad(torch.from_numpy(z["video"]).cuda(), (p, p, p, p), "constant", 255)
    out = v.draw_tracks_on_video(video, torch.from_numpy(z["tracks"]).cuda() + p, torch.from_numpy(z["visibility"]))
    assert torch.equal(out, torch.from_numpy(z["out"]))


def test_grid80_trails_memory_and_repeatability():
    """50 frames, 6400 tracks, trails of 8 steps at 360x640 + pad: peak device memory stays under the clip, its
    padded copy, one int32 key per pixel and the show_first_frame gather, plus 64 MiB; two runs give the same frames."""
    torch.manual_seed(0)
    T, H, W, G, pad = 50, 360, 640, 80, 20
    video = torch.randint(0, 256, (1, T, 3, H, W), dtype=torch.uint8, device="cuda")
    ys, xs = torch.meshgrid(torch.linspace(8, H - 8, G), torch.linspace(8, W - 8, G), indexing="ij")
    start = torch.stack([xs.flatten(), ys.flatten()], dim=1).cuda()
    walk = torch.cumsum(torch.randn(T, G * G, 2, device="cuda") * 3, dim=0)
    tracks = (start[None] + walk)[None]
    vis = torch.rand(1, T, G * G, device="cuda") > 0.2
    v = Visualizer(pad_value=pad, linewidth=3, tracks_leave_trace=8, show_first_frame=4)
    v.color_map = StubColormap("gist_rainbow")
    v.visualize(video, tracks, vis, save_video=False)          # warm-up (module load, allocator)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    a = v.visualize(video, tracks, vis, save_video=False)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    Hp, Wp = H + 2 * pad, W + 2 * pad
    frame = Hp * Wp * 3
    bound = T * frame + T * Hp * Wp * 4 + (T - 1 + 4) * frame + 64 * 2 ** 20
    assert peak < bound, (peak, bound)
    b = v.visualize(video, tracks, vis, save_video=False)
    assert torch.equal(a, b)
    assert a.shape == (1, T - 1 + 4, 3, Hp, Wp)
    # something was drawn beyond the padding and the clip
    assert (a[0, -1].permute(1, 2, 0) != torch.nn.functional.pad(video[0, -1].cpu(), (pad,) * 4, value=255)
            .permute(1, 2, 0)).any()
