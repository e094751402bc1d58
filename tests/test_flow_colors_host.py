"""CPU tests of the visualiser's optical_flow mode: the ct3_render_flow_* symbols and their argument validation before
any launch, the numpy restatement of flow_vis (oracle/flow_vis_oracle.py) against hand-derived anchors and, when the
package is installed, against flow_vis itself, the attainable-colour bounds, and the constructor without matplotlib."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from cotracker_b200 import engine
from oracle import flow_vis_oracle as fv

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = ["ct3_render_flow_workspace_bytes", "ct3_render_flow_colors"]


def test_flow_symbols_exported_and_declared():
    lib = engine.lib()
    with open(os.path.join(ROOT, "include", "ct3_b200.h")) as f:
        header = f.read()
    for s in SYMBOLS:
        assert hasattr(lib, s) and s in engine.EXPORTED_SYMBOLS
        assert re.search(rf"int {s}\(", header)


def test_flow_rejects_bad_arguments_without_gpu():
    """Each invalid argument returns CT3_EINVAL before any launch: fake pointers and the legacy stream would fail
    differently if a launch were reached."""
    lib = engine.lib()
    p = ctypes.c_void_p
    n = ctypes.c_size_t(0)
    assert lib.ct3_render_flow_workspace_bytes(50, 72000, ctypes.byref(n)) == 0 and n.value >= 8
    need = n.value
    for args, msg in [((0, 10), b">= 1"), ((4, 0), b">= 1"), ((-1, 10), b">= 1"), ((70000, 40000), b"T * N")]:
        assert lib.ct3_render_flow_workspace_bytes(*args, ctypes.byref(n)) == -1, args
        assert msg in lib.ct3_last_error(), (args, lib.ct3_last_error())
    assert lib.ct3_render_flow_workspace_bytes(4, 10, None) == -1 and b"null argument" in lib.ct3_last_error()

    good = dict(pts=p(1 << 20), T=4, N=10, q=0, colors=p(1 << 22), ws=p(1 << 23), wsb=need)

    def call(**kw):
        a = dict(good, **kw)
        return lib.ct3_render_flow_colors(a["pts"], a["T"], a["N"], a["q"], a["colors"], a["ws"], a["wsb"], None)

    for kw, msg in [(dict(pts=None), b"null argument"), (dict(colors=None), b"null argument"),
                    (dict(ws=None), b"null argument"), (dict(T=0), b">= 1"), (dict(N=0), b">= 1"),
                    (dict(T=70000, N=40000), b"T * N"), (dict(q=4), b"query_frame"), (dict(q=-1), b"query_frame"),
                    (dict(wsb=need - 1), b"workspace too small"), (dict(wsb=0), b"workspace too small")]:
        assert call(**kw) == -1, kw
        assert msg in lib.ct3_last_error(), (kw, lib.ct3_last_error())


def test_flow_wrapper_rejects_host_tensors():
    with pytest.raises(engine.EngineError):
        engine.render_flow_colors(torch.zeros(2, 3, 2), 0)


def test_colorwheel_anchor_rows():
    w = fv.make_colorwheel()
    assert w.shape == (55, 3)
    # the first row of each segment: red, yellow, green, cyan, blue, magenta
    for row, rgb in [(0, (255, 0, 0)), (15, (255, 255, 0)), (21, (0, 255, 0)), (25, (0, 255, 255)),
                     (36, (0, 0, 255)), (49, (255, 0, 255))]:
        assert tuple(w[row]) == rgb, (row, w[row])
    # one step into RY and the last row of MR: floor(255 * i / n)
    assert tuple(w[1]) == (255, 17, 0) and tuple(w[54]) == (255, 0, 255 - 212)


def test_flow_to_color_anchors():
    zero = np.zeros((3, 5, 2), np.int64)
    assert (fv.flow_to_color(zero) == 255).all()                      # no motion: white (rad_max = 0)
    tracks = np.zeros((2, 4, 2), np.int64)
    tracks[1, :, 0] = [7, 3, 1, 100]                                      # pure +x motion
    c = fv.flow_to_color(tracks - tracks[0][None])
    assert (c[0] == 255).all()                                            # the query frame is white
    assert tuple(c[1, 3]) == (255, 0, 0)                                  # the largest +x motion is red
    assert (c[1, :, 0] == 255).all() and (c[1, :, 2] == c[1, :, 1]).all()   # smaller ones: paler red
    assert c.dtype == np.uint8 and c.shape == (2, 4, 3)


def _adversarial_tracks(rng, T=6, N=400, r=600):
    tracks = rng.integers(-r, r + 1, size=(T, N, 2)).astype(np.int64)
    rows = np.array([(1, 0), (-1, 0), (0, 1), (0, -1), (1, 1), (-1, 1), (1, -1), (-1, -1), (0, 0)], np.int64)
    for k, d in enumerate(rows):          # pure +-x, +-y, diagonals and zeros relative to frame 0
        tracks[:, k] = tracks[0, k] + d[None] * np.arange(T)[:, None] * (k + 3)
    return tracks


def test_attainable_is_singleton_exactly_where_perturbation_changes_nothing():
    rng = np.random.default_rng(11)
    tracks = _adversarial_tracks(rng)
    for q in (0, 3):
        lo, hi = fv.attainable(tracks, q)
        u, v = fv._normalised(tracks - tracks[q][None])
        at = np.arctan2(-v, -u)
        cols = [fv._colors(u, v, at)]
        for d in (np.inf, -np.inf):
            p = at
            for _ in range(fv.ULPS):
                p = np.nextafter(p, d)
                cols.append(fv._colors(u, v, p))
        cols = np.stack(cols)
        assert (lo == cols.min(0)).all() and (hi == cols.max(0)).all()
        assert ((lo == hi) == (cols == cols[0]).all(0)).all()
        # the unperturbed colours are flow_to_color's, and lie inside
        want = fv.flow_to_color(tracks - tracks[q][None])
        assert (cols[0] == want).all() and (lo <= want).all() and (want <= hi).all()


def test_restatement_matches_flow_vis_package():
    flow_vis = pytest.importorskip("flow_vis", reason="the flow_vis package is not installed on this host")
    rng = np.random.default_rng(5)
    for r in (3, 300, 5000):
        flow = rng.integers(-r, r + 1, size=(7, 900, 2)).astype(np.int64)
        assert np.array_equal(fv.flow_to_color(flow), flow_vis.flow_to_color(flow))


def test_optical_flow_constructor_without_cuda_or_matplotlib():
    """The mode's colours exist only on the GPU: without a CUDA device the constructor says so; with one it builds
    without matplotlib, imageio or flow_vis, and color_map stays None as in the reference."""
    code = ("import sys\n"
            "for m in ('imageio', 'matplotlib', 'flow_vis'):\n"
            "    sys.modules[m] = None   # import of any of them now fails\n"
            "import torch\n"
            "from cotracker.utils.visualizer import Visualizer\n"
            "try:\n"
            "    v = Visualizer(save_dir='./videos', pad_value=20, linewidth=1, mode='optical_flow')\n"
            "except NotImplementedError as e:\n"
            "    assert not torch.cuda.is_available() and 'CUDA' in str(e), e\n"
            "else:\n"
            "    assert torch.cuda.is_available() and v.mode == 'optical_flow' and v.color_map is None\n"
            "print('ok')\n")
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.join(ROOT, "dropin"), ROOT]))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0 and r.stdout.strip() == "ok", r.stderr
