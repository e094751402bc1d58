"""CPU tests of the track visualiser: the ct3_render_* symbols and their argument validation before any launch, the
drop-in import path without imageio or matplotlib, the host colour logic against the reference's recorded colours, and
a host restatement of the Pillow footprint rules that csrc/render.cu implements (disc, outline, thin and wide lines)
against the installed Pillow."""
import ctypes
import glob
import json
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from cotracker_b200 import engine
from cotracker_b200.visualizer import Visualizer
from oracle.make_visualizer_golden import CASES, StubColormap

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDENS = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "visualizer_*.npz")))
SYMBOLS = ["ct3_render_prepare", "ct3_render_workspace_bytes", "ct3_render_tracks"]


def test_render_symbols_exported_and_declared():
    lib = engine.lib()
    with open(os.path.join(ROOT, "include", "ct3_b200.h")) as f:
        header = f.read()
    for s in SYMBOLS:
        assert hasattr(lib, s) and s in engine.EXPORTED_SYMBOLS
        assert re.search(rf"int {s}\(", header)


def test_render_rejects_bad_arguments_without_gpu():
    """Each invalid argument returns CT3_EINVAL (a short workspace CT3_ENOSPC) before any launch: fake pointers and
    the legacy stream would fail differently if a launch were reached."""
    lib = engine.lib()
    p = ctypes.c_void_p
    src, out = p(1 << 20), p(1 << 24)
    ok = dict(src=src, dtype=0, T=4, H=90, W=120, st=3 * 90 * 120, sc=90 * 120, sh=120, sw=1, pad=8, gray=0, out=out)

    def prep(**kw):
        a = dict(ok, **kw)
        return lib.ct3_render_prepare(a["src"], a["dtype"], a["T"], a["H"], a["W"], a["st"], a["sc"], a["sh"], a["sw"],
                                      a["pad"], a["gray"], a["out"], None)

    for kw, msg in [(dict(src=None), b"null argument"), (dict(out=None), b"null argument"),
                    (dict(T=0), b">= 1"), (dict(W=0), b">= 1"), (dict(T=70000), b"65535"),
                    (dict(pad=-1), b"pad"), (dict(gray=2), b"grayscale"), (dict(dtype=3), b"unknown frame dtype"),
                    (dict(st=2 ** 62), b"stride extent"), (dict(H=50000, W=50000, pad=0), b"plane too large"),
                    (dict(pad=2 ** 30), b"plane too large")]:
        assert prep(**kw) == -1, kw
        assert msg in lib.ct3_last_error(), (kw, lib.ct3_last_error())

    n = ctypes.c_size_t(0)
    assert lib.ct3_render_workspace_bytes(4, 90, 120, 10, 0, ctypes.byref(n)) == 0 and n.value >= 4 * 90 * 120 * 4
    for args, msg in [((0, 90, 120, 10, 0), b">= 1"), ((4, 90, 120, 0, 0), b">= 1"), ((4, 90, 120, 10, -2), b"trail"),
                      ((4, 50000, 50000, 10, 0), b"plane too large"), ((60000, 9, 9, 40000, -1), b"T * N"),
                      ((70000, 9, 9, 1, 0), b"65535")]:
        assert lib.ct3_render_workspace_bytes(*args, ctypes.byref(n)) == -1, args
        assert msg in lib.ct3_last_error(), (args, lib.ct3_last_error())

    fr, pts, col, ws = p(1 << 20), p(1 << 21), p(1 << 22), p(1 << 23)
    good = dict(frames=fr, T=4, H=90, W=120, pts=pts, vis=None, colors=col, mask=None, N=10, radius=6, lw=3, trail=2,
                q=0, alphas=p(1 << 25), diff=None, ws=ws, wsb=1 << 30)

    def tracks(**kw):
        a = dict(good, **kw)
        return lib.ct3_render_tracks(a["frames"], a["T"], a["H"], a["W"], a["pts"], a["vis"], a["colors"], a["mask"],
                                     a["N"], a["radius"], a["lw"], a["trail"], a["q"], a["alphas"], a["diff"], a["ws"],
                                     a["wsb"], None)

    for kw, msg in [(dict(frames=None), b"null argument"), (dict(pts=None), b"null argument"),
                    (dict(colors=None), b"null argument"), (dict(ws=None), b"null argument"),
                    (dict(radius=-1), b"radius"), (dict(radius=256), b"radius"), (dict(lw=-1), b"linewidth"),
                    (dict(q=4), b"query_frame"), (dict(q=-1), b"query_frame"), (dict(alphas=None), b"alphas"),
                    (dict(trail=-3), b"trail"), (dict(N=0), b">= 1")]:
        assert tracks(**kw) == -1, kw
        assert msg in lib.ct3_last_error(), (kw, lib.ct3_last_error())
    assert tracks(wsb=16) == -3 and b"workspace too small" in lib.ct3_last_error()


def test_render_wrappers_reject_host_tensors():
    with pytest.raises(engine.EngineError):
        engine.render_prepare(torch.zeros(2, 3, 8, 8, dtype=torch.uint8), 2, False)
    with pytest.raises(engine.EngineError):
        engine.render_tracks(torch.zeros(2, 8, 8, 3, dtype=torch.uint8), torch.zeros(2, 1, 2), torch.zeros(2, 1, 3),
                             2, 1)


def test_dropin_import_without_imageio_or_matplotlib():
    code = ("import sys\n"
            "for m in ('imageio', 'matplotlib'):\n"
            "    sys.modules[m] = None   # import of either now fails\n"
            "from cotracker.utils.visualizer import Visualizer, read_video_from_path\n"
            "import cotracker.utils\n"
            "assert Visualizer.__module__ == 'cotracker_b200.visualizer', Visualizer.__module__\n"
            "assert read_video_from_path.__module__ == 'cotracker_b200.visualizer'\n"
            "v = Visualizer(pad_value=120, linewidth=3)\n"
            "try:\n"
            "    v.save_video(None, 'x')\n"
            "except ImportError as e:\n"
            "    assert 'imageio' in str(e)\n"
            "else:\n"
            "    raise AssertionError('save_video without imageio must raise ImportError')\n"
            "print('ok')\n")
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.join(ROOT, "dropin"), ROOT]))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0 and r.stdout.strip() == "ok", r.stderr


def test_unsupported_modes_raise():
    with pytest.raises(NotImplementedError, match="flow_vis"):
        Visualizer(mode="optical_flow")
    with pytest.raises(NotImplementedError, match="gt_tracks"):
        Visualizer().visualize(torch.zeros(1, 2, 3, 8, 8), torch.zeros(1, 2, 1, 2), gt_tracks=torch.zeros(1, 2, 1, 2))


@pytest.mark.parametrize("path", GOLDENS, ids=lambda p: os.path.basename(p)[11:-4])
def test_host_colours_match_reference(path):
    """The colours Visualizer computes on the host equal the ones the reference passed to draw_circle, point by point
    and in draw order (goldens record every call)."""
    z = np.load(path)
    params = json.loads(str(z["params"]))
    ctor, kw = params["ctor"], params["kw"]
    v = Visualizer(**ctor)
    v.color_map = StubColormap("gist_rainbow" if v.mode == "rainbow" else "cool")
    pad = v.pad_value
    tracks = torch.from_numpy(z["tracks"])
    T, N = tracks.shape[1], tracks.shape[2]
    segm = None
    if z["segm_mask"].size:
        c = tracks[0, 0].round().long()
        segm = torch.from_numpy(z["segm_mask"])[0, 0][c[:, 1], c[:, 0]].long().numpy()
    tl = (tracks[0] + pad).long().numpy()
    colors = v._colors(tl[0, :, 1], tl[0, :, 1], segm, T)
    comp = kw.get("compensate_for_camera_motion", False)
    want = [(int(tl[t, i, 0]), int(tl[t, i, 1])) + tuple(int(c) for c in colors[t, i])
            for t in range(T) for i in range(N)
            if tl[t, i, 0] != 0 and tl[t, i, 1] != 0 and (not comp or segm[i] > 0)]
    assert np.array_equal(np.array(want, dtype=np.int64).reshape(-1, 5), z["point_colors"])


# ---- Pillow footprint rules (restated from csrc/render.cu) -----------------------------------------------------------
def quarter_rows(r):
    a = 2 * r
    a2 = a * a

    def delta(x, y):
        return abs(a2 * y * y + a2 * x * x - a2 * a2)
    cx, cy, rows = a, 0, {}
    while True:
        lo, hi = rows.get(cy // 2, (cx // 2, cx // 2))
        rows[cy // 2] = (min(lo, cx // 2), max(hi, cx // 2))
        if cx == 0 and cy == a:
            return rows
        nx, ny, nd = cx, cy + 2, delta(cx, cy + 2)
        if nx > 1:
            d = delta(cx - 2, cy + 2)
            if nd > d:
                nx, ny, nd = cx - 2, cy + 2, d
            d = delta(cx - 2, cy)
            if nd > d:
                nx, ny = cx - 2, cy
        cx, cy = nx, ny


def footprint(r, fill):
    rows = quarter_rows(r)
    m = np.zeros((2 * r + 1, 2 * r + 1), bool)
    if fill and r == 0:
        return m
    for dy in range(-r, r + 1):
        lo, hi = rows[abs(dy)]
        for dx in range(-r, r + 1):
            m[dy + r, dx + r] = abs(dx) <= hi if fill else lo <= abs(dx) <= hi
    return m


def test_disc_and_outline_footprints_match_pillow():
    from PIL import Image, ImageDraw
    for r in range(0, 17):
        S = 2 * r + 1
        for fill in (True, False):
            for cx, cy in ((r + 3, r + 3), (1, 2), (-r, 4), (S + 2, S + 3)):   # inside, straddling, outside
                im = Image.new("RGB", (S + 6, S + 6))
                c = (255, 0, 0, 127)
                ImageDraw.Draw(im).ellipse([(cx - r, cy - r), (cx + r, cy + r)], fill=c if fill else None, outline=c)
                got = np.array(im)[..., 0] > 0
                want = np.zeros((S + 6 + 2 * S, S + 6 + 2 * S), bool)
                want[cy + S - r: cy + S + r + 1, cx + S - r: cx + S + r + 1] = footprint(r, fill)
                assert np.array_equal(got, want[S: S + S + 6, S: S + S + 6]), (r, fill, cx, cy)


def _f32(v):
    return np.float32(v)


def _round_up(f):
    f = _f32(f)
    return int(math.floor(_f32(f + _f32(0.5)))) if f >= 0 else -int(math.floor(_f32(abs(f) + _f32(0.5))))


def _round_down(f):
    f = _f32(f)
    return int(math.ceil(_f32(f - _f32(0.5)))) if f >= 0 else -int(math.ceil(_f32(abs(f) - _f32(0.5))))


def _put_span(img, xa, y, xb):
    H, W = img.shape
    if 0 <= y < H:
        xa, xb = min(xa, xb), max(xa, xb)
        xa, xb = max(xa, 0), min(xb, W - 1)
        if xa <= xb:
            img[y, xa: xb + 1] = True


def line_footprint(H, W, x0, y0, x1, y1, width):
    img = np.zeros((H, W), bool)
    if width <= 1:   # Bresenham, both endpoints: step i of the major axis -> minor0 + s*floor((2 dmin i + dmaj)/(2 dmaj))
        dx, dy = abs(x1 - x0), abs(y1 - y0)
        xs, ys = (1 if x1 >= x0 else -1), (1 if y1 >= y0 else -1)
        dmaj, dmin = (dx, dy) if dx > dy else (dy, dx)
        for i in range(dmaj + 1):
            k = 0 if dmaj == 0 else (2 * dmin * i + dmaj) // (2 * dmaj)
            x, y = (x0 + xs * i, y0 + ys * k) if dx > dy else (x0 + xs * k, y0 + ys * i)
            if 0 <= x < W and 0 <= y < H:
                img[y, x] = True
        return img
    dx, dy = x1 - x0, y1 - y0
    if dx == 0 and dy == 0:
        if 0 <= x0 < W and 0 <= y0 < H:
            img[y0, x0] = True
        return img
    big, small = math.hypot(dx, dy), (width - 1) / 2.0
    rup = int(math.floor(small + 0.5))
    rdn = int(math.ceil(small - 0.5))

    def rd(f):
        return int(math.ceil(f - 0.5)) if f >= 0 else -int(math.ceil(abs(f) - 0.5))
    rmax, rmin = rup / big, rdn / big
    dxmin, dxmax, dymin, dymax = rd(rmin * dy), rd(rmax * dy), rd(rmin * dx), rd(rmax * dx)
    v = [(x0 - dxmin, y0 + dymax), (x1 - dxmin, y1 + dymax), (x1 + dxmax, y1 - dymin), (x0 + dxmax, y0 - dymin)]
    edges = []
    for k in range(4):
        (ax, ay), (bx, by) = v[k], v[(k + 1) % 4]
        if ay == by:
            _put_span(img, min(ax, bx), ay, max(ax, bx))
        else:
            edges.append((ax, ay, min(ay, by), max(ay, by), _f32(_f32(bx - ax) / _f32(by - ay))))
    ylo, yhi = min(p[1] for p in v), max(p[1] for p in v)
    for y in range(max(ylo, 0), min(yhi, H - 1) + 1):
        xx = []
        for ax, ay, emin, emax, edx in edges:
            if emin <= y <= emax:
                xx.append(_f32(_f32(_f32(y - ay) * edx) + _f32(ax)))
                if y == emax and y < yhi:
                    xx.append(xx[-1])
        xx.sort()
        for k in range(1, len(xx), 2):
            _put_span(img, _round_up(xx[k - 1]), y, _round_down(xx[k]))
    return img


def test_line_footprints_match_pillow():
    from PIL import Image, ImageDraw
    rng = np.random.default_rng(7)
    H, W = 40, 48
    for n in range(3000):
        w = 1 + n % 4
        L = int(rng.choice([1, 3, 8, 25, 70]))
        x0, y0 = int(rng.integers(-12, W + 12)), int(rng.integers(-12, H + 12))
        x1, y1 = x0 + int(rng.integers(-L, L + 1)), y0 + int(rng.integers(-L, L + 1))
        im = Image.new("RGB", (W, H))
        ImageDraw.Draw(im).line((x0, y0, x1, y1), fill=(255, 0, 0), width=w)
        got = np.array(im)[..., 0] > 0
        assert np.array_equal(got, line_footprint(H, W, x0, y0, x1, y1, w)), (x0, y0, x1, y1, w)


def test_golden_cases_cover_the_issue_list():
    names = {os.path.basename(p)[11:-4] for p in GOLDENS}
    assert names == set(CASES)
