"""CPU tests of YUV input: the integer restatement of cv2's conversion against the cv2 goldens, YUVClip validation and
shape semantics, chunk planning with YUV frame bytes, and argument checks of engine.prepare_frames_yuv and
ct3_prepare_frames_yuv before any launch."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from cotracker_b200 import YUVClip, engine, ingest
from yuv_cases import LAYOUTS, pack, yuv_to_rgb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_restatement_equals_cv2_goldens():
    g = np.load(os.path.join(ROOT, "tests", "golden", "yuv_cv2.npz"))
    keys = [k for k in g.files if k.endswith("/yuv")]
    assert {k.split("/")[0] for k in keys} == set(LAYOUTS)
    assert {k.split("/")[1] for k in keys} == {"random", "odd", "tiny", "flat", "corners"}
    for k in keys:
        layout = k.split("/")[0]
        want = torch.from_numpy(g[k[:-len("yuv")] + "rgb"])
        assert torch.equal(yuv_to_rgb(layout, torch.from_numpy(g[k])), want), k
    # the corner case reaches both clamps of every channel
    rgb = g["nv12/corners/rgb"]
    assert all(rgb[:, c].min() == 0 and rgb[:, c].max() == 255 for c in range(3))


def test_pack_matches_golden_layouts():
    """The test helper packs planes the way the goldens (and cv2) lay them out."""
    g = np.load(os.path.join(ROOT, "tests", "golden", "yuv_cv2.npz"))
    for layout in LAYOUTS:
        f = torch.from_numpy(g[f"{layout}/flat/yuv"])
        H, W = (f.shape[1], f.shape[2]) if layout == "yuyv" else (f.shape[1] // 3 * 2, f.shape[2])
        Y = torch.arange(H * W, dtype=torch.uint8).reshape(H, W)
        cw = (H, W // 2) if layout == "yuyv" else (H // 2, W // 2)
        U, V = torch.full(cw, 7, dtype=torch.uint8), torch.full(cw, 9, dtype=torch.uint8)
        x = pack(layout, Y, U, V)
        assert tuple(x.shape) == tuple(f.shape[1:])
        assert int((x == 7).sum()) == U.numel() + int((Y == 7).sum())


def test_yuvclip_shape_semantics():
    for layout, data, hw in (("nv12", torch.zeros(2, 5, 36, 32, dtype=torch.uint8), (24, 32)),
                             ("i420", torch.zeros(1, 3, 45, 46, dtype=torch.uint8), (30, 46)),
                             ("yuyv", torch.zeros(1, 4, 7, 10, 2, dtype=torch.uint8), (7, 10))):
        c = YUVClip(data, layout)
        assert c.shape == torch.Size((data.shape[0], data.shape[1], 3) + hw)
        B, T, C, H, W = c.shape
        assert c.dim() == 5 and (C, H, W) == (3,) + hw
        assert c.device == torch.device("cpu") and not c.is_cuda
        assert c.data is data and c.layout == layout
        moved = c.to("cpu")
        assert isinstance(moved, YUVClip) and moved.shape == c.shape
    assert ingest.YUVClip is YUVClip


def test_yuvclip_rejects_bad_data():
    bad = [
        (torch.zeros(1, 2, 36, 32), "nv12"),                              # not uint8
        (torch.zeros(1, 2, 36, 32, dtype=torch.int16), "i420"),
        (np.zeros((1, 2, 36, 32), np.uint8), "nv12"),                     # not a tensor
        (torch.zeros(2, 36, 32, dtype=torch.uint8), "nv12"),              # rank
        (torch.zeros(1, 2, 36, 32, 2, dtype=torch.uint8), "i420"),
        (torch.zeros(1, 2, 24, 32, dtype=torch.uint8), "yuyv"),
        (torch.zeros(1, 2, 24, 32, 3, dtype=torch.uint8), "yuyv"),        # not Y/UV pairs
        (torch.zeros(1, 2, 35, 32, dtype=torch.uint8), "nv12"),           # rows not H*3/2
        (torch.zeros(1, 2, 36, 31, dtype=torch.uint8), "nv12"),           # odd W
        (torch.zeros(1, 2, 36, 31, dtype=torch.uint8), "i420"),
        (torch.zeros(1, 2, 24, 31, 2, dtype=torch.uint8), "yuyv"),
        (torch.zeros(0, 2, 36, 32, dtype=torch.uint8), "nv12"),           # B, T >= 1
        (torch.zeros(1, 0, 36, 32, dtype=torch.uint8), "nv12"),
        (torch.zeros(1, 2, 0, 32, dtype=torch.uint8), "nv12"),
        (torch.zeros(1, 2, 36, 32, dtype=torch.uint8), "nv21"),           # layout
        (torch.zeros(1, 2, 36, 32, dtype=torch.uint8), "NV12"),
    ]
    for data, layout in bad:
        with pytest.raises(ValueError):
            YUVClip(data, layout)
    YUVClip(torch.zeros(1, 2, 7, 32, 2, dtype=torch.uint8), "yuyv")      # odd H is fine for YUYV


def test_chunk_plan_with_yuv_frame_bytes():
    """A host YUVClip is staged by its YUV frame bytes: 1.5 H W (4:2:0) or 2 H W (YUYV), the bound of DESIGN.md 4.8
    unchanged."""
    slot = ingest.STAGING_SLOT_BYTES
    for layout, per_px in (("nv12", 1.5), ("i420", 1.5), ("yuyv", 2)):
        for H, W in ((1080, 1920), (720, 1280), (2, 2)):
            shape = (1, 50, H, W, 2) if layout == "yuyv" else (1, 50, H * 3 // 2, W)
            c = YUVClip(torch.empty(shape, dtype=torch.uint8), layout)
            fb = c.data[0, 0].numel()
            assert fb == int(per_px * H * W)
            plan = ingest.plan_chunks(50, fb)
            k = ingest.chunk_frames(50, fb)
            assert k == min(50, max(1, slot // fb))
            assert [t for a, b in plan for t in range(a, b)] == list(range(50))
            assert ingest.staging_bytes(50, fb) <= 2 * max(slot, fb)
    assert ingest.chunk_frames(50, 1920 * 1620) == slot // (1920 * 1620) == 10     # 1080p I420: 10 frames a slot
    assert ingest.chunk_frames(50, 3 * 1920 * 1080) == 5                          # against 5 of RGB


def test_prepare_frames_yuv_wrapper_rejects_without_gpu():
    x = torch.zeros(2, 36, 32, dtype=torch.uint8)
    for args in ((x, "nv12"), (x, "i420"), (torch.zeros(2, 24, 32, 2, dtype=torch.uint8), "yuyv")):
        with pytest.raises(engine.EngineError, match="CUDA"):
            engine.prepare_frames_yuv(*args, (16, 16))
    bad = [
        (x.float(), "nv12", "uint8"),
        (x, "nv21", "layout"),
        (torch.zeros(2, 35, 32, dtype=torch.uint8), "nv12", r"\[T,H\*3/2,W\]"),
        (torch.zeros(36, 32, dtype=torch.uint8), "i420", r"\[T,H\*3/2,W\]"),
        (torch.zeros(2, 24, 32, dtype=torch.uint8), "yuyv", r"\[T,H,W,2\]"),
        (torch.zeros(0, 36, 32, dtype=torch.uint8), "nv12", r"\[T,H\*3/2,W\]"),
        (torch.zeros(2, 36, 64, dtype=torch.uint8)[:, :, ::2], "nv12", "contiguous"),
        (torch.zeros(2, 24, 32, 2, dtype=torch.uint8).transpose(2, 3).contiguous().transpose(2, 3), "yuyv",
         "contiguous"),
    ]
    for src, layout, msg in bad:
        with pytest.raises(engine.EngineError, match=msg):
            engine.prepare_frames_yuv(src, layout, (16, 16))


def test_prepare_frames_yuv_exported_and_declared():
    lib = engine.lib()
    assert hasattr(lib, "ct3_prepare_frames_yuv") and "ct3_prepare_frames_yuv" in engine.EXPORTED_SYMBOLS
    with open(os.path.join(ROOT, "include", "ct3_b200.h")) as f:
        header = f.read()
    assert re.search(r"int ct3_prepare_frames_yuv\(", header)
    assert "CT3_YUV_NV12 = 0, CT3_YUV_I420 = 1, CT3_YUV_YUYV = 2" in header
    assert engine.YUV_LAYOUTS == {"nv12": 0, "i420": 1, "yuyv": 2}
    assert lib.ct3_version() == 102


def test_prepare_frames_yuv_rejects_bad_arguments_without_gpu():
    """Each invalid argument returns CT3_EINVAL with a message before any launch (fake pointers, legacy stream:
    reaching a launch would fail differently)."""
    lib = engine.lib()
    src, out = ctypes.c_void_p(1 << 20), ctypes.c_void_p(1 << 24)
    H, W = 90, 120
    ok = dict(src=src, layout=0, T=4, H=H, W=W, st=H * W * 3 // 2, sr=W, oh=384, ow=512, out=out)

    def call(**kw):
        a = dict(ok, **kw)
        return lib.ct3_prepare_frames_yuv(a["src"], a["layout"], a["T"], a["H"], a["W"], a["st"], a["sr"], a["oh"],
                                          a["ow"], a["out"], None)

    cases = [
        (dict(src=None), b"null argument"), (dict(out=None), b"null argument"),
        (dict(layout=3), b"unknown YUV layout"), (dict(layout=-1), b"unknown YUV layout"),
        (dict(T=0), b"must be >= 1"), (dict(H=0), b"must be >= 1"), (dict(W=-2), b"must be >= 1"),
        (dict(oh=0), b"must be >= 1"), (dict(ow=0), b"must be >= 1"),
        (dict(H=91), b"even width and height"), (dict(W=121), b"even width and height"),
        (dict(layout=1, H=91), b"even width and height"),
        (dict(layout=2, W=121, sr=242), b"even width"),
        (dict(sr=W - 1), b"row stride is below"),
        (dict(sr=-W), b"row stride is below"),
        (dict(layout=2, sr=2 * W - 1), b"row stride is below"),
        (dict(layout=1, sr=W + 64), b"I420 rows must be dense"),
        (dict(st=2 ** 62), b"stride extent"),                        # 3 frames of 2^62 bytes
        (dict(st=-(2 ** 63)), b"stride extent"),
        (dict(sr=2 ** 60), b"stride extent"),                        # 134 rows of 2^60 bytes
        (dict(oh=65536, ow=32768), b"output plane too large"),
        (dict(T=2 ** 31 - 1, oh=1, ow=2 ** 31 - 1, st=0), b"output too large"),
    ]
    for kw, msg in cases:
        assert call(**kw) == -1, kw
        assert msg in lib.ct3_last_error(), (kw, lib.ct3_last_error())
