"""CPU tests of YUV colour and the layouts beyond NV12 / I420 / YUYV: the integer formula of ct3_prepare_frames_yuv_fmt
(restated in tests/yuv_color_cases.py) against its float64 definition and against cv2, the sample containers, YUVClip
validation and colour propagation, chunk planning with 2-byte samples, and argument checks of
engine.prepare_frames_yuv and ct3_prepare_frames_yuv_fmt before any launch."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import yuv_cases
import yuv_color_cases as C
from cotracker_b200 import YUVClip, engine, ingest
from cotracker_b200.corners import clip_frame

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# The exact rounding ties among the 8-bit triples (255 X = k + 1/2 in exact arithmetic), all full-range BT.601:
# B = Y + 1.772 (U - 128) at U = 3, 253 and G = Y - 0.714136 (V - 128) - 0.344136 (U - 128) at (U, V) = (78, 178),
# (178, 78).  There the float64 value may land on either side, so the formula is not held to it.

def _tie_mask(matrix, full_range, channel, U, V):
    if (matrix, full_range) != ("bt601", True) or channel == 0:
        return torch.zeros_like(U, dtype=torch.bool)
    if channel == 2:
        return (U == 3) | (U == 253)
    return ((U == 78) & (V == 178)) | ((U == 178) & (V == 78))


@pytest.mark.parametrize("colour", C.DERIVED, ids=lambda c: f"{c[0]}-{'full' if c[1] else 'limited'}")
def test_formula_equals_float64_on_every_8bit_triple(colour):
    matrix, full = colour
    s = torch.arange(256, dtype=torch.int64)
    U, V = (x.reshape(-1) for x in torch.meshgrid(s, s, indexing="ij"))
    near_ties = 0
    for y0 in range(0, 256, 32):                       # 32 luma values a chunk: 2M triples
        Y = torch.arange(y0, y0 + 32)[:, None].expand(-1, U.numel()).reshape(-1)
        UU, VV = U.repeat(32), V.repeat(32)
        got = C.convert(Y[:, None, None], UU[:, None, None], VV[:, None, None], matrix, full, 8)
        got = got.reshape(-1, 3).long()
        want, dist = C.round_exact(C.exact(Y.double(), UU.double(), VV.double(), matrix, full, 8))
        for c in range(3):
            tie = _tie_mask(matrix, full, c, UU, VV)
            near = dist[:, c] < 1e-9
            assert torch.equal(near, tie), (colour, c, y0)           # the listed ties, and no other triple near one
            assert torch.equal(got[~tie, c], want[~tie, c].long()), (colour, c, y0)
            assert float(dist[~tie, c].min()) > 100 * C.coeff_error_bound(8)
            near_ties += int(tie.sum())
    assert near_ties == (131072 + 512 if colour == ("bt601", True) else 0)


@pytest.mark.parametrize("bits", (10, 16))
@pytest.mark.parametrize("colour", C.DERIVED, ids=lambda c: f"{c[0]}-{'full' if c[1] else 'limited'}")
def test_formula_equals_float64_at_10_and_16_bits(colour, bits):
    """Every Y value against a sampled chroma set (the range ends, the midpoints, random pairs)."""
    matrix, full = colour
    g = torch.Generator().manual_seed(bits)
    top, mid = (1 << bits) - 1, 1 << (bits - 1)
    ends = torch.tensor([[0, top, mid, mid - 1, 0, top, 16 << (bits - 8)], [0, top, mid, mid, top, 0, 240 << (bits - 8)]])
    ch = torch.cat([ends, torch.randint(0, top + 1, (2, 57), generator=g)], 1)
    Y = torch.arange(top + 1)[:, None].expand(-1, ch.shape[1]).reshape(-1)
    U, V = ch[0].repeat(top + 1), ch[1].repeat(top + 1)
    got = C.convert(Y[:, None, None], U[:, None, None], V[:, None, None], matrix, full, bits).reshape(-1, 3).long()
    want, dist = C.round_exact(C.exact(Y.double(), U.double(), V.double(), matrix, full, bits))
    far = dist >= 1e-9
    assert torch.equal(got[far], want.long()[far])
    assert int((~far).sum()) < 64                              # ties are rare and only excused there


def test_bt601_limited_is_cv2_restatement_at_8_bits():
    for layout in yuv_cases.LAYOUTS:
        data = C.random_frames(layout, (3,), 24, 32, seed=1)
        assert torch.equal(C.yuv_to_rgb(layout, data), yuv_cases.yuv_to_rgb(layout, data)), layout
    g = np.load(os.path.join(ROOT, "tests", "golden", "yuv_cv2.npz"))
    for k in (k for k in g.files if k.endswith("/yuv")):
        layout = k.split("/")[0]
        assert torch.equal(C.yuv_to_rgb(layout, torch.from_numpy(g[k])), torch.from_numpy(g[k[:-3] + "rgb"])), k
    # the same constants at every depth: a 10-bit sample 4v converts as the 8-bit sample v
    data = C.random_frames("nv12", (2,), 24, 32, seed=2)
    wide = C.pack("p010", *(C.containers("p010", p << 2) for p in _nv12_planes(data)))
    assert torch.equal(C.yuv_to_rgb("p010", wide), yuv_cases.yuv_to_rgb("nv12", data))


def _nv12_planes(data):
    H = data.shape[-2] // 3 * 2
    uv = data[..., H:, :].long()
    return data[..., :H, :].long(), uv[..., 0::2], uv[..., 1::2]


def test_ignored_bits_change_nothing():
    """Junk in P010's low 6 bits or in yuv4xxp10's top 6 bits is not part of the sample."""
    for layout in ("p010", "yuv420p10", "yuv422p10", "yuv444p10"):
        junk = C.random_frames(layout, (2,), 16, 20, seed=3, junk=True)
        clean = C.random_frames(layout, (2,), 16, 20, seed=3, junk=False)
        assert not torch.equal(junk, clean)
        for m, f in C.COLOURS:
            assert torch.equal(C.yuv_to_rgb(layout, junk, m, f), C.yuv_to_rgb(layout, clean, m, f)), (layout, m, f)


def test_planes_and_packing_of_every_layout():
    """pack and planes are inverse on every layout, and the planar shapes are the documented ones."""
    H, W = 6, 8
    for layout, (dtype, bits, _, family, xs, ys) in C.FORMATS.items():
        data = C.random_frames(layout, (2,), H, W, seed=4, junk=False)
        assert data.dtype == dtype
        want = (2, H, W, 2) if layout == "yuyv" else (2, {3: H * 3 // 2, 4: 2 * H, 6: 3 * H}[
            engine._YUV_ROWS[layout]], W)
        assert tuple(data.shape) == want and engine.yuv_frame_hw(layout, data.shape) == (H, W), layout
        assert C.frame_hw(layout, data.shape) == (H, W) and engine.yuv_subsampling(layout) == (xs, ys)
        Y, U, V = C.planes(layout, data)
        assert Y.shape == U.shape == V.shape == (2, H, W)
        # the chroma sample of pixel (y, x) is the one of (y >> ys << ys, x >> xs << xs)
        assert torch.equal(U, U[:, (torch.arange(H) >> ys) << ys][:, :, (torch.arange(W) >> xs) << xs])


@pytest.mark.parametrize("bits", (8, 16))
def test_full_range_bt601_meets_cv2(bits):
    """cv2.cvtColor(COLOR_YCrCb2RGB) is full-range BT.601 on 4:4:4 Y, Cr, Cb frames; at 16 bits its 16-bit RGB is
    scaled to 8.  Both round on their own, so they agree within 1."""
    g = np.load(os.path.join(ROOT, "tests", "golden", "yuv_color_cv2.npz"))
    y, u, v = (torch.from_numpy(g[f"{bits}/{k}"].astype(np.int64)) for k in "yuv")
    want = torch.from_numpy(g[f"{bits}/rgb"].astype(np.int64))
    if bits == 16:
        want = torch.div(2 * want + 257, 514, rounding_mode="floor")      # round(x / 257)
    full = lambda c: c.repeat_interleave(2, -2).repeat_interleave(2, -1)   # noqa: E731
    layouts = ("nv12", "i420", "yuv444p") if bits == 8 else ("p016",)
    for layout in layouts:
        planes = (y, full(u), full(v)) if layout == "yuv444p" else (y, u, v)
        got = C.yuv_to_rgb(layout, C.pack(layout, *planes), "bt601", True).long()
        d = (got - want).abs()
        assert int(d.max()) <= 1 and float((d > 0).float().mean()) < 0.05, layout
    assert int(want.min()) == 0 and int(want.max()) == 255


def test_yuvclip_new_layouts_shape_and_colour():
    for layout in C.NEW_LAYOUTS:
        data = C.random_frames(layout, (2, 3), 6, 8, seed=5)
        c = YUVClip(data, layout, matrix="bt709", full_range=True)
        assert c.shape == torch.Size((2, 3, 3, 6, 8)) and c.dim() == 5 and not c.is_cuda
        assert (c.layout, c.matrix, c.full_range) == (layout, "bt709", True) and c.data is data
        assert "bt709 full range" in repr(c) and layout in repr(c)
        for d in (c.to("cpu"), clip_frame(c, 1)):
            assert isinstance(d, YUVClip) and (d.layout, d.matrix, d.full_range) == (layout, "bt709", True)
        assert torch.equal(clip_frame(c, 1).data, data[:, 1:2])
    d = YUVClip(torch.zeros(1, 2, 36, 32, dtype=torch.uint8), "nv12")
    assert (d.matrix, d.full_range) == ("bt601", False) and repr(d) == "YUVClip(nv12, shape=(1, 2, 3, 24, 32), device=cpu)"
    assert clip_frame(YUVClip(d.data, "i420", matrix="bt2020"), 0).matrix == "bt2020"


def test_yuvclip_rejects_bad_new_layouts_and_colour():
    u16, u8 = torch.uint16, torch.uint8
    bad = [
        (torch.zeros(1, 2, 36, 32, dtype=u8), "p010", {}),                  # dtype per layout
        (torch.zeros(1, 2, 36, 32, dtype=torch.int16), "p016", {}),
        (torch.zeros(1, 2, 48, 32, dtype=u16), "yuv422p", {}),
        (torch.zeros(1, 2, 72, 32, dtype=u8), "yuv444p10", {}),
        (torch.zeros(2, 36, 32, dtype=u16), "p010", {}),                    # rank
        (torch.zeros(1, 2, 36, 32, 2, dtype=u16), "yuv420p10", {}),
        (torch.zeros(1, 2, 35, 32, dtype=u16), "p010", {}),                 # rows not H*3/2, 2H, 3H
        (torch.zeros(1, 2, 47, 32, dtype=u8), "yuv422p", {}),
        (torch.zeros(1, 2, 71, 32, dtype=u16), "yuv444p10", {}),
        (torch.zeros(1, 2, 36, 31, dtype=u16), "p010", {}),                 # odd W for 4:2:x
        (torch.zeros(1, 2, 48, 31, dtype=u8), "yuv422p", {}),
        (torch.zeros(1, 2, 48, 31, dtype=u16), "yuv422p10", {}),
        (torch.zeros(0, 2, 48, 32, dtype=u8), "yuv422p", {}),               # B, T >= 1
        (torch.zeros(1, 0, 72, 32, dtype=u8), "yuv444p", {}),
        (torch.zeros(1, 2, 36, 32, dtype=u16), "P010", {}),                 # layout names are FFmpeg's
        (torch.zeros(1, 2, 36, 32, dtype=u16), "p012", {}),
        (torch.zeros(1, 2, 36, 32, dtype=u8), "nv12", dict(matrix="bt2100")),
        (torch.zeros(1, 2, 36, 32, dtype=u8), "nv12", dict(matrix="BT709")),
        (torch.zeros(1, 2, 36, 32, dtype=u8), "nv12", dict(matrix=None)),
        (torch.zeros(1, 2, 36, 32, dtype=u8), "nv12", dict(full_range=1)),
        (torch.zeros(1, 2, 36, 32, dtype=u8), "nv12", dict(full_range="yes")),
        (torch.zeros(1, 2, 36, 32, dtype=u8), "nv12", dict(full_range=None)),
    ]
    for data, layout, kw in bad:
        with pytest.raises(ValueError):
            YUVClip(data, layout, **kw)
    YUVClip(torch.zeros(1, 2, 45, 32, dtype=u16), "p016")                 # H = 30
    YUVClip(torch.zeros(1, 2, 21, 31, dtype=u8), "yuv444p")                # 4:4:4: any H and W
    YUVClip(torch.zeros(1, 2, 14, 32, dtype=u16), "yuv422p10")             # 4:2:2: odd H is fine
    with pytest.raises(TypeError):
        YUVClip(torch.zeros(1, 2, 36, 32, dtype=u8), "nv12", "bt709")       # the colour is keyword-only


def test_chunk_plan_with_2_byte_samples():
    """A 16-bit frame's bytes are 2 * rows * W: 3 H W for 4:2:0 (uint8 RGB's), 4 H W for 4:2:2, 6 H W for 4:4:4."""
    slot = ingest.STAGING_SLOT_BYTES
    for layout, per_px in (("p010", 3), ("p016", 3), ("yuv420p10", 3), ("yuv422p10", 4), ("yuv444p10", 6),
                           ("yuv422p", 2), ("yuv444p", 3)):
        for H, W in ((1080, 1920), (2160, 3840), (2, 2)):
            rows = {3: H * 3 // 2, 4: 2 * H, 6: 3 * H}[engine._YUV_ROWS[layout]]
            c = YUVClip(torch.empty((1, 50, rows, W), dtype=engine.yuv_dtype(layout)), layout)
            fb = c.data[0, 0].numel() * c.data.element_size()
            assert fb == per_px * H * W
            plan = ingest.plan_chunks(50, fb)
            assert [t for a, b in plan for t in range(a, b)] == list(range(50))
            assert ingest.chunk_frames(50, fb) == min(50, max(1, slot // fb))
            assert ingest.staging_bytes(50, fb) <= 2 * max(slot, fb)
    assert ingest.chunk_frames(50, 2 * 1920 * 1620) == ingest.chunk_frames(50, 3 * 1920 * 1080) == 5
    assert ingest.chunk_frames(50, 6 * 3840 * 2160) == 1                  # a 4K 4:4:4 16-bit frame: a slot of its own


def test_prepare_frames_yuv_wrapper_new_arguments_without_gpu():
    p010 = torch.zeros(2, 36, 32, dtype=torch.uint16)
    for args, kw in (((p010, "p010"), {}), ((torch.zeros(2, 48, 32, dtype=torch.uint8), "yuv422p"), {}),
                     ((torch.zeros(2, 36, 32, dtype=torch.uint8), "nv12"), dict(matrix="bt709", full_range=True))):
        with pytest.raises(engine.EngineError, match="CUDA"):
            engine.prepare_frames_yuv(*args, (16, 16), **kw)
    bad = [
        ((p010.int(), "p010"), {}, "uint8 or uint16"),
        ((p010.to(torch.uint8), "p010"), {}, "torch.uint16"),
        ((p010, "nv12"), {}, "torch.uint8"),
        ((p010, "p012"), {}, "layout"),
        ((p010, "p010"), dict(matrix="bt2100"), "matrix"),
        ((p010, "p010"), dict(full_range=1), "full_range"),
        ((torch.zeros(2, 35, 32, dtype=torch.uint16), "p010"), {}, r"\[T,H\*3/2,W\]"),
        ((torch.zeros(2, 47, 32, dtype=torch.uint8), "yuv422p"), {}, r"\[T,2H,W\]"),
        ((torch.zeros(2, 47, 32, dtype=torch.uint16), "yuv444p10"), {}, r"\[T,3H,W\]"),
        ((torch.zeros(2, 36, 64, dtype=torch.uint16)[:, :, ::2], "p010"), {}, "contiguous"),
    ]
    for args, kw, msg in bad:
        with pytest.raises(engine.EngineError, match=msg):
            engine.prepare_frames_yuv(*args, (16, 16), **kw)
    with pytest.raises(TypeError):
        engine.prepare_frames_yuv(p010, "p010", (16, 16), None, "bt709")


def test_prepare_frames_yuv_fmt_exported_and_declared():
    lib = engine.lib()
    assert hasattr(lib, "ct3_prepare_frames_yuv_fmt") and "ct3_prepare_frames_yuv_fmt" in engine.EXPORTED_SYMBOLS
    with open(os.path.join(ROOT, "include", "ct3_b200.h")) as f:
        header = f.read()
    assert re.search(r"int ct3_prepare_frames_yuv_fmt\(", header)
    for name, code in engine.YUV_FORMATS.items():
        assert re.search(rf"CT3_YUV_{name.upper()} = {code}\b", header), name
    for name, code in engine.YUV_MATRICES.items():
        assert f"CT3_MATRIX_{name.upper()} = {code}" in header
    assert set(engine.YUV_FORMATS) == set(C.FORMATS) and engine.YUV_LAYOUTS == {"nv12": 0, "i420": 1, "yuyv": 2}
    assert all(engine.yuv_dtype(k) == v[0] for k, v in C.FORMATS.items())
    assert lib.ct3_version() == 102


def test_prepare_frames_yuv_fmt_rejects_bad_arguments_without_gpu():
    """Each invalid argument returns CT3_EINVAL with a message before any launch (fake pointers, legacy stream:
    reaching a launch would fail differently)."""
    lib = engine.lib()
    src, out = ctypes.c_void_p(1 << 20), ctypes.c_void_p(1 << 24)
    H, W = 90, 120
    ok = dict(src=src, layout=5, matrix=1, full=0, T=4, H=H, W=W, st=H * W * 3, sr=2 * W, oh=384, ow=512, out=out)

    def call(**kw):
        a = dict(ok, **kw)
        return lib.ct3_prepare_frames_yuv_fmt(a["src"], a["layout"], a["matrix"], a["full"], a["T"], a["H"], a["W"],
                                              a["st"], a["sr"], a["oh"], a["ow"], a["out"], None)

    cases = [
        (dict(src=None), b"null argument"), (dict(out=None), b"null argument"),
        (dict(layout=10), b"unknown YUV layout"), (dict(layout=-1), b"unknown YUV layout"),
        (dict(matrix=3), b"unknown colour matrix"), (dict(matrix=-1), b"unknown colour matrix"),
        (dict(full=2), b"full_range must be 0 or 1"), (dict(full=-1), b"full_range must be 0 or 1"),
        (dict(T=0), b"must be >= 1"), (dict(H=0), b"must be >= 1"), (dict(W=-2), b"must be >= 1"),
        (dict(oh=0), b"must be >= 1"), (dict(ow=0), b"must be >= 1"),
        (dict(H=91), b"P010 frames must have an even width and height"),
        (dict(W=121, sr=242), b"P010 frames must have an even width and height"),
        (dict(layout=7, H=91, sr=2 * W), b"YUV420P10 frames must have an even width and height"),
        (dict(layout=3, W=121, sr=121), b"YUV422P frames must have an even width"),
        (dict(layout=8, W=121, sr=242), b"YUV422P10 frames must have an even width"),
        (dict(st=H * W * 3 + 1), b"strides must be even"), (dict(sr=2 * W + 1), b"strides must be even"),
        (dict(layout=9, sr=2 * W, st=-1), b"strides must be even"),
        (dict(sr=2 * W - 2), b"row stride is below"), (dict(sr=-2 * W), b"row stride is below"),
        (dict(layout=6, sr=W), b"row stride is below"),
        (dict(layout=4, sr=W - 1), b"row stride is below"),
        (dict(layout=3, sr=W + 64), b"YUV422P rows must be dense"),
        (dict(layout=9, sr=2 * W + 64), b"YUV444P10 rows must be dense"),
        (dict(st=2 ** 62), b"stride extent"),
        (dict(st=-(2 ** 63)), b"stride extent"),
        (dict(sr=2 ** 60), b"stride extent"),
        (dict(layout=4, sr=W, st=W * H * 3, H=H, W=W, T=2 ** 31 - 1, oh=1, ow=2 ** 31 - 1), b"output too large"),
        (dict(oh=65536, ow=32768), b"output plane too large"),
    ]
    for kw, msg in cases:
        assert call(**kw) == -1, kw
        assert msg in lib.ct3_last_error(), (kw, lib.ct3_last_error())
    # ct3_prepare_frames_yuv still takes only its three layouts, whatever the new entry point accepts
    assert lib.ct3_prepare_frames_yuv(src, 3, 4, H, W, H * W * 2, W, 384, 512, out, None) == -1
    assert b"unknown YUV layout" in lib.ct3_last_error()
