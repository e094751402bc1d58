"""CPU tests of `Crop`: validation of the window and its offsets, the coordinate helpers against hand-written loops,
time slices, the host staging plan of windows (chunks from the window's bytes; the chroma-aligned rectangle and
residual offsets of YUV windows), the entry points that refuse a Crop, and the argument checks of
ct3_prepare_frames_crop / ct3_prepare_frames_yuv_crop before any launch."""
import ctypes
import os
import re

import pytest
import torch

import yuv_color_cases as C
from cotracker_b200 import Crop, YUVClip, engine, ingest

B, T, H, W = 2, 5, 40, 60


def _video():
    return torch.zeros(B, T, 3, H, W, dtype=torch.uint8)


def test_shapes_broadcast_and_edges():
    v = _video()
    c = Crop(v, (10, 20), (3, 5))
    assert c.shape == (B, T, 3, 10, 20) and c.dim() == 5 and not c.is_cuda and c.device == v.device
    assert c.offsets.shape == (B, T, 2) and c.offsets.dtype == torch.int64
    assert bool((c.offsets == torch.tensor([3, 5])).all())
    per_frame = torch.arange(T * 2, dtype=torch.int32).view(T, 2)
    c = Crop(v, (10, 20), per_frame)
    assert torch.equal(c.offsets, per_frame.long().expand(B, T, 2))
    per_clip = torch.randint(0, 20, (B, T, 2), dtype=torch.int16)
    assert torch.equal(Crop(v, (10, 20), per_clip).offsets, per_clip.long())
    for off in [(0, 0), (H - 10, 0), (0, W - 20), (H - 10, W - 20)]:    # windows touching each edge
        Crop(v, (10, 20), off)
    Crop(v, (H, W), (0, 0))
    Crop(v, (1, 1), (H - 1, W - 1))
    y = YUVClip(torch.zeros(1, T, H * 3 // 2, W, dtype=torch.uint8), "nv12")
    assert Crop(y, (7, 9), (3, 5)).shape == (1, T, 3, 7, 9)


@pytest.mark.parametrize("size, off", [
    ((10, 20), (-1, 0)), ((10, 20), (0, -1)), ((10, 20), (H - 9, 0)), ((10, 20), (0, W - 19)),
    ((0, 20), (0, 0)), ((10, 0), (0, 0)), ((H + 1, 20), (0, 0)), ((10, W + 1), (0, 0))])
def test_out_of_frame_windows_are_rejected(size, off):
    with pytest.raises(ValueError):
        Crop(_video(), size, off)


def test_bad_arguments_are_rejected():
    v = _video()
    bad_t = torch.zeros(T, 2, dtype=torch.int64)
    bad_t[3, 1] = W - 19                                       # one frame of a per-frame tensor outside
    for size, off in [((10, 20), bad_t), ((10.0, 20), (0, 0)), ((10, 20), (0.0, 0)), ((True, 20), (0, 0)),
                      ((10, 20), torch.zeros(T, 2)), ((10, 20), torch.zeros(T + 1, 2, dtype=torch.int64)),
                      ((10, 20), torch.zeros(B, T, 3, dtype=torch.int64)), ((10, 20), (0, 0, 0)),
                      ((10, 20), torch.zeros(T, 2, dtype=torch.bool)), ((10, 20), "0,0")]:
        with pytest.raises(ValueError):
            Crop(v, size, off)
    with pytest.raises(ValueError):
        Crop(torch.zeros(1, 2, 4, 8, 8), (2, 2), (0, 0))
    with pytest.raises(TypeError):
        Crop(Crop(v, (10, 20), (0, 0)), (5, 5), (0, 0))


def test_a_crop_of_an_encoded_clip_is_rejected():
    from cotracker_b200 import EncodedClip
    clip = EncodedClip.__new__(EncodedClip)
    with pytest.raises(TypeError):
        Crop(clip, (5, 5), (0, 0))


def test_time_slices_slice_the_offsets():
    v = torch.arange(B * T, dtype=torch.uint8).view(B, T, 1, 1, 1).expand(B, T, 3, H, W)
    off = torch.stack([torch.arange(T), 2 * torch.arange(T)], -1)
    c = Crop(v, (10, 20), off)
    s = c[:, 1:4]
    assert s.shape == (B, 3, 3, 10, 20) and torch.equal(s.offsets, c.offsets[:, 1:4])
    assert torch.equal(s.video, v[:, 1:4])
    one = c[1:2]
    assert one.shape[0] == 1 and torch.equal(one.offsets, c.offsets[1:2])
    from cotracker_b200.corners import clip_frame
    f = clip_frame(c, 2)
    assert isinstance(f, Crop) and torch.equal(f.offsets, c.offsets[:, 2:3])
    y = YUVClip(torch.arange(T, dtype=torch.uint8).view(1, T, 1, 1).expand(1, T, H * 3 // 2, W), "nv12")
    ys = Crop(y, (4, 6), off)[:, 3:5]
    assert isinstance(ys.video, YUVClip) and torch.equal(ys.video.data, y.data[:, 3:5])
    assert torch.equal(ys.offsets, off[3:5].expand(1, 2, 2))
    with pytest.raises(TypeError):
        c[:, 2]
    with pytest.raises(TypeError):
        c[:, :, 0]


def test_to_frame_and_from_frame_against_loops():
    g = torch.Generator().manual_seed(1)
    off = torch.stack([torch.randint(0, H - 10 + 1, (B, T), generator=g),
                       torch.randint(0, W - 20 + 1, (B, T), generator=g)], -1)
    c = Crop(_video(), (10, 20), off)
    N = 7
    tracks = torch.rand(B, T, N, 2, generator=g) * 20
    want = tracks.clone()
    for b in range(B):
        for t in range(T):
            for n in range(N):
                want[b, t, n, 0] = tracks[b, t, n, 0] + float(off[b, t, 1])
                want[b, t, n, 1] = tracks[b, t, n, 1] + float(off[b, t, 0])
    assert torch.equal(c.to_frame(tracks), want)
    assert torch.equal(c.to_frame(tracks[:, 2:], frames=slice(2, T)), want[:, 2:])
    with pytest.raises(ValueError):
        c.to_frame(tracks[:, 2:])
    q = torch.cat([torch.randint(0, T, (B, N, 1), generator=g).float() + 0.5,     # frames differ per query
                   torch.rand(B, N, 2, generator=g) * 60], -1)
    want = q.clone()
    for b in range(B):
        for n in range(N):
            t = int(q[b, n, 0])
            want[b, n, 1] = q[b, n, 1] - float(off[b, t, 1])
            want[b, n, 2] = q[b, n, 2] - float(off[b, t, 0])
    assert torch.equal(c.from_frame(q), want)
    q[0, 3, 0] = T
    with pytest.raises(ValueError):
        c.from_frame(q)


def test_host_rgb_chunks_are_planned_from_the_window_bytes():
    """A 1024 x 768 window of a 3840 x 2160 uint8 frame stages 3 * 768 * 1024 bytes a frame, not 3 * 2160 * 3840."""
    frame, window = 3 * 2160 * 3840, 3 * 768 * 1024
    assert ingest.chunk_frames(48, frame) == 1 and ingest.chunk_frames(48, window) == 14
    assert ingest.staging_bytes(48, window) == 2 * 14 * window <= 2 * ingest.STAGING_SLOT_BYTES
    assert ingest._staged_strides((3, 768, 1024), (1, 3 * 3840, 3)) == (1, 3 * 1024, 3)     # channels-last kept
    assert ingest._staged_strides((3, 768, 1024), (2160 * 3840, 3840, 1)) == (768 * 1024, 1024, 1)


@pytest.mark.parametrize("layout", list(C.FORMATS))
def test_yuv_window_rectangles(layout):
    xs, ys = engine.yuv_subsampling(layout)
    h, w = 7, 10
    offsets = torch.tensor([[0, 0], [1, 1], [2, 3], [3, 2], [5, 7]])
    origin, extent, residual = ingest.yuv_window(layout, offsets, (h, w))
    for (top, left), (o0, o1), (e0, e1), (r0, r1) in zip(offsets.tolist(), origin.tolist(), extent.tolist(),
                                                          residual.tolist()):
        assert (o0, o1) == (top - (top % 2 if ys else 0), left - (left % 2 if xs else 0))
        assert (r0, r1) == (top - o0, left - o1) and r0 in (0, 1) and r1 in (0, 1)
        end_r, end_c = top + h, left + w
        assert o0 + e0 == end_r + (end_r % 2 if ys else 0) and o1 + e1 == end_c + (end_c % 2 if xs else 0)
        assert (not ys or (o0 % 2 == 0 and e0 % 2 == 0)) and (not xs or (o1 % 2 == 0 and e1 % 2 == 0))
    # the staged frame: h x w plus at most one row / column on each side of a subsampled axis, even there
    hs, ws = (int(x) for x in extent.amax(0))
    assert h <= hs <= h + 2 * ys and w <= ws <= w + 2 * xs
    assert (hs, ws) == ((h + 1 if h % 2 else h + 2) if ys else h, (w + 1 if w % 2 else w + 2) if xs else w)


def test_visualizer_rejects_a_crop():
    from cotracker_b200.visualizer import Visualizer
    c = Crop(torch.zeros(1, 2, 3, 16, 16), (8, 8), (0, 0))
    with pytest.raises(TypeError):
        Visualizer(save_dir="/nonexistent").visualize(c, torch.zeros(1, 2, 1, 2), save_video=False)
    with pytest.raises(TypeError):
        Visualizer(save_dir="/nonexistent").draw_tracks_on_video(c, torch.zeros(1, 2, 1, 2))


def test_entry_points_accept_a_crop_in_their_checks():
    from cotracker_b200.predictor import _check_list_call

    class _Offline:
        pass
    crops = [Crop(torch.zeros(1, 4, 3, 32, 48), s, (0, 0)) for s in ((16, 16), (20, 30))]
    _check_list_call(_Offline(), crops, None, None, 4, 0)


def _lib():
    if not os.path.exists(engine.LIB_PATH):
        pytest.skip("libct3_b200.so is not built")
    return engine.lib()


def test_crop_entry_points_exported_and_declared():
    lib = _lib()
    header = open(os.path.join(os.path.dirname(engine.__file__), "..", "include", "ct3_b200.h")).read()
    for name in ("ct3_prepare_frames_crop", "ct3_prepare_frames_yuv_crop"):
        assert hasattr(lib, name) and name in engine.EXPORTED_SYMBOLS
        assert re.search(rf"int {name}\(", header)


def test_crop_entry_points_reject_bad_arguments_without_gpu():
    lib = _lib()
    p = ctypes.c_void_p(16)                      # never dereferenced: every call fails its checks first
    Hh, Ww = 32, 48

    def rgb(**kw):
        a = dict(src=p, dtype=0, T=2, H=Hh, W=Ww, st=3 * Hh * Ww, sc=Hh * Ww, sh=Ww, sw=1, off=p, ch=8, cw=8, oh=16,
                 ow=16, out=p)
        a.update(kw)
        return lib.ct3_prepare_frames_crop(a["src"], a["dtype"], a["T"], a["H"], a["W"], a["st"], a["sc"], a["sh"],
                                           a["sw"], a["off"], a["ch"], a["cw"], a["oh"], a["ow"], a["out"], None)

    def yuv(**kw):
        a = dict(src=p, layout=0, m=0, f=0, T=2, H=Hh, W=Ww, st=Hh * Ww * 3 // 2, sr=Ww, off=p, ch=8, cw=8, oh=16,
                 ow=16, out=p)
        a.update(kw)
        return lib.ct3_prepare_frames_yuv_crop(a["src"], a["layout"], a["m"], a["f"], a["T"], a["H"], a["W"], a["st"],
                                               a["sr"], a["off"], a["ch"], a["cw"], a["oh"], a["ow"], a["out"], None)

    for call in (rgb, yuv):
        for kw in (dict(off=None), dict(ch=0), dict(cw=0), dict(ch=Hh + 1), dict(cw=Ww + 1), dict(src=None),
                   dict(out=None), dict(T=0), dict(oh=0)):
            assert call(**kw) == -1, (call.__name__, kw)
    assert rgb(dtype=7) == -1 and yuv(layout=99) == -1 and yuv(m=5) == -1 and yuv(f=2) == -1
    assert yuv(H=Hh + 1) == -1 and yuv(sr=Ww - 1) == -1
