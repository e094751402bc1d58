"""GPU tests of the YUV layouts beyond NV12 / I420 / YUYV and of YUV colour: ct3_prepare_frames_yuv_fmt is torch.equal
to ct3_prepare_frames on the uint8 RGB that the integer formula gives (restated in tests/yuv_color_cases.py, checked
against float64 and cv2 in test_yuv_color_host.py) for every layout, matrix and range, size class and stride form; host
and device clips take the same path; and the predictors, online streams and the corner detector give on such a clip
exactly what they give on that RGB clip."""
import ctypes

import pytest
import torch

import yuv_color_cases as C

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# (H, W) -> (oh, ow): a downscale, an upscale with odd chroma counts (15 x 23 at 4:2:0), the same-size copy, tiny
SIZES = [((96, 128), (64, 80)), ((30, 46), (64, 80)), ((48, 64), (48, 64)), ((2, 2), (7, 9))]
COLOUR_IDS = [f"{m}-{'full' if f else 'limited'}" for m, f in C.COLOURS]


def _rgb(layout, frames, matrix="bt601", full_range=False):
    return C.yuv_to_rgb(layout, frames.cpu(), matrix, full_range).to(frames.device)


@pytest.mark.parametrize("colour", C.COLOURS, ids=COLOUR_IDS)
@pytest.mark.parametrize("layout", C.NEW_LAYOUTS)
def test_kernel_equals_rgb_path(layout, colour):
    from cotracker_b200 import engine
    m, f = colour
    for (H, W), out_hw in SIZES:
        src = C.random_frames(layout, (3,), H, W, seed=H + W).to(DEV)
        got = engine.prepare_frames_yuv(src, layout, out_hw, matrix=m, full_range=f)
        assert torch.equal(got, engine.prepare_frames(_rgb(layout, src, m, f), out_hw)), (H, W)


@pytest.mark.parametrize("layout", ("nv12", "i420", "yuyv"))
def test_old_layouts_in_every_colour(layout):
    from cotracker_b200 import engine
    src = C.random_frames(layout, (3,), 30, 46, seed=7).to(DEV)
    for m, f in C.COLOURS:
        got = engine.prepare_frames_yuv(src, layout, (64, 80), matrix=m, full_range=f)
        assert torch.equal(got, engine.prepare_frames(_rgb(layout, src, m, f), (64, 80))), (m, f)


def test_1080p_downscale():
    from cotracker_b200 import engine
    for layout in ("p010", "yuv420p10", "yuv444p"):
        src = C.random_frames(layout, (2,), 1080, 1920, seed=9).to(DEV)
        got = engine.prepare_frames_yuv(src, layout, (384, 512), matrix="bt709")
        assert torch.equal(got, engine.prepare_frames(_rgb(layout, src, "bt709"), (384, 512))), layout


def test_pitched_rows_gapped_frames_and_a_negative_frame_stride():
    """P010 / P016 rows at a pitch, frames at a gapped stride and a storage offset, and (through the C ABI, which
    takes any frame stride) frames read last to first."""
    from cotracker_b200 import engine
    H, W = 30, 46
    for layout in ("p010", "p016", "nv12"):
        dense = C.random_frames(layout, (4,), H, W, seed=11).to(DEV)
        want = engine.prepare_frames(_rgb(layout, dense, "bt2020", True), (64, 80))
        rows = dense.shape[1]
        for pad, gap in ((0, 3), (32, 1), (32, 2)):
            big = torch.zeros((1 + 4 * gap, rows, W + pad), dtype=dense.dtype, device=DEV)
            v = big[1::gap][:4, :, :W]
            v.copy_(dense)
            assert torch.equal(engine.prepare_frames_yuv(v, layout, (64, 80), matrix="bt2020", full_range=True), want)
        lib, es = engine.lib(), dense.element_size()
        out = torch.empty(4, 3, 64, 80, device=DEV)
        last = ctypes.c_void_p(dense[3].data_ptr())
        fmt = engine.YUV_FORMATS[layout]
        rc = lib.ct3_prepare_frames_yuv_fmt(last, fmt, 2, 1, 4, H, W, -dense.stride(0) * es, W * es, 64, 80,
                                            ctypes.c_void_p(out.data_ptr()),
                                            ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc == 0, lib.ct3_last_error()
        assert torch.equal(out, want.flip(0))


def test_default_colour_is_the_old_entry_point():
    """The three original layouts in the default colour give the same floats through either entry point."""
    from cotracker_b200 import engine
    for layout in ("nv12", "i420", "yuyv"):
        src = C.random_frames(layout, (3,), 60, 80, seed=13).to(DEV)
        old = engine.prepare_frames_yuv(src, layout, (96, 128))
        out = torch.empty_like(old)
        H, W = C.frame_hw(layout, src.shape)
        rc = engine.lib().ct3_prepare_frames_yuv_fmt(ctypes.c_void_p(src.data_ptr()), engine.YUV_FORMATS[layout], 0, 0,
                                                     3, H, W, src.stride(0), src.stride(1), 96, 128,
                                                     ctypes.c_void_p(out.data_ptr()),
                                                     ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc == 0, engine.lib().ct3_last_error()
        assert torch.equal(out, old)


@pytest.mark.parametrize("layout", ("p010", "yuv422p10", "yuv444p"))
def test_host_clip_equals_device_clip_in_small_slots(layout, monkeypatch):
    """A host YUVClip of 2-byte (or 1-byte) samples goes through the two staging slots: many chunks, then slots
    smaller than a frame; B = 2."""
    from cotracker_b200 import YUVClip, ingest
    data = C.random_frames(layout, (2, 7), 60, 80, seed=17)
    kw = dict(matrix="bt709", full_range=layout != "p010")
    want = ingest.prepare_video(YUVClip(data.to(DEV), layout, **kw), (96, 128), DEV)
    fb = data[0, 0].numel() * data.element_size()
    for slot in (2 * fb + fb // 2, fb // 3):
        monkeypatch.setattr(ingest, "STAGING_SLOT_BYTES", slot)
        assert torch.equal(ingest.prepare_video(YUVClip(data, layout, **kw), (96, 128), DEV), want)
        gapped = torch.zeros((2, 14) + tuple(data.shape[2:]), dtype=data.dtype)
        gapped[:, ::2] = data
        assert torch.equal(ingest.prepare_video(YUVClip(gapped[:, ::2], layout, **kw), (96, 128), DEV), want)
    rgb = C.yuv_to_rgb(layout, data, **kw)
    assert torch.equal(want, ingest.prepare_video(rgb, (96, 128), DEV))


# ---- predictors, streams, corners ---------------------------------------------------------------------------------
def _video(layout, B, T, H, W, seed):
    """A moving texture as frames of `layout` [B,T,...] on the host."""
    from cotracker_b200.synthetic import texture_video
    clips = [texture_video(T, H, W, seed=seed + b, shift=(1 + (seed + b) % 3, 2))[0].to(torch.uint8) for b in range(B)]
    return C.as_frames(layout, torch.stack(clips))


def _offline(seed=43):
    from cotracker_b200.predictor import CoTrackerPredictor
    from cotracker_b200.synthetic import seeded_state_dict
    p = CoTrackerPredictor(checkpoint=None, window_len=60)
    p.model.load_state_dict(seeded_state_dict(seed, offline=True, window_len=60, head_gain=10.0, vis_gain=100.0))
    return p.to(DEV)


def _online(seed=47, S=16):
    from cotracker_b200.predictor import CoTrackerOnlinePredictor
    from cotracker_b200.synthetic import seeded_state_dict
    p = CoTrackerOnlinePredictor(checkpoint=None, window_len=S)
    p.model.load_state_dict(seeded_state_dict(seed, offline=False, window_len=S, head_gain=10.0, vis_gain=100.0))
    return p.to(DEV)


def _equal(a, b):
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_equal(x, y) for x, y in zip(a, b))
    return torch.equal(a, b)


def test_predictor_p010_bt709_and_a_mixed_list():
    from cotracker_b200 import YUVClip
    from cotracker_b200.synthetic import random_queries
    p = _offline()
    data = _video("p010", 2, 12, 96, 128, seed=11)
    rgb = C.yuv_to_rgb("p010", data, "bt709")
    assert _equal(p(YUVClip(data[:1], "p010", matrix="bt709"), grid_size=6), p(rgb[:1], grid_size=6))    # host
    q = random_queries(20, 12, 96, 128, seed=4).to(DEV).expand(2, -1, -1)
    dev = YUVClip(data.to(DEV), "p010", matrix="bt709")                                                 # B = 2
    assert _equal(p(dev, queries=q), p(rgb.to(DEV), queries=q))
    a = _video("yuv422p", 1, 7, 64, 80, seed=12)
    b = _video("yuv444p10", 1, 9, 48, 64, seed=13)
    clips = [YUVClip(data[:1].to(DEV), "p010", matrix="bt709"), YUVClip(a, "yuv422p", full_range=True),
             YUVClip(b.to(DEV), "yuv444p10", matrix="bt2020"), C.yuv_to_rgb("nv12", _video("nv12", 1, 5, 48, 64, 14))]
    rgbs = [rgb[:1].to(DEV), C.yuv_to_rgb("yuv422p", a, full_range=True), C.yuv_to_rgb("yuv444p10", b, "bt2020"),
            clips[3]]
    assert _equal(p(clips, grid_size=4, backward_tracking=True), p(rgbs, grid_size=4, backward_tracking=True))


def test_online_streams_yuv422p_full_range_with_a_preview():
    from cotracker_b200 import OnlineStreams, YUVClip
    S = 16
    data = _video("yuv422p", 1, 32, 80, 96, seed=19)
    rgb = C.yuv_to_rgb("yuv422p", data, full_range=True)
    res = []
    for as_yuv in (True, False):
        hub = OnlineStreams(_online(S=S))
        sid = hub.open(frame_size=(80, 96), grid_size=4)
        chunk = (lambda a, b: YUVClip(data[:, a:b], "yuv422p", full_range=True)) if as_yuv else \
            (lambda a, b: rgb[:, a:b].to(DEV))
        steps = []
        for kind, a, b in (("c", 0, S), ("p", S // 2, S + 4), ("c", S // 2, S + S // 2), ("c", S, 2 * S)):
            hub.push(sid, chunk(a, b), preview=kind == "p")
            steps.append(hub.step()[sid])
        res.append(steps)
    assert _equal(res[0], res[1])


def test_detect_corners_yuv420p10_bt2020():
    from cotracker_b200 import YUVClip
    from cotracker_b200.corners import detect_corners
    data = _video("yuv420p10", 2, 4, 96, 128, seed=23)
    rgb = C.yuv_to_rgb("yuv420p10", data, "bt2020")
    for dev in ("cpu", DEV):
        got = detect_corners(YUVClip(data.to(dev), "yuv420p10", matrix="bt2020"), 30, frame=2, min_distance=6)
        want = detect_corners(rgb.to(dev), 30, frame=2, min_distance=6)
        assert _equal(got, want) and sum(g.shape[1] for g in got) > 10
