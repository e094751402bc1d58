"""GPU tests of YUV input: ct3_prepare_frames_yuv is torch.equal to ct3_prepare_frames on the RGB that cv2 makes of the
frames (restated in tests/yuv_cases.py, checked against cv2 in test_yuv_host.py), for every layout, size class and
stride form; a host YUVClip equals the device one; and every predictor entry point gives on a YUVClip exactly what it
gives on that RGB clip."""
import pytest
import torch

from yuv_cases import LAYOUTS, yuv_to_rgb, yuv_video

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# (H, W) -> (oh, ow): the same-size copy, a 1080p downscale, an upscale, odd chroma height, the smallest frame
SIZES = [((48, 64), (48, 64)), ((1080, 1920), (384, 512)), ((240, 320), (384, 512)), ((30, 46), (384, 512)),
         ((30, 46), (30, 46)), ((2, 2), (384, 512))]


def _random_frames(layout, T, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    shape = (T, H, W, 2) if layout == "yuyv" else (T, H * 3 // 2, W)
    return torch.randint(0, 256, shape, generator=g, dtype=torch.uint8)


def _rgb(layout, frames):
    return yuv_to_rgb(layout, frames.cpu()).to(frames.device)


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("size", SIZES, ids=lambda s: f"{s[0][0]}x{s[0][1]}-{s[1][0]}x{s[1][1]}")
def test_kernel_equals_rgb_path(layout, size):
    from cotracker_b200 import engine
    (H, W), out_hw = size
    src = _random_frames(layout, 3, H, W, seed=H + W).to(DEV)
    got = engine.prepare_frames_yuv(src, layout, out_hw)
    want = engine.prepare_frames(_rgb(layout, src), out_hw)
    assert torch.equal(got, want)


@pytest.mark.parametrize("layout", LAYOUTS)
def test_kernel_strided_sources(layout):
    """Pitched rows (NV12, YUYV), a gapped frame stride and a storage offset all read the same frames."""
    from cotracker_b200 import engine
    H, W = 30, 46
    dense = _random_frames(layout, 4, H, W, seed=5).to(DEV)
    want = engine.prepare_frames(_rgb(layout, dense), (64, 80))
    rows = dense.shape[2]
    pads = [0] if layout == "i420" else [0, 64 if layout == "nv12" else 128]      # I420 rows must be dense
    views = []
    for pad in pads:
        for gap in (1, 3):
            big = torch.zeros((1 + 4 * gap,) + tuple(dense.shape[1:2]) + (rows + pad,) + tuple(dense.shape[3:]),
                              dtype=torch.uint8, device=DEV)
            v = big[1::gap][:4, :, :rows]
            v.copy_(dense)
            views.append(v)
    assert len(views) == 2 * len(pads) and any(v.stride(0) > v[0].numel() for v in views)
    for v in views:
        assert torch.equal(v.cpu(), dense.cpu())
        assert torch.equal(engine.prepare_frames_yuv(v, layout, (64, 80)), want), v.stride()


@pytest.mark.parametrize("layout", LAYOUTS)
def test_host_clip_equals_device_clip_in_small_slots(layout, monkeypatch):
    """A host YUVClip goes through the two staging slots: many chunks, then slots smaller than a frame."""
    from cotracker_b200 import YUVClip, ingest
    data = yuv_video(layout, 2, 7, 60, 80, seed=3)
    want = ingest.prepare_video(YUVClip(data.to(DEV), layout), (96, 128), DEV)
    fb = data[0, 0].numel()
    for slot in (2 * fb + fb // 2, fb // 3):
        monkeypatch.setattr(ingest, "STAGING_SLOT_BYTES", slot)
        assert torch.equal(ingest.prepare_video(YUVClip(data, layout), (96, 128), DEV), want)
        gapped = torch.zeros((2, 14) + tuple(data.shape[2:]), dtype=torch.uint8)
        gapped[:, ::2] = data
        assert torch.equal(ingest.prepare_video(YUVClip(gapped[:, ::2], layout), (96, 128), DEV), want)
    rgb = yuv_to_rgb(layout, data)
    assert torch.equal(want, ingest.prepare_video(rgb, (96, 128), DEV))


# ---- predictors ---------------------------------------------------------------------------------------------------
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


@pytest.mark.parametrize("layout", LAYOUTS)
def test_predictor_yuv_equals_rgb(layout):
    from cotracker_b200 import YUVClip
    from cotracker_b200.synthetic import random_queries
    p = _offline()
    data = yuv_video(layout, 2, 12, 96, 128, seed=11)
    rgb = yuv_to_rgb(layout, data)
    one, one_rgb = YUVClip(data[:1], layout), rgb[:1]
    assert _equal(p(one, grid_size=6), p(one_rgb, grid_size=6))                                    # host
    q = random_queries(20, 12, 96, 128, seed=4).to(DEV)
    dev, dev_rgb = YUVClip(data[:1].to(DEV), layout), rgb[:1].to(DEV)
    assert _equal(p(dev, queries=q, backward_tracking=True), p(dev_rgb, queries=q, backward_tracking=True))
    assert _equal(p(YUVClip(data, layout), grid_size=5), p(rgb, grid_size=5))                      # a batch of 2
    other = yuv_video("nv12", 1, 7, 64, 80, seed=12)
    clips = [YUVClip(data[:1].to(DEV), layout), yuv_to_rgb("nv12", other)]                        # YUV next to RGB
    got = p(clips, grid_size=4, backward_tracking=True)
    want = p([rgb[:1].to(DEV), yuv_to_rgb("nv12", other)], grid_size=4, backward_tracking=True)
    assert _equal(got, want)


def test_predictor_yuv_dense_and_segm_mask():
    from cotracker_b200 import YUVClip
    p = _offline()
    data = yuv_video("i420", 1, 6, 64, 80, seed=13)
    rgb = yuv_to_rgb("i420", data)
    clip = YUVClip(data, "i420")
    mask = torch.zeros(1, 1, 64, 80)
    mask[..., 10:50, 20:70] = 1
    assert _equal(p(clip, grid_size=8, segm_mask=mask), p(rgb, grid_size=8, segm_mask=mask))
    assert _equal(p(clip, grid_query_frame=2), p(rgb, grid_query_frame=2))                        # dense mode


def test_online_predictor_yuv_chunks():
    from cotracker_b200 import YUVClip
    S = 16
    data = yuv_video("nv12", 1, 32, 96, 128, seed=17)
    rgb = yuv_to_rgb("nv12", data)
    outs = []
    for src in ("yuv", "rgb"):
        p = _online(S=S)
        chunk = (lambda a, b: YUVClip(data[:, a:b].to(DEV), "nv12")) if src == "yuv" else (lambda a, b: rgb[:, a:b])
        p(video_chunk=chunk(0, S), is_first_step=True, grid_size=5)
        res = [p(video_chunk=chunk(a, a + S)) for a in (0, S // 2, S)]     # 3 chunks
        outs.append(res)
    assert _equal(outs[0], outs[1])


def test_online_streams_yuv_and_rgb_stream():
    from cotracker_b200 import OnlineStreams, YUVClip
    S = 16
    yuv = yuv_video("yuyv", 1, 24, 80, 96, seed=19)
    yuv_rgb = yuv_to_rgb("yuyv", yuv)
    from cotracker_b200.synthetic import texture_video
    other = texture_video(24, 64, 80, seed=20).to(torch.uint8)
    res = []
    for as_yuv in (True, False):
        hub = OnlineStreams(_online(S=S))
        a = hub.open(frame_size=(80, 96), grid_size=4)
        b = hub.open(frame_size=(64, 80), grid_size=3)
        with pytest.raises(ValueError):
            hub.push(a, YUVClip(torch.zeros(1, 4, 64, 80, 2, dtype=torch.uint8), "yuyv"))    # another frame size
        steps = []
        for t0 in (0, S // 2):
            hub.push(a, YUVClip(yuv[:, t0:t0 + S], "yuyv") if as_yuv else yuv_rgb[:, t0:t0 + S])
            hub.push(b, other[:, t0:t0 + S].to(DEV))
            steps.append(hub.step())
        res.append(steps)
    for sa, sb in zip(*res):
        assert sa.keys() == sb.keys() and all(_equal(sa[k], sb[k]) for k in sa)


def test_evaluation_predictor_single_point_yuv():
    from cotracker_b200 import YUVClip
    from cotracker_b200.evaluation import EvaluationPredictor
    from cotracker_b200.synthetic import random_queries
    p = _offline()
    ev = EvaluationPredictor(p.model, single_point=True, grid_size=5, local_grid_size=8)
    data = yuv_video("i420", 1, 10, 96, 128, seed=23)
    q = random_queries(3, 10, 96, 128, seed=6)
    torch.manual_seed(0)
    got = ev(YUVClip(data, "i420"), q)
    torch.manual_seed(0)
    want = ev(yuv_to_rgb("i420", data), q)
    assert _equal(got, want)
