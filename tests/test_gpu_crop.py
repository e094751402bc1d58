"""GPU tests of `Crop`: ingestion of a window of each frame is torch.equal to ingestion of the materialised window, for
RGB clips of both dtypes on the host and the device in every stride form, every YUV layout at odd and even offsets in
three colours, and windows of one pixel, touching the last row and column, and of the whole frame; and every entry
point gives on a Crop exactly what it gives on the materialised clip (tracks, visibility and scores), with no new
goldens."""
import ctypes

import pytest
import torch

import yuv_color_cases as C
from cotracker_b200 import Crop, OnlineStreams, YUVClip, detect_corners, engine, ingest
from cotracker_b200.evaluation import EvaluationPredictor
from cotracker_b200.predictor import CoTrackerOnlinePredictor, CoTrackerPredictor
from cotracker_b200.synthetic import random_queries, seeded_state_dict, texture_video

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _materialise(video, offset, size):
    """The clip a Crop stands for, built by hand: frame (b, t) = video[b, t, :, top:top+h, left:left+w]."""
    B, T = video.shape[:2]
    h, w = size
    off = torch.as_tensor(offset).expand(B, T, 2)
    return torch.stack([torch.stack([video[b, t, :, int(off[b, t, 0]):int(off[b, t, 0]) + h,
                                           int(off[b, t, 1]):int(off[b, t, 1]) + w] for t in range(T)])
                        for b in range(B)]).contiguous()


def _forms(x):
    """The same clip [B,T,3,H,W] contiguous, channels-last (a permuted [B,T,H,W,3] buffer) and with gaps between
    frames and rows (a strided view of a larger buffer)."""
    big = torch.zeros(x.shape[:2] + (2 * x.shape[2], x.shape[3] + 3, x.shape[4] + 5), dtype=x.dtype, device=x.device)
    big[:, :, ::2, 1:x.shape[3] + 1, 2:x.shape[4] + 2] = x
    return {"contiguous": x, "channels-last": x.permute(0, 1, 3, 4, 2).contiguous().permute(0, 1, 4, 2, 3),
            "strided": big[:, :, ::2, 1:x.shape[3] + 1, 2:x.shape[4] + 2]}


def _offsets(B, T, H, W, h, w, seed):
    """Fixed offsets at the last row and column, a random [T,2] and a random [B,T,2]."""
    g = torch.Generator().manual_seed(seed)
    rand = lambda *lead: torch.stack([torch.randint(0, H - h + 1, lead, generator=g),     # noqa: E731
                                      torch.randint(0, W - w + 1, lead, generator=g)], -1)
    return [(H - h, W - w), rand(T), rand(B, T)]


WINDOWS = [(1, 1), (17, 30), (37, 53)]     # one pixel, a window, the whole 37 x 53 frame


@pytest.mark.parametrize("form", ["contiguous", "channels-last", "strided"])
@pytest.mark.parametrize("where", ["host", "device"])
@pytest.mark.parametrize("dtype", [torch.uint8, torch.float32])
def test_rgb_ingest_equals_the_materialised_window(dtype, where, form, monkeypatch):
    B, T, H, W = 2, 5, 37, 53
    g = torch.Generator().manual_seed(3)
    x = torch.randint(0, 256, (B, T, 3, H, W), generator=g).to(dtype)
    video = _forms(x.to(DEV) if where == "device" else x)[form]
    for size in WINDOWS:
        for off in _offsets(B, T, H, W, *size, seed=size[0]):
            want_clip = _materialise(x, off, size).to(DEV)
            for out_hw in ((24, 40), size):          # a resize and the same-size copy
                want = ingest.prepare_video(want_clip, out_hw, DEV)
                assert torch.equal(ingest.prepare_video(Crop(video, size, off), out_hw, DEV), want), (size, off)
    if where == "host":   # chunks of two frames and slots smaller than a frame, windows moving inside a chunk
        size, off = (17, 30), _offsets(B, T, H, W, 17, 30, seed=5)[2]
        want = ingest.prepare_video(_materialise(x, off, size).to(DEV), (24, 40), DEV)
        for slot in (2 * 3 * 17 * 30 * x.element_size(), 100):
            monkeypatch.setattr(ingest, "STAGING_SLOT_BYTES", slot)
            assert torch.equal(ingest.prepare_video(Crop(video, size, off), (24, 40), DEV), want)


COLOURS = [("bt601", False), ("bt709", False), ("bt2020", True)]


@pytest.mark.parametrize("where", ["host", "device"])
@pytest.mark.parametrize("colour", COLOURS, ids=[f"{m}-{'full' if f else 'limited'}" for m, f in COLOURS])
@pytest.mark.parametrize("layout", list(C.FORMATS))
def test_yuv_ingest_equals_the_window_of_its_rgb(layout, colour, where):
    m, f = colour
    B, T, H, W = 2, 4, 36, 52
    data = C.random_frames(layout, (B, T), H, W, seed=7)
    rgb = C.yuv_to_rgb(layout, data, m, f)
    clip = YUVClip(data.to(DEV) if where == "device" else data, layout, matrix=m, full_range=f)
    odd_even = torch.tensor([[0, 0], [1, 1], [2, 3], [3, 2]])           # every parity of (top, left)
    for size in ((17, 23), (16, 22), (1, 1), (H, W)):
        h, w = size
        offs = [(H - h, W - w), (min(1, H - h), min(1, W - w)),
                torch.minimum(odd_even, torch.tensor([H - h, W - w])),
                torch.stack([torch.minimum(odd_even, torch.tensor([H - h, W - w])),
                             torch.tensor([H - h, W - w]) - torch.minimum(odd_even, torch.tensor([H - h, W - w]))])]
        for off in offs:
            want = ingest.prepare_video(_materialise(rgb, off, size).to(DEV), (24, 40), DEV)
            assert torch.equal(ingest.prepare_video(Crop(clip, size, off), (24, 40), DEV), want), (size, off)


def test_negative_frame_stride_through_the_abi():
    """The crop entry points read a clip played backwards (a negative frame stride) as the kernel reads any stride."""
    T, H, W, h, w = 4, 30, 44, 13, 21
    g = torch.Generator().manual_seed(9)
    x = torch.randint(0, 256, (T, 3, H, W), generator=g, dtype=torch.uint8).to(DEV)
    off = torch.tensor([[0, 0], [17, 23], [5, 8], [9, 1]], dtype=torch.int32)
    rev = torch.flip(off, [0])
    want = ingest.prepare_video(_materialise(x.flip(0)[None], rev, (h, w))[0][None], (20, 28), DEV)
    out = torch.empty(T, 3, 20, 28, device=DEV)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    last = ctypes.c_void_p(x[T - 1].data_ptr())
    rc = engine.lib().ct3_prepare_frames_crop(last, 0, T, H, W, -x.stride(0), *x.stride()[1:],
                                              ctypes.c_void_p(rev.to(DEV).data_ptr()), h, w, 20, 28,
                                              ctypes.c_void_p(out.data_ptr()), stream)
    assert rc == 0 and torch.equal(out, want)
    data = C.random_frames("nv12", (T,), H, W, seed=10).to(DEV)
    rgb = C.yuv_to_rgb("nv12", data.cpu()).to(DEV)
    want = ingest.prepare_video(_materialise(rgb.flip(0)[None], rev, (h, w)), (20, 28), DEV)
    rc = engine.lib().ct3_prepare_frames_yuv_crop(ctypes.c_void_p(data[T - 1].data_ptr()), 0, 0, 0, T, H, W,
                                                  -data.stride(0), W, ctypes.c_void_p(rev.to(DEV).data_ptr()), h, w,
                                                  20, 28, ctypes.c_void_p(out.data_ptr()), stream)
    assert rc == 0 and torch.equal(out, want)


# ---- entry points ---------------------------------------------------------------------------------------------------
def _offline(seed=43):
    p = CoTrackerPredictor(checkpoint=None, window_len=60)
    p.model.load_state_dict(seeded_state_dict(seed, offline=True, window_len=60, head_gain=10.0, vis_gain=100.0))
    return p.to(DEV)


def _online(seed=47, S=16):
    p = CoTrackerOnlinePredictor(checkpoint=None, window_len=S)
    p.model.load_state_dict(seeded_state_dict(seed, offline=False, window_len=S, head_gain=10.0, vis_gain=100.0))
    return p.to(DEV)


def _equal(a, b):
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_equal(x, y) for x, y in zip(a, b))
    return torch.equal(a, b) if torch.is_tensor(a) else a == b      # None, or the ids seed_corners returns


def _moving(T, H, W, h, w, B=None):
    """A window sweeping down and right, [T,2], or B of them at different speeds [B,T,2]."""
    t = torch.arange(T)
    one = lambda k: torch.stack([(k * t) % (H - h + 1), (2 * k * t + 3) % (W - w + 1)], -1)   # noqa: E731
    return one(1) if B is None else torch.stack([one(k + 1) for k in range(B)])


def test_offline_predictor_every_mode():
    p = _offline()
    T, H, W, h, w = 12, 96, 160, 64, 96
    video = texture_video(T, H, W, seed=5).to(torch.uint8)                           # on the host
    off = _moving(T, H, W, h, w)
    crop, mat = Crop(video, (h, w), off), _materialise(video, off, (h, w))
    q = random_queries(24, T, h, w, seed=6).to(DEV)
    mask = torch.zeros(1, 1, h, w, device=DEV)
    mask[..., 10:50, 20:80] = 1
    for kw in (dict(queries=q), dict(grid_size=8, segm_mask=mask), dict(queries=q, backward_tracking=True),
               dict(grid_size=6, grid_query_frame=5, backward_tracking=True)):
        assert _equal(p(crop, return_scores=True, **kw), p(mat, return_scores=True, **kw)), kw
    small = (32, 80)                   # dense: grid step W // 80 = 1, 2560 tracks (dense mode needs W >= 80)
    dense_off = _moving(T, H, W, *small)
    assert _equal(p(Crop(video.to(DEV), small, dense_off), return_scores=True),
                  p(_materialise(video, dense_off, small).to(DEV), return_scores=True))
    video2 = torch.cat([video, texture_video(T, H, W, seed=8).to(torch.uint8)]).to(DEV)     # B = 2, per-clip offsets
    off2 = _moving(T, H, W, h, w, B=2)
    q2 = q.expand(2, -1, -1)
    assert _equal(p(Crop(video2, (h, w), off2), queries=q2, return_scores=True),
                  p(_materialise(video2, off2, (h, w)), queries=q2, return_scores=True))


def test_list_call_and_encoded_clip():
    p = _offline()
    T, H, W = 10, 96, 160
    video = texture_video(T, H, W, seed=9).to(torch.uint8).to(DEV)
    sizes = [(64, 96), (48, 48), (80, 128)]
    offs = [_moving(T, H, W, *s) for s in sizes]
    crops = [Crop(video, s, o) for s, o in zip(sizes, offs)]
    mats = [_materialise(video, o, s) for s, o in zip(sizes, offs)]
    qs = [random_queries(12, T, s[0], s[1], seed=k).to(DEV) for k, s in enumerate(sizes)]
    assert _equal(p(crops, queries=qs, return_scores=True), p(mats, queries=qs, return_scores=True))
    clip = p.encode(Crop(video.cpu(), sizes[0], offs[0]))
    want = p(mats[0], queries=qs[0], return_scores=True)
    assert _equal(p(clip, queries=qs[0], return_scores=True), want)
    clip.to("cpu")
    clip.to(DEV)
    assert _equal(p(clip, queries=qs[0], return_scores=True), want)


def test_online_predictor_over_a_moving_window():
    S = 16
    T, H, W, h, w = 40, 96, 128, 64, 80
    video = texture_video(T, H, W, seed=12).to(torch.uint8)
    off = _moving(T, H, W, h, w)
    crop, mat = Crop(video, (h, w), off), _materialise(video, off, (h, w))
    res = []
    for clip in (crop, mat):
        p = _online(S=S)
        p(clip[:, :S], is_first_step=True, grid_size=5)
        steps = []
        for ind in range(0, T - p.step, p.step):   # the reference's loop; results are copied before the next step
            tr, vi, sc = p(clip[:, ind:ind + 2 * p.step], return_scores=True)
            steps.append((tr.clone(), vi.clone(), tuple(x.clone() for x in sc)))
        res.append(steps)
    assert _equal(res[0], res[1])
    tracks = res[0][-1][0]
    assert torch.equal(crop.to_frame(tracks, frames=slice(T - tracks.shape[1], T)),
                       tracks + off.flip(-1)[T - tracks.shape[1]:].float().to(DEV)[None, :, None])


def test_online_streams_moving_window_preview_and_seed_corners():
    S = 16
    T, H, W, h, w = 32, 96, 128, 64, 96
    data = C.as_frames("nv12", texture_video(T, H, W, seed=19)[0].to(torch.uint8))[None]     # host NV12
    rgb = C.yuv_to_rgb("nv12", data)
    off = _moving(T, H, W, h, w)
    crop = Crop(YUVClip(data, "nv12"), (h, w), off)
    mat = _materialise(rgb, off, (h, w)).to(DEV)
    res = []
    for clip in (crop, mat):
        hub = OnlineStreams(_online(S=S))
        sid = hub.open(frame_size=(h, w), grid_size=4)
        steps = []
        for kind, a, b in (("c", 0, S), ("p", S // 2, S + 4), ("c", S // 2, S + S // 2), ("c", S, 2 * S)):
            hub.push(sid, clip[:, a:b], preview=kind == "p")
            if kind == "c" and a:
                steps.append(hub.seed_corners(sid, 8, min_distance=8))
            steps.append(hub.step(return_scores=True)[sid])
        res.append(steps)
    assert _equal(res[0], res[1])


def test_detect_corners_and_evaluation_predictor():
    T, H, W, h, w = 6, 96, 128, 48, 64
    video = texture_video(2 * T, H, W, seed=23).to(torch.uint8).view(2, T, 3, H, W)
    off = _moving(T, H, W, h, w, B=2)
    mat = _materialise(video, off, (h, w))
    for dev in ("cpu", DEV):
        got = detect_corners(Crop(video.to(dev), (h, w), off), 20, frame=3, min_distance=4)
        want = detect_corners(mat.to(dev), 20, frame=3, min_distance=4)
        assert _equal(got, want) and sum(g.shape[1] for g in got) > 5
    ev = EvaluationPredictor(_offline().model, interp_shape=(384, 512), grid_size=3, local_grid_size=0,
                             num_uniformly_sampled_pts=0)
    q = random_queries(1, T, h, w, seed=2).to(DEV)
    assert _equal(ev(Crop(video[:1], (h, w), off[0]), q), ev(mat[:1], q))


def test_to_frame_of_a_moving_window_call():
    p = _offline()
    T, H, W, h, w = 8, 96, 160, 64, 96
    video = texture_video(T, H, W, seed=31).to(torch.uint8).to(DEV)
    off = _moving(T, H, W, h, w)
    crop = Crop(video, (h, w), off)
    q = random_queries(10, T, h, w, seed=3).to(DEV)
    tracks = p(crop, queries=q)[0]
    want = p(_materialise(video, off, (h, w)), queries=q)[0] + off.flip(-1).float().to(DEV)[None, :, None]
    assert torch.equal(crop.to_frame(tracks), want)
    in_frame = q + 7.0    # frame pixels: (x, y) - (left, top) of each query's frame, one fp32 subtraction
    in_frame[..., 0] = q[..., 0]
    want = in_frame.clone()
    want[0, :, 1:] -= off.flip(-1)[q[0, :, 0].long().cpu()].float().to(DEV)
    assert torch.equal(crop.from_frame(in_frame), want)
