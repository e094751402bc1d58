"""GPU tests of `CoTrackerPredictor.encode` and `EncodedClip`: every offline predictor golden through an encoded clip,
`torch.equal` to the direct call and within the goldens' tolerance of the reference; one clip queried many times in
every mode without a byte of its pyramid changing; batches, host uint8, YUV and sliding-window clips; parking on the
host and back, bit-identical; `ct3_pyramid_pools` against the encoder's own levels, odd sizes included; and every
rejection at the boundary."""
import copy

import pytest
import torch

from cases import CASES, case_inputs, compare, load_golden, predictor_kwargs
from cotracker_b200 import EncodedClip, YUVClip, detect_corners, engine
from cotracker_b200.evaluation import EvaluationPredictor
from cotracker_b200.predictor import CoTrackerOnlinePredictor, CoTrackerPredictor
from cotracker_b200.streams import OnlineStreams
from cotracker_b200.synthetic import random_queries, seeded_state_dict, texture_video
from cotracker_b200.visualizer import Visualizer

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FIXTURES = ["predictor_grid", "predictor_queries", "pred_segm_mask", "pred_backward", "pred_grid_query_frame",
            "pred_dense"]


def _predictor(offline=True, window_len=60, seed=61):
    p = CoTrackerPredictor(checkpoint=None, offline=offline, window_len=window_len)
    p.model.load_state_dict(seeded_state_dict(seed, offline=offline, window_len=window_len, head_gain=10.0,
                                              vis_gain=100.0))
    return p.to(DEV)


def _bits(t):
    return t.contiguous().view(torch.int32)


def _assert_same(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        if isinstance(w, tuple):   # TrackScores
            _assert_same(g, w)
        else:
            assert g.dtype == w.dtype and torch.equal(g, w)


def _tracked_equal(p, clip, video, **kw):
    """p(clip, **kw) is torch.equal to p(video, **kw) and leaves every byte of the clip's pyramid as it was."""
    before = clip.pyr.clone()
    got = p(clip, **kw)
    _assert_same(got, p(video, **kw))
    assert torch.equal(_bits(clip.pyr), _bits(before)), kw
    return got


@pytest.mark.parametrize("scores", [False, True])
@pytest.mark.parametrize("name", FIXTURES)
def test_goldens_through_an_encoded_clip(name, scores):
    cfg = CASES[name]
    sd, video, queries = case_inputs(cfg)
    p = CoTrackerPredictor(checkpoint=None, window_len=cfg["window_len"])
    p.model.load_state_dict(sd)
    p = p.to(DEV)
    video = video.to(DEV)
    kw = predictor_kwargs(cfg, video, None if queries is None else queries.to(DEV))
    clip = p.encode(video)
    assert isinstance(clip, EncodedClip) and clip.B == 1 and clip.T == cfg["T"]
    assert clip.input_hw == (cfg["H"], cfg["W"]) and clip.interp_shape == tuple(p.interp_shape)
    assert clip.stride == p.model.stride and clip.device == torch.device(DEV)
    assert clip.weights == p.model.weights_fingerprint() and clip.nbytes == clip.pyr.numel() * 4
    got = _tracked_equal(p, clip, video, return_scores=scores, **kw)
    compare(dict(tracks=got[0].cpu(), visibility=got[1].cpu()), load_golden(name))


@pytest.mark.parametrize("offline", [True, False])
def test_one_clip_many_query_sets(offline):
    """Sparse, grid, backward, segm_mask, dense and sparse again on one clip: each equal to its own direct call."""
    p = _predictor(offline, 60 if offline else 16)
    T, H, W = 21, 96, 160
    video = texture_video(T, H, W, seed=62).to(DEV)
    clip = p.encode(video)
    mask = torch.zeros(1, 1, H, W, device=DEV)
    mask[:, :, 20:80, 30:120] = 1
    for kw in (dict(queries=random_queries(11, T, H, W, seed=63).to(DEV)),
               dict(grid_size=6),
               dict(queries=random_queries(7, T, H, W, seed=64).to(DEV), backward_tracking=True),
               dict(grid_size=5, grid_query_frame=T - 4, backward_tracking=True, return_scores=True),
               dict(grid_size=8, segm_mask=mask),
               dict(),
               dict(queries=random_queries(11, T, H, W, seed=63).to(DEV), return_scores=True)):
        _tracked_equal(p, clip, video, **kw)


def _nv12(T, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return YUVClip(torch.randint(16, 236, (1, T, H * 3 // 2, W), generator=g, dtype=torch.uint8), "nv12")


@pytest.mark.parametrize("source", ["batch2", "host_uint8", "yuv_host", "yuv_device", "sliding_batch2"])
def test_sources(source):
    T, H, W = 19, 120, 176
    p = _predictor(offline=not source.startswith("sliding"), window_len=60 if source != "sliding_batch2" else 16)
    if source in ("batch2", "sliding_batch2"):
        video = torch.cat([texture_video(T, H, W, seed=65), texture_video(T, H, W, seed=66)]).to(DEV)
        queries = torch.cat([random_queries(9, T, H, W, seed=67), random_queries(9, T, H, W, seed=68)]).to(DEV)
    elif source == "host_uint8":   # a channels-last decoder buffer seen as [B,T,3,H,W]
        video = texture_video(T, H, W, seed=65).to(torch.uint8).permute(0, 1, 3, 4, 2).contiguous()
        video = video.permute(0, 1, 4, 2, 3)
        queries = random_queries(9, T, H, W, seed=67).to(DEV)
    else:
        video = _nv12(T, H, W, 69)
        video = video.to(DEV) if source == "yuv_device" else video
        queries = random_queries(9, T, H, W, seed=67).to(DEV)
    clip = p.encode(video)
    assert clip.B == video.shape[0] and clip.video_shape == video.shape
    _tracked_equal(p, clip, video, queries=queries, backward_tracking=True, return_scores=True)
    _tracked_equal(p, clip, video, grid_size=7)


@pytest.mark.parametrize("offline,B", [(True, 1), (False, 1), (False, 2)])
def test_park_and_return(offline, B):
    T, H, W = 21, 144, 192
    p = _predictor(offline, 60 if offline else 16)
    video = torch.cat([texture_video(T, H, W, seed=70 + b) for b in range(B)]).to(DEV)
    kw = dict(queries=torch.cat([random_queries(10, T, H, W, seed=72 + b) for b in range(B)]).to(DEV),
              backward_tracking=True, return_scores=True)
    clip = p.encode(video)
    want = p(clip, **kw)
    full = clip.pyr.clone()
    H4, W4 = 384 // 4, 512 // 4
    lv0 = full[:B * (T + clip.pad) * H4 * W4 * 128].view(B, T + clip.pad, -1)
    pad_is_copies = clip.pad > 0 and torch.equal(lv0[:, T:], lv0[:, T - 1:T].expand(-1, clip.pad, -1))
    assert offline == (clip.pad == 0)
    torch.cuda.synchronize()
    held, before = clip.nbytes, torch.cuda.memory_allocated(DEV)
    assert clip.to("cpu") is clip
    assert before - torch.cuda.memory_allocated(DEV) >= held
    assert clip.parked and clip.nbytes == 0 and clip.pyr is None and clip.host.is_pinned()
    kept = T if (clip.pad == 0 or pad_is_copies) else T + clip.pad
    assert clip.host.shape == (B, kept, H4, W4, 128)   # level 0 only
    assert torch.equal(_bits(clip.host.view(B, kept, -1)), _bits(lv0[:, :kept].cpu()))
    print(f"parked {clip.host.numel() * 4 / 2**20:.1f} MiB of {held / 2**20:.1f} MiB, padding frames "
          f"{'remade' if kept == T else 'parked'}")
    with pytest.raises(ValueError, match="parked"):
        p(clip, **kw)
    clip.to("cpu")   # parking twice is a no-op
    assert clip.to("cuda") is clip and clip.device == torch.device(DEV) and clip.host is None
    assert torch.equal(_bits(clip.pyr), _bits(full))
    _assert_same(p(clip, **kw), want)
    _assert_same(p(clip.to("cpu").to(DEV), **kw), want)


def test_pyramid_pools_rebuild_the_encoder_levels():
    m = _predictor().model
    g = torch.Generator().manual_seed(80)
    for T, H, W in ((5, 100, 132), (3, 36, 68), (2, 384, 512)):   # odd level sizes: 25x33 .. 3x4, 9x17 .. 1x2
        frames = (torch.rand(T, 3, H, W, generator=g) * 2 - 1).to(DEV)
        pyr = m._encode_clip(frames)
        off, *_ = engine.pyramid_layout(T, H // 4, W // 4)
        again = pyr.clone()
        again[off[1]:] = 0
        assert engine.pyramid_pools(again, T, H // 4, W // 4) is again
        assert torch.equal(_bits(again), _bits(pyr)), (T, H, W)
    p = _predictor(offline=False, window_len=16)   # a batch of two clips, each with its padding frames
    clip = p.encode(torch.cat([texture_video(11, 96, 128, seed=81), texture_video(11, 96, 128, seed=82)]).to(DEV))
    T_all = 2 * (clip.T + clip.pad)
    off, *_ = engine.pyramid_layout(T_all, 96, 128)
    again = clip.pyr.clone()
    again[off[1]:] = 0
    engine.pyramid_pools(again, T_all, 96, 128)
    assert torch.equal(_bits(again), _bits(clip.pyr))
    with pytest.raises(engine.EngineError, match="floats"):
        engine.pyramid_pools(again[:-1], T_all, 96, 128)


def test_rejections():
    T, H, W = 8, 96, 128
    p = _predictor()
    video = texture_video(T, H, W, seed=90).to(DEV)
    clip = p.encode(video)
    q = random_queries(4, T, H, W, seed=91).to(DEV)
    p(clip, queries=q)

    # the predictor's weights changed after the clip was encoded
    p2 = _predictor()
    c2 = p2.encode(video)
    with torch.no_grad():
        next(p2.model.fnet.parameters()).add_(0.5)
    with pytest.raises(ValueError, match="weights"):
        p2(c2, queries=q)
    # another predictor with the same weights tracks it, on its own model
    _assert_same(_predictor()(clip, queries=q), p(clip, queries=q))

    old = p.interp_shape
    p.interp_shape = (192, 256)
    with pytest.raises(ValueError, match="interp_shape"):
        p(clip, queries=q)
    p.interp_shape = old
    bad = copy.copy(clip)
    bad.stride = 8
    with pytest.raises(ValueError, match="stride"):
        p(bad, queries=q)
    with pytest.raises(ValueError, match="sliding-window"):
        p(_predictor(offline=False, window_len=16).encode(video), queries=q)
    with pytest.raises(ValueError, match="B == 1"):
        p(p.encode(torch.cat([video, video])), grid_size=5, segm_mask=torch.ones(1, 1, H, W, device=DEV))

    online = CoTrackerOnlinePredictor(checkpoint=None, window_len=16).to(DEV)
    with pytest.raises(TypeError, match="EncodedClip"):
        online(clip, is_first_step=True, grid_size=5)
    hub = OnlineStreams(online)
    sid = hub.open((H, W), grid_size=5)
    with pytest.raises(TypeError, match="EncodedClip"):
        hub.push(sid, clip)
    for call in (lambda: p([clip], grid_size=5), lambda: p([video, clip], queries=[q, q]),
                 lambda: EvaluationPredictor(p.model)(clip, q[:, :1]), lambda: detect_corners(clip, 10),
                 lambda: Visualizer(save_dir="/nonexistent").visualize(clip, torch.zeros(1, T, 4, 2), save_video=False),
                 lambda: p.encode(clip), lambda: p.encode([video])):
        with pytest.raises(TypeError, match="EncodedClip|list"):
            call()
    with pytest.raises(ValueError, match="CUDA device"):
        clip.to("meta")
    _assert_same(p(clip, queries=q), p(video, queries=q))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_clip_on_another_device_is_rejected():
    T, H, W = 8, 96, 128
    p = _predictor()
    video = texture_video(T, H, W, seed=92).to(DEV)
    q = random_queries(4, T, H, W, seed=93).to(DEV)
    clip = p.encode(video).to("cuda:1")
    with pytest.raises(ValueError, match="cuda:1"):
        p(clip, queries=q)
    _assert_same(p(clip.to(DEV), queries=q), p(video, queries=q))
