"""GPU tests of clip ingestion (ct3_prepare_frames, cotracker_b200.ingest) and of encoding once per predictor call:
the kernel against the ATen expression bit for bit, every predictor on uint8 host / device clips against the float
device path bit for bit and against its golden, the reversed pyramid against the pyramid of the reversed clip, and the
peak device memory of a 1080p host clip."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from cases import CASES, case_inputs, compare, load_golden, predictor_kwargs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _aten(src, oh, ow):
    """Today's preprocessing: the ATen expression the kernel reproduces."""
    return 2.0 * (F.interpolate(src.float(), (oh, ow), mode="bilinear", align_corners=True) / 255.0) - 1.0


def _clip(T, H, W, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    if dtype == torch.uint8:
        x = torch.randint(0, 256, (T, 3, H, W), generator=g, dtype=torch.uint8)
    else:
        x = torch.rand(T, 3, H, W, generator=g) * 255.0      # not integers: every rounding of the blend shows
    return x.to(DEV)


SHAPES = [  # (T, H, W, oh, ow)
    (2, 720, 1296, 384, 512),    # down
    (3, 97, 131, 384, 512),      # up, odd
    (2, 384, 512, 384, 512),     # same size: ATen's copy
    (1, 1, 77, 5, 33),           # H == 1
    (2, 45, 1, 20, 7),           # W == 1
    (2, 61, 83, 1, 1),           # output 1 x 1 (scale 0)
    (1, 384, 300, 384, 512),     # one axis equal
    (3, 200, 256, 77, 91),
]


@pytest.mark.parametrize("dtype", [torch.uint8, torch.float32])
@pytest.mark.parametrize("shape", SHAPES)
def test_prepare_frames_bitwise_equals_aten(shape, dtype):
    from cotracker_b200 import engine
    T, H, W, oh, ow = shape
    x = _clip(T, H, W, dtype, seed=T * 7 + H + W)
    want = _aten(x, oh, ow)
    got = engine.prepare_frames(x, (oh, ow))
    assert got.is_contiguous() and got.dtype == torch.float32
    assert torch.equal(got, want), float((got - want).abs().max())
    # the same frames stored channels-last [T,H,W,3] and seen through permute: read in place, same result
    thwc = x.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
    assert torch.equal(engine.prepare_frames(thwc, (oh, ow)), want)


def test_prepare_frames_strided_views():
    """Frame/row/column subsampling views (non-dense strides) go through the same kernel."""
    from cotracker_b200 import engine
    x = _clip(6, 130, 170, torch.uint8, seed=5)
    v = x[::2, :, 1::3, ::2]
    assert torch.equal(engine.prepare_frames(v, (384, 512)), _aten(v, 384, 512))


@pytest.mark.parametrize("dtype", [torch.uint8, torch.float32])
def test_prepare_video_host_chunks_match_device(dtype):
    """The host path (chunked pinned upload, small slot -> many chunks, both slot reuse paths) equals the device path."""
    from cotracker_b200 import ingest
    x = _clip(11, 90, 120, dtype, seed=9)
    want = _aten(x, 384, 512)
    host = x.cpu()
    old = ingest.STAGING_SLOT_BYTES
    try:
        ingest.STAGING_SLOT_BYTES = 3 * 3 * 90 * 120 * x.element_size()       # 3 frames per chunk, 4 chunks
        assert len(ingest.plan_chunks(11, 3 * 90 * 120 * x.element_size())) == 4
        variants = [host[None],                                                     # TCHW
                    host.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)[None],  # THWC, dense frames
                    host[::2][None],                                                # dense frames, gaps between them
                    host[:, :, :, :100][None]]                                      # frames not dense
        assert [ingest.frame_is_dense(v.shape[2:], v.stride()[2:]) for v in variants] == [True, True, True, False]
        for v in variants:
            ref = want if v.shape[1:] == host.shape else _aten(v[0].to(DEV), 384, 512)
            got = ingest.prepare_video(v, (384, 512), DEV)
            torch.cuda.synchronize()
            assert torch.equal(got, ref)
    finally:
        ingest.STAGING_SLOT_BYTES = old


@pytest.mark.parametrize("dtype", [torch.float16, torch.float64])
@pytest.mark.parametrize("where", ["host", "device"])
def test_other_float_dtypes_are_the_float32_path(dtype, where):
    """float16 / float64 clips are cast to float32 before the kernel; for pixel values 0..255 that cast is exact, so the
    result is the float32 clip's, bit for bit."""
    from cotracker_b200 import ingest
    x = _clip(5, 97, 131, torch.uint8, seed=3).float()
    v = x.to(dtype)
    assert torch.equal(v.float(), x)
    v = v if where == "device" else v.cpu()
    assert torch.equal(ingest.prepare_video(v[None], (384, 512), DEV), _aten(x, 384, 512))


# ---- end to end -------------------------------------------------------------------------------------------------
E2E_CASES = ["predictor_grid", "predictor_queries", "pred_segm_mask", "pred_backward", "pred_grid_query_frame",
             "pred_dense", "c1_apple_grid10", "predictor_online", "pred_online_support_grid"]


def _predictor(name):
    from cotracker_b200.predictor import CoTrackerOnlinePredictor, CoTrackerPredictor
    cfg = CASES[name]
    sd, video, queries = case_inputs(cfg)
    cls = CoTrackerOnlinePredictor if cfg["kind"] == "predictor_online" else CoTrackerPredictor
    p = cls(checkpoint=None, window_len=cfg["window_len"])
    p.model.load_state_dict(sd)
    return cfg, p.to(DEV), video, queries


def _run(cfg, p, video, queries):
    """The case's public predictor calls on `video` as given (host or device, any dtype); queries as given."""
    out = {}
    with torch.no_grad():
        if cfg["kind"] == "predictor_online":
            p(video_chunk=video, is_first_step=True, **predictor_kwargs(cfg, video, queries))
            for k, ind in enumerate(range(0, video.shape[1] - p.step, p.step)):
                tr, vi = p(video_chunk=video[:, ind:ind + p.step * 2], add_support_grid=cfg.get("add_support_grid", False))
                out[f"tracks{k}"], out[f"visibility{k}"] = tr.clone(), vi.clone()
        else:
            tr, vi = p(video, **predictor_kwargs(cfg, video, queries))
            out = dict(tracks=tr, visibility=vi)
    for v in out.values():
        assert v.device == torch.device(DEV)
    return {k: v.cpu() for k, v in out.items()}


def _as_uint8(name, video):
    if CASES[name].get("video") == "apple":       # natively uint8 [T,H,W,3]: the decoder's layout, read in place
        with np.load(CASES_APPLE) as z:
            return torch.from_numpy(z["frames"]).permute(0, 3, 1, 2)[None]
    assert torch.equal(video, video.round()) and float(video.max()) <= 255
    return video.to(torch.uint8)


from oracle.make_golden import APPLE_FIXTURE as CASES_APPLE  # noqa: E402


@pytest.mark.parametrize("name", E2E_CASES)
def test_uint8_host_and_device_clips_bit_identical(name):
    cfg, p, video, queries = _predictor(name)
    want = _run(cfg, p, video.to(DEV), None if queries is None else queries.to(DEV))      # float device path
    u8 = _as_uint8(name, video)
    assert torch.equal(u8.float(), video)
    for clip, q in ((u8, queries), (u8.to(DEV), None if queries is None else queries.to(DEV))):
        got = _run(cfg, p, clip, q)
        assert got.keys() == want.keys()
        for k in want:
            assert torch.equal(got[k], want[k]), (name, k, clip.device)
    print(name, compare(want, load_golden(name), tol_px=1e-3, tol_logit=1e-3))


def test_evaluation_predictor_uint8_host_and_device_bit_identical():
    from cotracker_b200.build import build_cotracker
    from cotracker_b200.evaluation import EvaluationPredictor
    from oracle.make_eval_single_golden import eval_single_inputs
    sd, video, queries = eval_single_inputs()
    model = build_cotracker(None, offline=True, window_len=60).eval()
    model.load_state_dict(sd)
    ev = EvaluationPredictor(model.to(DEV), single_point=True, grid_size=5, local_grid_size=8)
    want = ev(video.to(DEV), queries.to(DEV))
    for clip, q in ((video.to(torch.uint8), queries), (video.to(torch.uint8).to(DEV), queries.to(DEV))):
        got = ev(clip, q)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]), clip.device
    gold = load_golden("eval_predictor_single_t24")
    e_t = float((want[0].cpu() - gold["tracks"]).abs().max())
    e_v = float((want[1].cpu() - gold["vis"]).abs().max())
    assert e_t < 1e-3 and e_v < 1e-3, (e_t, e_v)


# ---- encode once ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T", [21, 40])
@pytest.mark.parametrize("offline", [True, False])
def test_reversed_pyramid_equals_pyramid_of_reversed_clip(T, offline):
    """The encoder output of a frame does not depend on which frames share its 16-frame chunk, so the pyramid reversed
    in place (with the sliding-window model's padding, copies of the original frame 0) is the reversed clip's."""
    from cotracker_b200.build import build_cotracker
    from cotracker_b200.synthetic import seeded_state_dict, texture_video
    sd = seeded_state_dict(3, offline=offline, window_len=60 if offline else 16)
    m = build_cotracker(None, offline=offline, window_len=60 if offline else 16).eval()
    m.load_state_dict(sd)
    m = m.to(DEV)
    frames = 2.0 * (texture_video(T, 128, 160, seed=T)[0].to(DEV) / 255.0) - 1.0
    with torch.no_grad():
        pyr = m._encode_clip(frames)
        orig = pyr.clone()
        rev = m._reverse_clip_pyramid_(pyr, T, 128, 160)
        want = m._encode_clip(frames.flip(0).contiguous())
    assert rev.data_ptr() == pyr.data_ptr()                  # in place: no second pyramid
    assert rev.shape == want.shape
    assert torch.equal(rev, want)
    m._reverse_clip_pyramid_(pyr, T, 128, 160)
    assert torch.equal(pyr, orig)                            # reversing again restores the clip's pyramid


def _old_sparse(p, video, queries, backward, support):
    """The predictor's sequence before the clip was encoded once: ATen resize, model.forward on the resized clip and,
    for backward tracking, model.forward on the flipped clip.  support: append the 6x6 support grid (what the
    predictor does for explicit queries) and drop its columns at the end."""
    from cotracker_b200.predictor import get_points_on_a_grid
    B, T, C, H, W = video.shape
    ih, iw = p.interp_shape
    v = F.interpolate(video.reshape(T, C, H, W), (ih, iw), mode="bilinear", align_corners=True).reshape(1, T, 3, ih, iw)
    q = queries.clone()
    q[:, :, 1:] *= q.new_tensor([(iw - 1) / (W - 1), (ih - 1) / (H - 1)])
    n = q.shape[1]
    if support:
        sup = get_points_on_a_grid(6, p.interp_shape, device=q.device)
        q = torch.cat([q, torch.cat([torch.zeros_like(sup[:, :, :1]), sup], dim=2)], dim=1)
    tracks, vis, *_ = p.model(video=v, queries=q, iters=6)
    if backward:
        iq = q.clone()
        iq[:, :, 0] = T - iq[:, :, 0] - 1
        it, ivis, *_ = p.model(video=v.flip(1).clone(), queries=iq, iters=6)
        it, ivis = it.flip(1), ivis.flip(1)
        before = torch.arange(T, device=q.device)[None, :, None] < q[:, None, :, 0]
        tracks = torch.where(before[..., None], it, tracks)
        vis = torch.where(before, ivis, vis)
    tracks, vis, q = tracks[:, :, :n], vis[:, :, :n], q[:, :n]
    vis = vis > 0.9
    idx = torch.arange(tracks.size(2), device=tracks.device)
    qt = q[0, :, 0].to(torch.int64)
    tracks[0, qt, idx] = q[0, :, 1:]
    vis[0, qt, idx] = True
    tracks *= tracks.new_tensor([(W - 1) / (iw - 1), (H - 1) / (ih - 1)])
    return tracks, vis


@pytest.mark.parametrize("offline", [True, False])
def test_backward_tracking_equals_explicit_flipped_pass(offline):
    from cotracker_b200.predictor import CoTrackerPredictor
    from cotracker_b200.synthetic import random_queries, seeded_state_dict, texture_video
    S = 60 if offline else 16
    p = CoTrackerPredictor(checkpoint=None, offline=offline, window_len=S)
    p.model.load_state_dict(seeded_state_dict(41, offline=offline, window_len=S, head_gain=10.0, vis_gain=100.0))
    p = p.to(DEV)
    T, H, W = 21, 144, 192
    video = texture_video(T, H, W, seed=42).to(DEV)
    queries = random_queries(13, T, H, W, seed=43).to(DEV)
    assert int(queries[0, :, 0].max()) > T // 2                # queries at later frames: the backward pass matters
    with torch.no_grad():
        got = p(video, queries=queries, backward_tracking=True)
        want = _old_sparse(p, video, queries, backward=True, support=True)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


@pytest.mark.parametrize("backward", [False, True])
def test_dense_equals_per_offset_passes(backward):
    """Dense passes on one shared pyramid; with backward tracking every pass flips that pyramid in place and back."""
    cfg, p, video, _ = _predictor("pred_dense")
    video = video.to(DEV)
    H, W = video.shape[3:]
    gq = video.shape[1] - 1 if backward else 0        # queries at the last frame: the backward pass decides the tracks
    with torch.no_grad():
        got = p(video, grid_query_frame=gq, backward_tracking=backward)
        step = W // 80
        gw, gh = W // step, H // step
        base_x = (torch.arange(gw, device=DEV).repeat(gh) * step).float()
        base_y = (torch.arange(gh, device=DEV).repeat_interleave(gw) * step).float()
        parts = []
        for offset in range(step * step):
            pts = torch.zeros(1, gw * gh, 3, device=DEV)
            pts[:, :, 0] = gq
            pts[:, :, 1] = base_x + offset % step
            pts[:, :, 2] = base_y + offset // step
            parts.append(_old_sparse(p, video, pts, backward=backward, support=False))
    assert step > 1
    assert torch.equal(got[0], torch.cat([t for t, _ in parts], dim=2))
    assert torch.equal(got[1], torch.cat([v for _, v in parts], dim=2))


# ---- memory -----------------------------------------------------------------------------------------------------
def test_host_uint8_1080p_clip_peak_memory():
    """A 1920x1080x48 uint8 host clip at grid 10: the device never holds the clip, only two staging chunks of it."""
    from cotracker_b200 import engine, ingest
    from cotracker_b200.predictor import CoTrackerPredictor
    from cotracker_b200.synthetic import seeded_state_dict
    T, H, W, grid = 48, 1080, 1920, 10
    p = CoTrackerPredictor(checkpoint=None, window_len=60)
    p.model.load_state_dict(seeded_state_dict(7, offline=True, window_len=60))
    p = p.to(DEV)
    g = torch.Generator().manual_seed(0)
    clip = torch.randint(0, 256, (T, H, W, 3), generator=g, dtype=torch.uint8).permute(0, 3, 1, 2)[None]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    with torch.no_grad():
        tracks, vis = p(clip, grid_size=grid)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    assert tracks.shape == (1, T, grid * grid, 2)
    ih, iw = p.interp_shape
    N = grid * grid
    frames = T * 3 * ih * iw * 4
    pyramid = engine.pyramid_layout(T, ih // 4, iw // 4)[3] * 4
    bound = (frames + pyramid + engine.encoder_workspace_bytes(T, ih, iw)
             + engine.workspace_bytes(T, N, ih // 4, iw // 4) + N * 4 * 49 * 128 * 4
             + engine.packed_weights_bytes() + (64 << 20)                     # packed weights (both nets) < 64 MiB
             + ingest.staging_bytes(T, 3 * H * W)                            # two raw chunks on the device
             + (64 << 20))                                                    # slack: state, outputs, small temporaries
    float_clip = T * 3 * H * W * 4
    print(f"peak {peak / 2**20:.0f} MiB, bound {bound / 2**20:.0f} MiB, float clip {float_clip / 2**20:.0f} MiB, "
          f"staging {ingest.staging_bytes(T, 3 * H * W) / 2**20:.0f} MiB")
    assert peak <= bound
    assert ingest.staging_bytes(T, 3 * H * W) < float_clip // 10
    # the bound is tight enough to catch the clip on the device: holding the float clip (or half of it) would not fit
    # in the slack between the measured peak and the bound
    assert bound - peak < float_clip // 2, (bound - peak, float_clip)
