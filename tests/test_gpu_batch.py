"""GPU tests of batched tracking: slot b of a call on B clips is bit-identical to the call on clip b alone, for the
models, both predictors in every mode and a batch split by a small memory budget; a reference golden placed in a batch
still meets its bound; ct3_finish_tracks equals the torch expression it replaces bit for bit.  The clips of a batch
come from different seeds (pixels and queries), so cross-talk between clips cannot hide."""
import pytest
import torch

from cases import CASES, case_inputs, compare, load_golden, predictor_kwargs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
H, W = 96, 128


def _model(offline, seed=41):
    from cotracker_b200.build import build_cotracker
    from cotracker_b200.synthetic import seeded_state_dict
    S = 60 if offline else 16
    m = build_cotracker(None, offline=offline, window_len=S).eval()
    m.load_state_dict(seeded_state_dict(seed, offline=offline, window_len=S, head_gain=10.0, vis_gain=100.0))
    return m.to(DEV)


def _batch(B, T, N, h=H, w=W, seed=100):
    from cotracker_b200.synthetic import random_queries, texture_video
    video = torch.cat([texture_video(T, h, w, seed=seed + b, shift=(1 + b, 2)) for b in range(B)]).to(DEV)
    queries = torch.cat([random_queries(N, T, h, w, seed=seed + 50 + b) for b in range(B)]).to(DEV)
    return video, queries


def _assert_slots_equal(batched, single, what=""):
    """batched: tuple of [B,...] tensors; single(b) -> the same tuple of [1,...] tensors for clip b alone."""
    B = batched[0].shape[0]
    for b in range(B):
        for k, (got, want) in enumerate(zip(batched, single(b))):
            assert got[b:b + 1].shape == want.shape, (what, b, k, got.shape, want.shape)
            assert torch.equal(got[b:b + 1], want), (what, b, k)


# ---- models -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [2, 3])
@pytest.mark.parametrize("T", [60, 11])
def test_offline_model_slots_equal_single_clip_calls(B, T):
    m = _model(True)
    video, queries = _batch(B, T, 9)
    with torch.no_grad():
        got = m(video, queries, iters=3)[:3]
        assert got[0].shape == (B, T, 9, 2) and got[1].shape == (B, T, 9) and got[2].shape == (B, T, 9)
        _assert_slots_equal(got, lambda b: m(video[b:b + 1], queries[b:b + 1], iters=3)[:3])


@pytest.mark.parametrize("B", [2, 3])
def test_sliding_model_slots_equal_single_clip_calls(B):
    m = _model(False)
    video, queries = _batch(B, 40, 9)
    with torch.no_grad():
        got = m(video, queries, iters=3)[:3]
        assert got[0].shape == (B, 40, 9, 2)
        _assert_slots_equal(got, lambda b: m(video[b:b + 1], queries[b:b + 1], iters=3)[:3])


@pytest.mark.parametrize("B", [2, 3])
@pytest.mark.parametrize("offline", [True, False])
def test_forward_groups_with_a_reversed_group(B, offline):
    m = _model(offline)
    T = 21
    video, queries = _batch(B, T, 12)
    sizes, rev = [5, 4, 3], [False, True, False]
    with torch.no_grad():
        got = m.forward_groups(video, queries, sizes, iters=3, reversed_groups=rev)[:3]
        _assert_slots_equal(got, lambda b: m.forward_groups(video[b:b + 1], queries[b:b + 1], sizes, iters=3,
                                                            reversed_groups=rev)[:3], offline)


@pytest.mark.parametrize("B", [2, 3])
def test_streaming_model_slots_equal_single_streams(B):
    """B streams in lockstep, with one stream whose overlap frames change between chunks (so only it is re-encoded)."""
    S, T = 16, 48
    video, queries = _batch(B, T, 9)
    chunks = [video[:, ind:ind + S].clone() for ind in range(0, T - S // 2, S // 2)]
    chunks[2][1, :S // 2] += 1.0                         # stream 1: the overlap no longer matches its cache
    m, singles = _model(False), [_model(False) for _ in range(B)]
    m.init_video_online_processing()
    for s in singles:
        s.init_video_online_processing()
    with torch.no_grad():
        for chunk in chunks:
            got = m(chunk, queries, iters=3, is_online=True)[:3]
            _assert_slots_equal(got, lambda b: singles[b](chunk[b:b + 1], queries[b:b + 1], iters=3, is_online=True)[:3])


def test_a_clip_does_not_see_its_neighbour():
    for offline in (True, False):
        m = _model(offline)
        video, queries = _batch(2, 21, 9)
        other_v, other_q = _batch(2, 21, 9, seed=300)
        with torch.no_grad():
            base = m(video, queries, iters=3)[:3]
            for v1, q1 in ((other_v[1], queries[1]), (video[1], other_q[1])):
                got = m(torch.stack([video[0], v1]), torch.stack([queries[0], q1]), iters=3)[:3]
                assert all(torch.equal(g[0], w[0]) for g, w in zip(got, base)), offline
                assert not torch.equal(got[0][1], base[0][1])


# ---- predictors -------------------------------------------------------------------------------------------------
def _predictor(offline, seed=43):
    from cotracker_b200.predictor import CoTrackerPredictor
    from cotracker_b200.synthetic import seeded_state_dict
    S = 60 if offline else 16
    p = CoTrackerPredictor(checkpoint=None, offline=offline, window_len=S)
    p.model.load_state_dict(seeded_state_dict(seed, offline=offline, window_len=S, head_gain=10.0, vis_gain=100.0))
    return p.to(DEV)


MODES = {
    "grid": dict(grid_size=5),
    "queries": dict(queries=True),
    "grid_query_frame_backward": dict(grid_size=4, grid_query_frame=7, backward_tracking=True),
    "queries_backward": dict(queries=True, backward_tracking=True),
}


@pytest.mark.parametrize("offline", [True, False])
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("B", [2, 3])
def test_predictor_slots_equal_single_clip_calls(B, mode, offline):
    p = _predictor(offline)
    T, h, w = 21, 144, 192
    video, queries = _batch(B, T, 7, h, w)
    kw = dict(MODES[mode])
    use_q = kw.pop("queries", False)
    with torch.no_grad():
        got = p(video, queries=queries if use_q else None, **kw)
        assert got[1].dtype == torch.bool and got[0].shape[:2] == (B, T)
        _assert_slots_equal(got, lambda b: p(video[b:b + 1], queries=queries[b:b + 1] if use_q else None, **kw), mode)
        # the same batch as a decoder hands it over: uint8 [B,T,H,W,3] on the host, seen through permute
        host = video.to(torch.uint8).permute(0, 1, 3, 4, 2).contiguous().cpu().permute(0, 1, 4, 2, 3)
        again = p(host, queries=queries if use_q else None, **kw)
        assert torch.equal(again[0], got[0]) and torch.equal(again[1], got[1])


@pytest.mark.parametrize("offline", [True, False])
@pytest.mark.parametrize("backward", [False, True])
def test_dense_slots_equal_single_clip_calls(offline, backward):
    p = _predictor(offline, seed=93)
    video, _ = _batch(2, 8, 1, 96, 160)            # grid step 2: 4 offsets of 48 x 80 tracks per clip
    gq = 7 if backward else 0
    with torch.no_grad():
        got = p(video, grid_query_frame=gq, backward_tracking=backward)
        _assert_slots_equal(got, lambda b: p(video[b:b + 1], grid_query_frame=gq, backward_tracking=backward))


@pytest.mark.parametrize("offline", [True, False])
def test_small_budget_splits_the_batch_and_keeps_the_bits(offline, monkeypatch):
    import cotracker_b200.predictor as P
    p = _predictor(offline)
    video, queries = _batch(3, 21, 7, 144, 192)
    calls = []
    track = type(p.model)._track_pyramid

    def spy(self, *a, **k):
        calls.append(k.get("clips"))
        return track(self, *a, **k)

    with torch.no_grad():
        want = p(video, queries=queries, backward_tracking=True)
        monkeypatch.setattr(P, "pass_budget_bytes", lambda *a, **k: 1)
        monkeypatch.setattr(type(p.model), "_track_pyramid", spy)
        got = p(video, queries=queries, backward_tracking=True)
    assert [list(c) for c in calls] == [[0], [1], [2]]            # one clip per pass
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


@pytest.mark.parametrize("support", [False, True])
def test_online_predictor_slots_equal_single_streams(support):
    from cotracker_b200.predictor import CoTrackerOnlinePredictor
    from cotracker_b200.synthetic import seeded_state_dict
    B, T, h, w = 3, 48, 144, 192

    def make():
        p = CoTrackerOnlinePredictor(checkpoint=None, window_len=16)
        p.model.load_state_dict(seeded_state_dict(47, offline=False, window_len=16, head_gain=10.0, vis_gain=100.0))
        return p.to(DEV)

    video, queries = _batch(B, T, 6, h, w)
    first = dict(queries=queries, add_support_grid=True) if support else dict(grid_size=4, grid_query_frame=2)
    p, singles = make(), [make() for _ in range(B)]
    n_chunks = 0
    with torch.no_grad():
        p(video_chunk=video, is_first_step=True, **first)
        for b, s in enumerate(singles):
            one = {k: (v[b:b + 1] if torch.is_tensor(v) else v) for k, v in first.items()}
            s(video_chunk=video[b:b + 1], is_first_step=True, **one)
        for ind in range(0, T - p.step, p.step):
            chunk = video[:, ind:ind + 2 * p.step]
            got = p(video_chunk=chunk, add_support_grid=support)
            assert got[0].shape[0] == B and got[0].shape[2] == (6 if support else 16)
            _assert_slots_equal(got, lambda b: singles[b](video_chunk=chunk[b:b + 1], add_support_grid=support))
            n_chunks += 1
    assert n_chunks >= 4


def test_reference_golden_in_a_batch_meets_its_bound():
    """A case pinned from the reference, tracked as clip 1 of a batch next to an unrelated clip."""
    from cotracker_b200.predictor import CoTrackerPredictor
    from cotracker_b200.synthetic import texture_video
    name = "predictor_grid"
    cfg = CASES[name]
    sd, video, queries = case_inputs(cfg)
    p = CoTrackerPredictor(checkpoint=None, window_len=cfg["window_len"])
    p.model.load_state_dict(sd)
    p = p.to(DEV)
    other = texture_video(video.shape[1], video.shape[3], video.shape[4], seed=977, shift=(3, 1))
    with torch.no_grad():
        tr, vi = p(torch.cat([other, video]).to(DEV), **predictor_kwargs(cfg, video, queries))
    print(compare(dict(tracks=tr[1:2].cpu(), visibility=vi[1:2].cpu()), load_golden(name), tol_px=1e-3, tol_logit=1e-3))


# ---- ct3_finish_tracks --------------------------------------------------------------------------------------------
def _finish_torch(queries, fwd, bwd, n_support, thr, scale):
    """The expression the kernel replaces (the predictor's tail as ATen ops)."""
    T = fwd[0].shape[1]
    tracks, vis = fwd[0].clone(), fwd[1].clone()
    if bwd is not None:
        before = torch.arange(T, device=DEV)[None, :, None] < queries[:, None, :, 0]
        tracks = torch.where(before[..., None], bwd[0].flip(1), tracks)
        vis = torch.where(before, bwd[1].flip(1), vis)
    if n_support:
        tracks, vis = tracks[:, :, :-n_support], vis[:, :, :-n_support]
    vis = vis > thr
    n = tracks.size(2)
    idx = torch.arange(n, device=DEV)
    for b in range(len(queries)):
        qt = queries[b, :n, 0].to(torch.int64)
        tracks[b, qt, idx] = queries[b, :n, 1:]
        vis[b, qt, idx] = True
    return tracks * tracks.new_tensor(scale), vis


@pytest.mark.parametrize("backward", [False, True])
@pytest.mark.parametrize("n_support", [0, 36])
@pytest.mark.parametrize("shape", [(1, 8, 50), (3, 21, 137), (2, 1, 40)])
def test_finish_tracks_bitwise_equals_torch(shape, n_support, backward):
    from cotracker_b200 import engine
    B, T, N = shape
    g = torch.Generator().manual_seed(B * 1000 + T * 10 + N)
    thr = 0.9
    t32 = float(torch.tensor(thr, dtype=torch.float32))

    def pair():
        tr = (torch.rand(B, T, N, 2, generator=g) * 600 - 50).to(DEV)
        vi = torch.rand(B, T, N, generator=g)
        pick = torch.rand(B, T, N, generator=g)
        vi[pick < 0.2] = t32                                                    # exactly at the threshold: not visible
        vi[(pick >= 0.2) & (pick < 0.3)] = float(torch.nextafter(torch.tensor(t32), torch.tensor(2.0)))
        return tr, vi.to(DEV)

    fwd, bwd = pair(), (pair() if backward else None)
    queries = torch.cat([torch.randint(0, T, (B, N, 1), generator=g).float(),
                         torch.rand(B, N, 2, generator=g) * 500], dim=2).to(DEV)
    scale = ((1280 - 1) / (512 - 1), (720 - 1) / (384 - 1))
    want = _finish_torch(queries, fwd, bwd, n_support, thr, scale)
    got = engine.finish_tracks(fwd, bwd, queries, N - n_support, thr, scale)
    assert got[0].dtype == torch.float32 and got[1].dtype == torch.bool
    assert got[0].shape == want[0].shape and got[1].shape == want[1].shape
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    if T > 1:                                   # with one frame every point is its own, visible, query point
        assert int(got[1].sum()) not in (0, got[1].numel())
