"""CPU tests of batched tracking (B > 1 clips in one call): the frame maps that make clip b a set of query groups
reading its own frames of one shared pyramid, the split of a batch into sub-batches by device memory, the input checks
of the batched entry points, and the ABI of ct3_finish_tracks."""
import ctypes

import pytest
import torch

from cotracker_b200 import engine, evaluation, ingest
from cotracker_b200.model import batch_frame_map, batch_gather_plan, clip_frame_map, gather_plan, window_frame_map

FLAGS = [[False], [False, True], [True, False, True]]


@pytest.mark.parametrize("B", [1, 2, 3])
@pytest.mark.parametrize("flags", FLAGS)
def test_offline_batch_frame_map_is_the_clip_map_plus_clip_offset(B, flags):
    T = 11
    one = clip_frame_map(T, flags)
    got = batch_frame_map(one, range(B), T)
    assert len(got) == B * len(flags)
    for b in range(B):
        for g, row in enumerate(one):
            assert got[b * len(flags) + g] == [f + b * T for f in row]
    assert batch_frame_map(one, [0], T) == one


@pytest.mark.parametrize("B", [1, 2, 3])
@pytest.mark.parametrize("flags", FLAGS)
@pytest.mark.parametrize("T,S", [(27, 16), (16, 16), (9, 8)])
def test_window_batch_gather_plan(B, flags, T, S):
    """Every window of the sliding-window model: group (b, g) reads the one-clip map plus b * T_pad, and the runs
    gathered for clip b lie inside clip b's frames of the pyramid, also where two clips' runs touch (T_pad == S)."""
    step = S // 2
    T_pad = T + (S - T % S) % S
    clips = list(range(B))
    for ind in range(0, step * ((T - S + step - 1) // step + 1), step):
        one = window_frame_map(T, S, ind, flags)
        runs1, remap1 = gather_plan(one)
        runs, remap = batch_gather_plan(one, clips, T_pad)
        if B == 1:
            assert (runs, remap) == (runs1, remap1)
        assert len(runs) == B * len(runs1) and len(remap) == B * len(flags)
        for i, (a, b) in enumerate(runs):
            c = i // len(runs1)
            assert c * T_pad <= a < b <= (c + 1) * T_pad
        # the gathered pyramid, frame by frame, in terms of the batch pyramid
        gathered = [f for a, b in runs for f in range(a, b)]
        want = batch_frame_map(one, clips, T_pad)
        assert [[gathered[p] for p in row] for row in remap] == want


def test_batch_maps_of_a_sub_batch_use_the_clips_own_offsets():
    one = clip_frame_map(5, [False, True])
    assert batch_frame_map(one, [2, 3], 5) == [[10, 11, 12, 13, 14], [14, 13, 12, 11, 10],
                                               [15, 16, 17, 18, 19], [19, 18, 17, 16, 15]]
    runs, remap = batch_gather_plan(window_frame_map(10, 8, 0, [False]), [1, 3], 16)
    assert runs == [(16, 24), (48, 56)] and remap == [list(range(8)), list(range(8, 16))]


@pytest.mark.parametrize("B", [1, 2, 5, 8])
def test_plan_clip_passes_covers_every_clip_once_within_budget(B):
    sizes, T, H4, W4 = [100, 100], 50, 96, 128
    frames = lambda n: B * T                                                   # noqa: E731
    cost = lambda n: evaluation.pass_bytes(T, n * 200, n * 2, H4, W4, frames(n))  # noqa: E731
    for budget in (1, cost(1), cost(2), cost(3) + 1, cost(B), 1 << 50):
        passes = evaluation.plan_clip_passes(B, sizes, T, H4, W4, budget, frames)
        assert [b for b0, b1 in passes for b in range(b0, b1)] == list(range(B))
        for b0, b1 in passes:
            assert b1 - b0 == 1 or cost(b1 - b0) <= budget
        fit = max([n for n in range(1, B + 1) if cost(n) <= budget], default=1)
        assert len(passes) == -(-B // fit)                                     # as few passes as the budget allows
        assert max(b1 - b0 for b0, b1 in passes) - min(b1 - b0 for b0, b1 in passes) <= 1
    assert evaluation.plan_clip_passes(B, sizes, T, H4, W4, 1 << 50) == [(0, B)]
    assert evaluation.plan_clip_passes(1, sizes, T, H4, W4, 1) == [(0, 1)]     # B = 1: one pass, as before


def test_batched_pass_cost_grows_with_the_clips():
    """What the planner relies on: more clips in a pass never cost less."""
    costs = [evaluation.pass_bytes(16, n * 100, n, 96, 128, n * 16) for n in range(1, 9)]
    assert costs == sorted(costs) and costs[0] < costs[-1]


def test_prepare_video_validates_batches():
    for bad in (torch.zeros(4, 3, 8, 8), torch.zeros(0, 4, 3, 8, 8), torch.zeros(2, 0, 3, 8, 8),
                torch.zeros(2, 4, 1, 8, 8)):
        with pytest.raises(ValueError):
            ingest.prepare_video(bad, (8, 8), "cuda:0")
    with pytest.raises(engine.EngineError):          # a well-formed batch still needs the GPU
        ingest.prepare_video(torch.zeros(2, 4, 3, 8, 8, dtype=torch.uint8), (8, 8), "cpu")
    # a [B,T,H,W,3] decoder batch seen through permute keeps dense frames: uploaded as raw bytes, clip after clip
    v = torch.zeros(2, 4, 8, 8, 3, dtype=torch.uint8).permute(0, 1, 4, 2, 3)
    assert all(ingest.frame_is_dense(v[b].shape[1:], v[b].stride()[1:]) for b in range(2))


def test_models_reject_mismatched_batches():
    from cotracker_b200.build import build_cotracker
    m = build_cotracker(None, offline=True, window_len=8)
    with pytest.raises(ValueError):
        m(torch.zeros(2, 4, 3, 64, 64), torch.zeros(1, 5, 3))
    with pytest.raises(ValueError):
        m._track_frames(torch.zeros(7, 3, 64, 64), torch.zeros(2, 5, 3))
    with pytest.raises(engine.EngineError):          # B = 2 is well-formed; the CPU is not
        m(torch.zeros(2, 4, 3, 64, 64), torch.zeros(2, 5, 3))


def test_segm_mask_needs_one_clip():
    from cotracker_b200.predictor import CoTrackerPredictor
    p = CoTrackerPredictor(checkpoint=None, window_len=8)
    with pytest.raises(ValueError, match="segm_mask"):
        p(torch.zeros(2, 4, 3, 64, 64), grid_size=3, segm_mask=torch.ones(2, 1, 64, 64))


def test_online_predictor_keeps_its_stream_count():
    from cotracker_b200.predictor import CoTrackerOnlinePredictor
    op = CoTrackerOnlinePredictor(checkpoint=None, window_len=4)
    clip = torch.zeros(3, 4, 3, 64, 64, dtype=torch.uint8)
    op(video_chunk=clip, is_first_step=True, grid_size=2)
    assert op.queries.shape == (3, 4, 3)
    op(video_chunk=clip, is_first_step=True, queries=torch.zeros(3, 5, 3), add_support_grid=True)
    assert op.queries.shape == (3, 5 + 36, 3)
    with pytest.raises(ValueError, match="streams"):
        op(video_chunk=clip[:2])


def test_finish_tracks_abi():
    """ct3_finish_tracks is exported and rejects bad arguments with CT3_EINVAL before any launch."""
    assert "ct3_finish_tracks" in engine.EXPORTED_SYMBOLS
    lib = engine.lib()
    p, f = ctypes.c_void_p(256), ctypes.c_float
    ok = dict(B=2, T=5, N=7, n_keep=7)

    def call(fwd_t=p, fwd_v=p, bwd_t=None, bwd_v=None, q=p, out_t=p, out_v=p, **kw):
        a = {**ok, **kw}
        return lib.ct3_finish_tracks(fwd_t, fwd_v, bwd_t, bwd_v, q, a["B"], a["T"], a["N"], a["n_keep"], f(0.9), f(1.0),
                                     f(1.0), out_t, out_v, None)

    for bad in (dict(fwd_t=None), dict(fwd_v=None), dict(q=None), dict(out_t=None), dict(out_v=None)):
        assert call(**bad) == -1 and b"null argument" in lib.ct3_last_error()
    assert call(bwd_t=p) == -1 and b"given together" in lib.ct3_last_error()
    assert call(bwd_v=p) == -1
    for bad in (dict(B=0), dict(T=0), dict(N=0)):
        assert call(**bad) == -1 and b"must be >= 1" in lib.ct3_last_error()
    for bad in (dict(n_keep=0), dict(n_keep=8)):
        assert call(**bad) == -1 and b"n_keep" in lib.ct3_last_error()
    assert call(fwd_t=ctypes.c_void_p(260)) == -1 and b"8-byte aligned" in lib.ct3_last_error()
    assert call(B=1 << 20, T=1 << 20, N=1 << 10) == -1 and b"too large" in lib.ct3_last_error()
    with pytest.raises(engine.EngineError):          # the wrapper takes CUDA tensors only
        engine.finish_tracks((torch.zeros(1, 2, 3, 2), torch.zeros(1, 2, 3)), None, torch.zeros(1, 3, 3), 3, 0.9, (1, 1))
