"""Host tests of clips of different lengths in one pass: the list call's argument checks, the pass planner, the frame
map of a padded pass, the ct3_loop_shape mirror with its group_T field and the library's checks of it."""
import ctypes

import pytest
import torch

from cotracker_b200 import engine
from cotracker_b200.evaluation import pass_bytes, plan_ragged_passes
from cotracker_b200.model import ragged_frame_map
from cotracker_b200.predictor import _check_list_call

EINVAL = -1


class _Offline:
    pass


class _Online:
    def init_video_online_processing(self):
        pass


def _clip(T, h=32, w=48):
    return torch.zeros(1, T, 3, h, w, dtype=torch.uint8)


def _q(*frames):
    return torch.tensor([[[float(t), 1.0, 2.0] for t in frames]])


@pytest.mark.parametrize("kw,msg", [
    (dict(clips=[_clip(4), _clip(5)], queries=[_q(0)]), "queries must be a list of 2"),
    (dict(clips=[_clip(4), _clip(5)], grid_size=3, segm_mask=[None]), "segm_mask must be a list of 2"),
    (dict(clips=[_clip(4), torch.zeros(2, 5, 3, 8, 8)], grid_size=3), "clip 1 must be a [1,T,3,H,W]"),
    (dict(clips=[torch.zeros(5, 3, 8, 8)], grid_size=3), "clip 0 must be a [1,T,3,H,W]"),
    (dict(clips=[_clip(4), _clip(5)], queries=[_q(3), _q(0, 5)]), "clip 1: a query frame lies outside its 5"),
    (dict(clips=[_clip(4)], queries=[_q(-1)]), "clip 0: a query frame lies outside its 4"),
    (dict(clips=[_clip(4), _clip(5)], grid_size=3, grid_query_frame=4), "clip 0: grid_query_frame 4"),
    (dict(clips=[_clip(4), _clip(5)]), "grid_size > 0"),
    (dict(clips=[_clip(4), _clip(5)], queries=[_q(0), None]), "grid_size > 0"),
    (dict(clips=[], grid_size=3), "empty"),
    (dict(clips=[_clip(4)], grid_size=3, model=_Online()), "offline model"),
])
def test_list_call_rejections(kw, msg):
    args = dict(model=_Offline(), queries=None, segm_mask=None, grid_size=0, grid_query_frame=0)
    args.update(kw)
    with pytest.raises(ValueError, match=msg.replace("[", r"\[").replace("]", r"\]")):
        _check_list_call(args["model"], args["clips"], args["queries"], args["segm_mask"], args["grid_size"],
                         args["grid_query_frame"])


def test_list_call_accepts_valid_arguments():
    _check_list_call(_Offline(), [_clip(4), _clip(9)], [_q(3), None], [None, None], 4, 0)
    _check_list_call(_Offline(), [_clip(4), _clip(9)], [_q(3), _q(0, 8)], None, 0, 0)


def test_predictor_forwards_a_list_to_the_list_call():
    from cotracker_b200.predictor import CoTrackerPredictor
    p = CoTrackerPredictor(checkpoint=None, offline=False, window_len=16)
    with pytest.raises(ValueError, match="offline model"):
        p([_clip(4)], grid_size=3)


# ---- planner ------------------------------------------------------------------------------------------------------
BIG = 1 << 50


def test_planner_one_pass_when_everything_fits():
    assert plan_ragged_passes([40, 40, 40], [10, 10, 10], [1, 1, 1], 96, 128, BIG, 0.5, 120) == [[0, 1, 2]]


def test_planner_sorts_by_length_and_every_clip_appears_once():
    lengths = [30, 10, 20, 10, 25]
    passes = plan_ragged_passes(lengths, [5] * 5, [2] * 5, 96, 128, BIG, 1.0, sum(lengths))
    flat = [b for p in passes for b in p]
    assert sorted(flat) == list(range(5))
    assert [lengths[b] for b in flat] == sorted(lengths)
    assert flat == [1, 3, 2, 4, 0]   # ties keep input order


@pytest.mark.parametrize("frac", [0.0, 0.1, 0.5, 2.0])
def test_planner_respects_the_padding_bound(frac):
    lengths = [16, 20, 24, 33, 40, 48, 64, 64, 17]
    tracks = [100, 7, 30, 50, 5, 80, 10, 20, 1]
    passes = plan_ragged_passes(lengths, tracks, [1] * 9, 96, 128, BIG, frac, sum(lengths))
    for p in passes:
        if len(p) == 1:
            continue
        T = max(lengths[b] for b in p)
        real = sum((tracks[b] + 64) * lengths[b] for b in p)   # virtual tracks are padded too
        assert sum(tracks[b] + 64 for b in p) * T - real <= frac * real
    if frac == 0.0:   # only equal lengths share a pass
        assert all(len({lengths[b] for b in p}) == 1 for p in passes)


def test_planner_absolute_padding_rows():
    """pad_rows admits a fixed number of padded token rows per pass on top of the fraction."""
    lengths, tracks = [10, 12, 20], [36, 36, 36]   # 100 token rows per frame each (36 points + 64 virtual)
    assert plan_ragged_passes(lengths, tracks, [1] * 3, 96, 128, BIG, 0.0, 42) == [[0], [1], [2]]
    assert plan_ragged_passes(lengths, tracks, [1] * 3, 96, 128, BIG, 0.0, 42, pad_rows=200) == [[0, 1], [2]]
    assert plan_ragged_passes(lengths, tracks, [1] * 3, 96, 128, BIG, 0.0, 42, pad_rows=1800) == [[0, 1, 2]]
    assert plan_ragged_passes(lengths, tracks, [1] * 3, 96, 128, BIG, 0.0, 42, pad_rows=1799) == [[0, 1], [2]]


def test_planner_respects_the_budget():
    lengths, tracks, groups = [20, 24, 30, 30, 31], [400, 300, 200, 500, 100], [2] * 5
    one = pass_bytes(31, sum(tracks), 10, 96, 128, 135, ragged=True)
    budget = one // 2
    passes = plan_ragged_passes(lengths, tracks, groups, 96, 128, budget, 10.0, 135)
    assert len(passes) > 1
    for p in passes:
        T = max(lengths[b] for b in p)
        if len(p) > 1:
            assert pass_bytes(T, sum(tracks[b] for b in p), 2 * len(p), 96, 128, 135, ragged=True) <= budget
    assert plan_ragged_passes(lengths, tracks, groups, 96, 128, 1, 10.0, 135) == [[b] for b in [0, 1, 2, 3, 4]]


def test_planner_rejects_mismatched_lists():
    with pytest.raises(ValueError):
        plan_ragged_passes([1, 2], [3], [1, 1], 96, 128, BIG, 0.5, 3)


# ---- frame maps ---------------------------------------------------------------------------------------------------
def test_ragged_frame_map_offsets_reversal_and_clamped_padding():
    fm = ragged_frame_map(5, [(0, 3, False), (0, 3, True), (3, 5, False), (8, 1, True), (9, 2, True)])
    assert fm == [[0, 1, 2, 2, 2],
                  [2, 1, 0, 0, 0],
                  [3, 4, 5, 6, 7],
                  [8, 8, 8, 8, 8],
                  [10, 9, 9, 9, 9]]


# ---- ABI ----------------------------------------------------------------------------------------------------------
def test_loop_shape_mirror_matches_the_header():
    names = [f[0] for f in engine.LoopShape._fields_]
    assert names == ["T", "N", "H4", "W4", "G", "group_sizes", "T_pyr", "group_frames", "slab_tracks", "group_T"]
    assert engine.LoopShape.group_T.offset == 56 and ctypes.sizeof(engine.LoopShape) == 64
    assert engine.lib().ct3_version() == 102


def _shape(T, N, G, lengths, sizes=None):
    arr = (ctypes.c_int32 * G)(*lengths)
    sz = None if sizes is None else (ctypes.c_int32 * G)(*sizes)
    return engine.LoopShape(T, N, 24, 32, G, sz, 0, None, 0, arr), arr, sz


@pytest.mark.parametrize("lengths", [[0, 8], [8, 9], [-1, 3], [3, 1 << 20]])
def test_workspace_bytes_rejects_group_lengths_outside_1_T(lengths):
    shape, *_ = _shape(8, 4, 2, lengths)
    n = ctypes.c_size_t(0)
    assert engine.lib().ct3_workspace_bytes(ctypes.byref(shape), ctypes.byref(n)) == EINVAL
    assert b"group_T" in engine.lib().ct3_last_error()


@pytest.mark.parametrize("group_T", [[8], [8, 8, 8], []])
def test_workspace_bytes_rejects_a_group_T_of_another_length(group_T):
    with pytest.raises(engine.EngineError, match="group_T has"):
        engine.workspace_bytes(8, 4, 24, 32, groups=2, group_T=group_T)


def test_workspace_bytes_sizes_group_lengths():
    plain = engine.workspace_bytes(8, 4, 24, 32, groups=2)
    ragged = engine.workspace_bytes(8, 4, 24, 32, groups=2, group_T=[3, 8])
    assert ragged > plain
    assert engine.workspace_bytes(8, 4, 24, 32, groups=2, group_T=[1, 1]) == ragged   # sized by T, not the lengths
    assert engine.workspace_bytes(8, 4, 24, 32, groups=1, group_T=[8]) > engine.workspace_bytes(8, 4, 24, 32)


@pytest.mark.parametrize("lengths", [[0, 8], [8, 9]])
def test_update_loop_rejects_group_lengths_outside_1_T(lengths):
    """Before anything is enqueued: every pointer is fake."""
    lib = engine.lib()
    fake = ctypes.c_void_p(1 << 20)
    ws = ctypes.c_void_p(1 << 24)
    shape, *_ = _shape(8, 4, 2, lengths, [2, 2])
    rc = lib.ct3_update_loop(fake, fake, fake, None, fake, fake, fake, fake, 1, ctypes.byref(shape), ws, 1 << 40, None)
    assert rc == EINVAL
    assert b"group_T" in lib.ct3_last_error()
