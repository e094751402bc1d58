"""CPU tests of the track-slabbed update loop (ct3_loop_shape.slab_tracks, DESIGN.md §4.4.5): argument checks, workspace
sizes and the size limit of the C ABI, and when the model chooses slabs."""
import ctypes

import pytest
import torch

from cotracker_b200 import engine

EINVAL, ENOSPC = -1, -3


def _i32(*v):
    return (ctypes.c_int32 * max(1, len(v)))(*v)


def _ws(T, T_pyr, N, G, H4, W4, slab, out=True):
    """ct3_workspace_bytes of a shape without arrays (T_pyr 0: no frame map, slab 0: no slabs) -> (rc, bytes)"""
    n = ctypes.c_size_t(0)
    shape = engine._loop_shape(T, N, H4, W4, G, None, T_pyr, None, slab)
    rc = engine.lib().ct3_workspace_bytes(ctypes.byref(shape), ctypes.byref(n) if out else None)
    return rc, n.value


def _frames(T, T_pyr, N, G, H4, W4):
    rc, n = _ws(T, T_pyr, N, G, H4, W4, 0)
    assert rc == 0
    return n


@pytest.mark.parametrize("T,T_pyr,N,G,H4,W4", [(16, 16, 6400, 1, 96, 128), (4, 8, 10, 2, 24, 32),
                                               (60, 60, 300, 3, 96, 128), (1, 1, 1, 1, 24, 32),
                                               (160, 200, 129, 1, 96, 128)])
@pytest.mark.parametrize("frame_map", [True, False])
def test_slabbed_workspace_at_N_is_the_unslabbed_workspace_and_never_shrinks(T, T_pyr, N, G, H4, W4, frame_map):
    """slab_tracks >= N is the same shape with slab_tracks = 0, with a frame map (T_pyr frames) and without one (T
    frames)."""
    tp = T_pyr if frame_map else 0
    full = _frames(T, tp, N, G, H4, W4)
    for slab in (N, N + 1, 10 * N):
        assert _ws(T, tp, N, G, H4, W4, slab) == (0, full)
    slabs = sorted({1, 2, 7, 64, 129, N // 3, N // 2, N - 1, N} & set(range(1, N + 1)))
    sizes = [_ws(T, tp, N, G, H4, W4, s)[1] for s in slabs]
    assert all(a <= b for a, b in zip(sizes, sizes[1:])), list(zip(slabs, sizes))
    assert sizes[-1] == full
    assert engine.workspace_bytes(T, N, H4, W4, G, tp or None, slab_tracks=slabs[0]) == sizes[0]
    if T_pyr == T:   # the map's only cost: its [G, T] int32 table, in a 1024-byte aligned block
        for s in (1, N):
            assert _ws(T, T, N, G, H4, W4, s)[1] - _ws(T, 0, N, G, H4, W4, s)[1] == -(-G * T * 4 // 1024) * 1024


@pytest.mark.parametrize("G", [1, 4])
def test_full_size_workspace_per_point_row_with_one_track_slabs(G):
    """What grows with the point rows at slab_tracks = 1: the fp32 token (1536 B) and the point side of the space
    attentions (3072 B), against 65,024 B without slabs."""
    T, H4, W4 = 48, 96, 128
    n1, n2 = 4000, 6400
    per_row = (_ws(T, T, n2, G, H4, W4, 1)[1] - _ws(T, T, n1, G, H4, W4, 1)[1]) / ((n2 - n1) * T)
    full = (_frames(T, T, n2, G, H4, W4) - _frames(T, T, n1, G, H4, W4)) / ((n2 - n1) * T)
    assert per_row <= 8192
    # G > 1 adds the virtual<-point split-K partials, which grow with the tracks in both workspaces alike
    assert abs(per_row - 4608 - (full - 65024)) < 1, (per_row, full)
    assert G > 1 or (per_row, full) == (4608, 65024)


def test_slabbed_size_limit_of_the_loop_shape():
    """(N + 64 G) * T <= 2^21 token rows; larger problems return CT3_EINVAL, as do slab_tracks < 1."""
    lib = engine.lib()
    assert _ws(300, 300, 6400, 1, 128, 128, 1000)[0] == 0                   # grid 80 x 300 frames fits
    assert _ws(1, 1, (1 << 21) - 64, 1, 24, 32, 7)[0] == 0                  # exactly 2^21 rows
    assert _ws(1, 1, (1 << 21) - 63, 1, 24, 32, 7)[0] == EINVAL
    assert b"2^21" in lib.ct3_last_error()
    assert _ws(400, 400, 6400, 1, 128, 128, 6400)[0] == EINVAL              # also with slab_tracks >= N
    assert _ws(16, 16, 100, 1, 96, 128, -1)[0] == EINVAL
    assert _ws(16, 16, 100, 1, 96, 128, -3)[0] == EINVAL
    assert b"slab_tracks" in lib.ct3_last_error()
    assert _ws(16, 16, 100, 1, 96, 128, 8, out=False)[0] == EINVAL
    assert _ws(0, 16, 100, 1, 96, 128, 8)[0] == EINVAL                      # the frame-map checks still apply
    assert _ws(16, -1, 100, 1, 96, 128, 8)[0] == EINVAL
    assert _ws(16, 16, 100, 0, 96, 128, 8)[0] == EINVAL
    assert _ws(16, 16, 100, 1, 2, 2, 8)[0] == EINVAL                        # pyramid too small
    assert _ws(16, 0, 100, 1, 0, 0, 8)[0] == EINVAL                         # slabs need the pyramid
    with pytest.raises(engine.EngineError):
        engine.workspace_bytes(16, 100, 96, 128, slab_tracks=-1)
    assert _ws(1, 0, 1 << 21, 1, 24, 32, 0)[0] == 0                         # the limit is the slabbed loop's only


def test_update_loop_rejects_bad_slab_shapes_without_gpu():
    """Every invalid argument returns CT3_EINVAL / CT3_ENOSPC before anything is enqueued (all pointers are fake and
    the stream is the legacy default: reaching a launch would fail differently)."""
    lib = engine.lib()
    fake = ctypes.c_void_p(1 << 20)
    ws = ctypes.c_void_p(1 << 24)
    T = 4

    def loop(frames=None, T_pyr=0, sizes=_i32(5, 5), G=2, N=10, slab=3, nbytes=1 << 40, iters=1, workspace=ws,
             shape=True):
        sh = engine._loop_shape(T, N, 24, 32, G, sizes, T_pyr, frames, slab)
        return lib.ct3_update_loop(fake, fake, fake, None, fake, fake, fake, fake, iters,
                                   ctypes.byref(sh) if shape else None, workspace, nbytes, None)

    good = _i32(0, 1, 2, 3, 7, 6, 5, 4)
    cases = [
        (dict(shape=False), b"null shape"),
        (dict(slab=-1), b"slab_tracks"),
        (dict(T_pyr=8), b"null group_frames"),                             # T_pyr >= 1 needs a map
        (dict(frames=_i32(0, 1, 2, 8, 7, 6, 5, 4), T_pyr=8), b"outside"),
        (dict(frames=good, T_pyr=0), b"T_pyr"),
        (dict(sizes=_i32(4, 5)), b"sum to N"),
        (dict(sizes=None), b"null group_sizes"),
        (dict(iters=-1), b"iters"),
        (dict(N=(1 << 19), sizes=_i32(1 << 19), G=1), b"2^21"),
        (dict(workspace=None), b"null argument"),
        (dict(workspace=ctypes.c_void_p((1 << 24) + 8)), b"aligned"),
    ]
    for kw, msg in cases:
        assert loop(**kw) == EINVAL, (kw, msg)
        assert msg in lib.ct3_last_error(), (kw, lib.ct3_last_error())
    need = _ws(T, 0, 10, 2, 24, 32, 3)[1]
    assert loop(nbytes=need - 1) == ENOSPC
    assert loop(frames=good, T_pyr=8, nbytes=_ws(T, 8, 10, 2, 24, 32, 3)[1] - 1) == ENOSPC


# ---- when the model runs in slabs ------------------------------------------------------------------------------
def _refine_slab(monkeypatch, budget, T=24, N=500, G=2, H4=24, W4=32, frames=None):
    """slab_tracks of the update loop _refine runs under a patched pass budget (the library call itself is caught)."""
    import cotracker_b200.model as M
    model = M.CoTrackerThreeOffline(stride=4, corr_radius=3, window_len=60)
    seen = {}
    monkeypatch.setattr(M, "pass_budget_bytes", lambda *a, **k: budget)
    monkeypatch.setattr(M.engine, "update_loop", lambda *a, **k: seen.update(k))

    class Cache:
        def get(self, *a):
            seen["ws_args"] = a
            return None

    model._ws = Cache()
    monkeypatch.setattr(model, "packed_weights", lambda dev: None)
    T_pyr = T if frames is None else frames
    pyr = torch.empty(engine.pyramid_layout(T_pyr, H4, W4)[3])
    coords = torch.zeros(T, N, 2)
    gf = None if frames is None else [[t % frames for t in range(T)]] * G
    sizes = [N // G] * (G - 1) + [N - (N // G) * (G - 1)]
    model._refine(pyr, H4, W4, None, None, coords, None, None, 4, sizes, gf)
    return seen


@pytest.mark.parametrize("frames", [None, 30])
def test_refine_slabs_only_when_the_full_workspace_exceeds_the_budget(monkeypatch, frames):
    T, N, G, H4, W4 = 24, 500, 2, 24, 32
    full = engine.workspace_bytes(T, N, H4, W4, G, frames)
    for budget in (full, full + 1, 1 << 50):                                 # fits: the call of today
        seen = _refine_slab(monkeypatch, budget, T, N, G, H4, W4, frames)
        assert seen["slab_tracks"] is None
        assert seen["group_sizes"] == [250, 250] and seen["ws_args"][-1] is None
    for budget in (full - 1, full // 2, full // 4):
        seen = _refine_slab(monkeypatch, budget, T, N, G, H4, W4, frames)
        s = seen["slab_tracks"]
        assert 1 <= s < N
        assert engine.workspace_bytes(T, N, H4, W4, G, frames, slab_tracks=s) <= budget
        assert s == N - 1 or engine.workspace_bytes(T, N, H4, W4, G, frames, slab_tracks=s + 1) > budget
        assert seen["ws_args"][-1] == s and seen["group_frames"] == (None if frames is None else seen["group_frames"])
    assert _refine_slab(monkeypatch, 1, T, N, G, H4, W4, frames)["slab_tracks"] == 1   # nothing fits: smallest slab


def test_planner_splits_are_unchanged_and_oversized_passes_get_slabs():
    """The planners keep their splits; a pass that exceeds the budget on its own gets the largest slab that fits."""
    from cotracker_b200.evaluation import pass_bytes, plan_passes, slab_tracks_for
    T, H4, W4 = 40, 96, 128
    sizes = [90] * 4 + [3000]
    budget = pass_bytes(T, 360, 4, H4, W4)
    passes = plan_passes(sizes, T, H4, W4, budget)
    assert passes == [(0, 4), (4, 5)]
    assert slab_tracks_for(T, 360, 4, H4, W4, None, budget) is None
    s = slab_tracks_for(T, 3000, 1, H4, W4, None, budget)
    assert s is not None and 1 <= s < 3000
    assert engine.workspace_bytes(T, 3000, H4, W4, 1, slab_tracks=s) <= budget
