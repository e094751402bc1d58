"""CPU tests of frame maps (ct3_loop_shape.T_pyr, group_frames): exported symbols, argument validation before any
launch, the host frame-map builders of both models against a brute-force restatement of the padded / reversed clip,
the window gather, and the dense-mode pass planner."""
import ctypes

import numpy as np
import pytest
import torch

from cotracker_b200 import engine
from cotracker_b200.build import build_cotracker
from cotracker_b200.evaluation import pass_bytes, plan_dense_passes, plan_passes
from cotracker_b200.model import clip_frame_map, gather_plan, gather_pyramid, window_frame_map

FRAME_SYMBOLS = ("ct3_workspace_bytes", "ct3_update_loop")


def _i32(*v):
    return (ctypes.c_int32 * max(1, len(v)))(*v)


def test_frame_map_is_a_loop_shape_field():
    """A frame map is a field of the loop shape: the size and loop entry points take it."""
    lib = engine.lib()
    for name in FRAME_SYMBOLS:
        assert hasattr(lib, name) and name in engine.EXPORTED_SYMBOLS, name


def _ws(T, T_pyr, N, G, H4, W4, frames=None):
    n = ctypes.c_size_t(0)
    shape = engine._loop_shape(T, N, H4, W4, G, None, T_pyr, frames)
    return engine.lib().ct3_workspace_bytes(ctypes.byref(shape), ctypes.byref(n)), n.value


def test_workspace_bytes_with_frame_map():
    lib = engine.lib()
    rc, n = _ws(16, 32, 500, 2, 96, 128)
    assert rc == 0 and n == engine.workspace_bytes(16, 500, 96, 128, groups=2, frames=32)
    same = engine.workspace_bytes(16, 500, 96, 128, groups=2, frames=16)
    assert same >= engine.workspace_bytes(16, 500, 96, 128, groups=2)             # + the [G, T] frame map
    *_, per_frame = engine.pyramid_layout(1, 96, 128)
    assert n - same >= 16 * per_frame * 4 - 4096                                  # split pyramid copy sized by T_pyr
    assert _ws(16, -1, 500, 2, 96, 128)[0] == -1 and b"T_pyr" in lib.ct3_last_error()     # T_pyr < 0
    assert _ws(16, 16, 500, 0, 96, 128)[0] == -1                                          # G < 1
    with pytest.raises(engine.EngineError):
        engine.workspace_bytes(4, 10, 24, 32, frames=-1)
    # the size needs no map; one that is given is checked and changes nothing
    good = _i32(*(list(range(16)) + list(range(31, 15, -1))))
    assert _ws(16, 32, 500, 2, 96, 128, good) == (0, n)
    assert _ws(16, 0, 500, 2, 96, 128, good)[0] == -1 and b"T_pyr" in lib.ct3_last_error()   # a map needs T_pyr
    assert _ws(16, 31, 500, 2, 96, 128, good)[0] == -1 and b"outside" in lib.ct3_last_error()


def test_update_loop_rejects_bad_frame_maps_without_gpu():
    """Every invalid frame-map argument returns CT3_EINVAL before anything is enqueued (all pointers are fake and the
    stream is the legacy default: reaching a launch would fail differently)."""
    lib = engine.lib()
    fake = ctypes.c_void_p(1 << 20)
    ws = ctypes.c_void_p(1 << 24)
    T = 4

    def loop(frames, T_pyr=8, sizes=_i32(5, 5), G=2, N=10):
        shape = engine._loop_shape(T, N, 24, 32, G, sizes, T_pyr, frames)
        return lib.ct3_update_loop(fake, fake, fake, None, fake, fake, fake, fake, 1, ctypes.byref(shape), ws, 1 << 40,
                                   None)

    good = _i32(*([0, 1, 2, 3] + [7, 6, 5, 4]))
    cases = [
        (None, 8, _i32(5, 5), 2, b"null group_frames"),                    # null table, G > 1
        (None, 8, _i32(10), 1, b"null group_frames"),                      # null table, G = 1
        (_i32(0, 1, 2, 8, 7, 6, 5, 4), 8, _i32(5, 5), 2, b"outside"),      # index == T_pyr
        (_i32(0, 1, 2, 3, 7, 6, -1, 4), 8, _i32(5, 5), 2, b"outside"),     # negative index
        (_i32(0, 1, 2, 3), 3, _i32(10), 1, b"outside"),                    # index >= a smaller T_pyr
        (good, 0, _i32(5, 5), 2, b"T_pyr"),                                # a map with T_pyr = 0
        (good, -5, _i32(5, 5), 2, b"T_pyr"),                               # T_pyr < 0
        (None, -5, _i32(5, 5), 2, b"T_pyr"),
        (good, 8, _i32(4, 5), 2, b"sum to N"),                             # the group checks still apply
    ]
    for frames, T_pyr, sizes, G, msg in cases:
        assert loop(frames, T_pyr, sizes, G) == -1, (T_pyr, G, msg)
        assert msg in lib.ct3_last_error(), lib.ct3_last_error()


# ---- host frame-map builders --------------------------------------------------------------------------------
def _padded_clip(T, pad, reverse):
    """Frame ids of the clip the reference's model encodes: played backwards if `reverse` (video.flip(1)), then padded
    with `pad` copies of its last frame."""
    ids = np.arange(T)[::-1] if reverse else np.arange(T)
    return np.concatenate([ids, np.full(pad, ids[-1])])


@pytest.mark.parametrize("T", [1, 2, 7, 12, 50])
def test_clip_frame_map(T):
    flags = [False, True, True, False]
    fm = clip_frame_map(T, flags)
    assert len(fm) == 4
    for row, r in zip(fm, flags):
        assert row == _padded_clip(T, 0, r).tolist()


@pytest.mark.parametrize("T,S", [(16, 16), (37, 16), (16, 8), (23, 8), (5, 8), (60, 16), (9, 4)])
def test_window_frame_map_matches_padded_flipped_clip(T, S):
    """window_frame_map against _clip_pad + flip + slice_pyramid restated on frame ids; gather_plan's runs, and the
    remapped table, address exactly the referenced frames."""
    model = build_cotracker(None, offline=False, window_len=S)
    pad = model._clip_pad(T)
    assert (T + pad) % S == 0
    step = S // 2
    num_windows = (T - S + step - 1) // step + 1
    flags = [True, False, True]
    forward = _padded_clip(T, pad, False)      # what frame j of the model's (forward, padded) pyramid holds
    for ind in range(0, step * num_windows, step):
        fm = window_frame_map(T, S, ind, flags)
        for row, r in zip(fm, flags):
            assert all(0 <= f < T + pad for f in row)
            # the reversed clip's frame j is forward frame T-1-j; its padding copies forward frame 0
            want = _padded_clip(T, pad, r)[ind:ind + S]
            assert forward[row].tolist() == want.tolist(), (ind, r)
        runs, local = gather_plan(fm)
        gathered = np.concatenate([np.arange(a, b) for a, b in runs])
        assert len(gathered) <= 2 * S and len(set(gathered.tolist())) == len(gathered)
        assert all(b0 < a1 for (_, b0), (a1, _) in zip(runs, runs[1:]))      # sorted, disjoint, not adjacent
        for row, lrow in zip(fm, local):
            assert gathered[lrow].tolist() == row
    # forward groups only: the window's own S frames, identity map
    runs, local = gather_plan(window_frame_map(T, S, 0, [False, False]))
    assert runs == [(0, S)] and local == [list(range(S))] * 2


def test_gather_pyramid_copies_the_referenced_frames():
    """gather_pyramid (concat_pyramid_runs) on a host pyramid whose every value is its frame id."""
    T, H4, W4 = 24, 16, 20
    off, h, w, total = engine.pyramid_layout(T, H4, W4)
    pyr = torch.empty(total)
    for lv in range(4):
        n = h[lv] * w[lv] * 128
        pyr[off[lv]:off[lv] + T * n] = torch.arange(T, dtype=torch.float32).repeat_interleave(n) + 100 * lv
    fm = window_frame_map(21, 8, 12, [False, True])     # T = 21 -> padded to 24
    runs, local = gather_plan(fm)
    out = gather_pyramid(pyr, T, H4, W4, runs)
    Tg = sum(b - a for a, b in runs)
    assert engine.pyramid_frames(out, H4, W4) == Tg
    levels = engine.pyramid_levels(out, Tg, H4, W4)
    for row, lrow in zip(fm, local):
        for f, lf in zip(row, lrow):
            for lv in range(4):
                assert bool((levels[lv][lf] == f + 100 * lv).all())


def test_pyramid_frames():
    *_, total = engine.pyramid_layout(7, 24, 32)
    assert engine.pyramid_frames(torch.empty(total), 24, 32) == 7
    with pytest.raises(engine.EngineError):
        engine.pyramid_frames(torch.empty(total + 1), 24, 32)


# ---- dense pass planner ----------------------------------------------------------------------------------
@pytest.mark.parametrize("backward", [False, True])
@pytest.mark.parametrize("budget_mib", [1, 300, 2000, 1 << 20])
def test_dense_planner_is_plan_passes(backward, budget_mib):
    T, H4, W4, n, n_off = 8, 40, 56, 2800, 4
    frames = T if backward else None
    sizes, passes = plan_dense_passes(n_off, n, backward, T, H4, W4, budget_mib << 20, frames)
    assert sizes == [n] * (n_off * (2 if backward else 1))
    want = plan_passes(sizes, T, H4, W4, budget_mib << 20,
                       lambda T_, N, G, a, b: pass_bytes(T_, N, G, a, b, frames))
    assert passes == want
    assert passes[0][0] == 0 and passes[-1][1] == len(sizes)
    assert all(p[1] == q[0] for p, q in zip(passes, passes[1:]))
    if budget_mib == 1:
        assert passes == [(g, g + 1) for g in range(len(sizes))]       # every group alone
    if budget_mib == 1 << 20:
        assert passes == [(0, len(sizes))]
