"""CPU tests of grouped calls (ct3_update_loop_groups / ct3_updateformer_groups): exported symbols, argument
validation before any launch, and the single-point evaluation pass planner."""
import ctypes

import pytest

from cotracker_b200 import engine
from cotracker_b200.evaluation import pass_bytes, plan_passes

GROUP_SYMBOLS = ("ct3_workspace_bytes_groups", "ct3_update_loop_groups", "ct3_updateformer_groups")


def _sizes(*v):
    return (ctypes.c_int32 * max(1, len(v)))(*v)


def test_group_symbols_exported():
    lib = engine.lib()
    for name in GROUP_SYMBOLS:
        assert hasattr(lib, name) and name in engine.EXPORTED_SYMBOLS, name


def test_workspace_bytes_groups():
    lib = engine.lib()
    n = ctypes.c_size_t(0)
    assert lib.ct3_workspace_bytes_groups(16, 500, 1, 96, 128, ctypes.byref(n)) == 0
    assert n.value == engine.workspace_bytes(16, 500, 96, 128)          # G = 1 is the plain call
    one = engine.workspace_bytes(16, 500, 96, 128, groups=1)
    five = engine.workspace_bytes(16, 500, 96, 128, groups=5)
    assert five > one + 4 * 64 * 16 * 384 * 4                           # 64 virtual token rows per frame per group
    assert lib.ct3_workspace_bytes_groups(16, 500, 0, 0, 0, ctypes.byref(n)) == -1       # G < 1
    assert lib.ct3_workspace_bytes_groups(16, 3, 4, 0, 0, ctypes.byref(n)) == -1         # more groups than tracks
    with pytest.raises(engine.EngineError):
        engine.workspace_bytes(4, 10, groups=0)


def test_grouped_calls_reject_bad_groups_without_gpu():
    """Every invalid group argument returns CT3_EINVAL before anything is enqueued (all pointers are fake and the
    stream is the legacy default: reaching a launch would fail differently)."""
    lib = engine.lib()
    fake = ctypes.c_void_p(1 << 20)
    ws = ctypes.c_void_p(1 << 24)

    def loop(sizes, G, N=10):
        return lib.ct3_update_loop_groups(fake, fake, 24, 32, fake, None, fake, fake, fake, fake, 4, N, 1, ws, 1 << 40,
                                          None, sizes, G)

    def former(sizes, G):
        return lib.ct3_updateformer_groups(fake, fake, 4, sizes, G, fake, ws, 1 << 40, None)

    cases = [
        (None, 2, b"null group"),             # null group array
        (_sizes(5, 5), 0, b"G must be"),       # G < 1
        (_sizes(5, 5), -3, b"G must be"),
        (_sizes(10, 0), 2, b"size must be"),   # a size < 1
        (_sizes(11, -1), 2, b"size must be"),
        (_sizes(4, 5), 2, b"sum to N"),        # sum != N
        (_sizes(6, 5), 2, b"sum to N"),
    ]
    for sizes, G, msg in cases:
        assert loop(sizes, G) == -1, (G, msg)
        assert msg in lib.ct3_last_error(), (lib.ct3_last_error(), msg)
    for sizes, G, msg in cases[:5]:
        assert former(sizes, G) == -1, (G, msg)
        assert msg in lib.ct3_last_error()
    # the Python wrappers raise EngineError for the same arguments
    with pytest.raises(engine.EngineError):
        engine._group_array(["x"])


def _check_plan(sizes, T, budget, fn):
    passes = plan_passes(sizes, T, 96, 128, budget, fn)
    covered = [g for a, b in passes for g in range(a, b)]
    assert covered == list(range(len(sizes)))                           # every group once, in order
    assert all(b > a for a, b in passes)
    for a, b in passes:
        if b - a > 1:
            assert fn(T, sum(sizes[a:b]), b - a, 96, 128) <= budget         # multi-group passes fit the budget
        if b < len(sizes):                                               # greedy: the next group would not have fit
            assert fn(T, sum(sizes[a:b + 1]), b + 1 - a, 96, 128) > budget
    return passes


def test_pass_planner_covers_groups_in_order_within_budget():
    fn = lambda T, N, G, H4, W4: 1000 * N * T + 7 * G   # noqa: E731
    sizes = [90, 1, 129, 300, 64, 255, 90, 90]
    total = fn(16, sum(sizes), len(sizes), 96, 128)
    assert _check_plan(sizes, 16, total, fn) == [(0, len(sizes))]
    assert len(_check_plan(sizes, 16, total // 2, fn)) >= 2
    assert _check_plan(sizes, 16, 1, fn) == [(g, g + 1) for g in range(len(sizes))]   # one group per pass
    for budget in range(1, total + 1, total // 37):
        _check_plan(sizes, 16, budget, fn)
    assert plan_passes([], 16, 96, 128, 1 << 30, fn) == []


def test_pass_planner_with_library_sizes():
    sizes = [90] * 30
    one = pass_bytes(50, 90, 1, 96, 128)
    every = pass_bytes(50, 90 * 30, 30, 96, 128)
    assert every > 5 * one
    for budget in (one, 3 * one, every // 2, every):
        _check_plan(sizes, 50, budget, pass_bytes)
    assert plan_passes(sizes, 50, 96, 128, every) == [(0, 30)]
