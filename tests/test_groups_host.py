"""CPU tests of grouped calls (ct3_loop_shape.G / ct3_updateformer's group sizes): exported symbols, argument
validation before any launch, and the single-point evaluation pass planner."""
import ctypes

import pytest

from cotracker_b200 import engine
from cotracker_b200.evaluation import pass_bytes, plan_passes

GROUP_SYMBOLS = ("ct3_workspace_bytes", "ct3_update_loop", "ct3_updateformer")


def _sizes(*v):
    return (ctypes.c_int32 * max(1, len(v)))(*v)


def test_groups_are_a_loop_shape_field():
    """Groups are a field of the loop shape: one entry point each for the size, the loop and the updateformer."""
    lib = engine.lib()
    for name in GROUP_SYMBOLS:
        assert hasattr(lib, name) and name in engine.EXPORTED_SYMBOLS, name


def _ws(T, N, G, H4, W4, sizes=None):
    n = ctypes.c_size_t(0)
    rc = engine.lib().ct3_workspace_bytes(ctypes.byref(engine._loop_shape(T, N, H4, W4, G, sizes)), ctypes.byref(n))
    return rc, n.value


def test_workspace_bytes_with_groups():
    lib = engine.lib()
    assert _ws(16, 500, 1, 96, 128) == (0, engine.workspace_bytes(16, 500, 96, 128))   # G = 1 is the plain call
    one = engine.workspace_bytes(16, 500, 96, 128, groups=1)
    five = engine.workspace_bytes(16, 500, 96, 128, groups=5)
    assert five > one + 4 * 64 * 16 * 384 * 4                           # 64 virtual token rows per frame per group
    assert _ws(16, 500, 0, 0, 0)[0] == -1                               # G < 1
    assert _ws(16, 3, 4, 0, 0)[0] == -1                                 # more groups than tracks
    with pytest.raises(engine.EngineError):
        engine.workspace_bytes(4, 10, groups=0)
    # the size needs no sizes array; one that is given is checked and changes nothing
    assert _ws(16, 500, 2, 96, 128, _sizes(100, 400)) == _ws(16, 500, 2, 96, 128)
    assert _ws(16, 500, 2, 96, 128, _sizes(100, 399))[0] == -1 and b"sum to N" in lib.ct3_last_error()
    assert _ws(16, 500, 2, 96, 128, _sizes(500, 0))[0] == -1 and b"size must be" in lib.ct3_last_error()


def test_loop_and_updateformer_reject_bad_groups_without_gpu():
    """Every invalid group argument returns CT3_EINVAL before anything is enqueued (all pointers are fake and the
    stream is the legacy default: reaching a launch would fail differently)."""
    lib = engine.lib()
    fake = ctypes.c_void_p(1 << 20)
    ws = ctypes.c_void_p(1 << 24)

    def loop(sizes, G, N=10):
        shape = engine._loop_shape(4, N, 24, 32, G, sizes)
        return lib.ct3_update_loop(fake, fake, fake, None, fake, fake, fake, fake, 1, ctypes.byref(shape), ws, 1 << 40,
                                   None)

    def former(sizes, G, N=10):
        return lib.ct3_updateformer(fake, fake, 4, N, sizes, G, fake, ws, 1 << 40, None)

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
    for sizes, G, msg in cases:
        assert former(sizes, G) == -1, (G, msg)
        assert msg in lib.ct3_last_error()
    assert former(_sizes(5, 5), 2, N=0) == -1 and b"T and N" in lib.ct3_last_error()
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
