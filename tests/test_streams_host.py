"""CPU tests of independent online streams: the track pool's bookkeeping on open / close, pass planning over streams
of different sizes, and every error OnlineStreams and the window kernels' ABI report before touching a device."""
import ctypes

import pytest
import torch

from cotracker_b200 import engine
from cotracker_b200.evaluation import pass_bytes, plan_clip_passes
from cotracker_b200.model import StreamPool, StreamState


def _open(pool, n, tag):
    return pool.open(torch.full((n,), tag, dtype=torch.int32), torch.full((n, 2), float(tag)))


def test_pool_appends_and_compacts_on_close():
    pool = StreamPool()
    a, b, c = _open(pool, 3, 1), _open(pool, 5, 2), _open(pool, 2, 3)
    assert [(s.first, s.n) for s in pool.streams] == [(0, 3), (3, 5), (8, 2)]
    assert pool.support.shape == (4, 49, 10, 128) and pool.qframes.tolist() == [1] * 3 + [2] * 5 + [3] * 2
    pool.support[:, :, 8:] = 7.0
    pool.close(b)
    assert pool.streams == [a, c] and (c.first, c.n) == (3, 2)
    assert pool.qframes.tolist() == [1, 1, 1, 3, 3] and pool.qcoords[:, 0].tolist() == [1, 1, 1, 3, 3]
    assert pool.support.shape == (4, 49, 5, 128) and bool((pool.support[:, :, 3:] == 7).all())
    d = _open(pool, 4, 4)
    assert (d.first, d.n) == (5, 4) and pool.qframes.tolist()[5:] == [4] * 4
    for s in (a, c, d):
        pool.close(s)
    assert pool.streams == [] and pool.support is None


def test_history_grows_geometrically_and_keeps_its_frames():
    s = StreamState(3, 0)
    s.reserve(16, "cpu")
    s.hist[0][:16] = torch.arange(16.0)[:, None, None]
    s.length = 16
    s.reserve(24, "cpu")
    assert s.hist[1].shape[0] == 32 and torch.equal(s.hist[0][:16, 0, 0], torch.arange(16.0))
    s.reserve(30, "cpu")
    assert s.hist[1].shape[0] == 32                      # room left: no reallocation


def test_ragged_pass_plan_covers_every_stream_once_within_budget():
    sizes = [[100], [2500], [36], [700], [1], [900]]
    T, H4, W4 = 16, 96, 128

    def cost(b0, b1):
        return pass_bytes(T, sum(s[0] for s in sizes[b0:b1]), b1 - b0, H4, W4, 6 * T)

    budget = cost(1, 3)
    passes = plan_clip_passes(len(sizes), sizes, T, H4, W4, budget, lambda n: 6 * T)
    assert [i for b0, b1 in passes for i in range(b0, b1)] == list(range(len(sizes)))
    assert all(cost(b0, b1) <= budget or b1 - b0 == 1 for b0, b1 in passes)
    assert all(cost(b0, b1 + 1) > budget for b0, b1 in passes[:-1])          # greedy: each pass as long as fits
    assert plan_clip_passes(len(sizes), sizes, T, H4, W4, 1 << 62, lambda n: 6 * T) == [(0, 6)]
    assert plan_clip_passes(3, [[5], [6], [7]], T, H4, W4, 1) == [(0, 1), (1, 2), (2, 3)]
    with pytest.raises(ValueError):
        plan_clip_passes(2, [[5]], T, H4, W4, 1)


def test_stream_errors_before_any_launch():
    from cotracker_b200.predictor import CoTrackerOnlinePredictor
    from cotracker_b200.streams import OnlineStreams
    p = CoTrackerOnlinePredictor(checkpoint=None, window_len=8)
    hub = OnlineStreams(p)
    with pytest.raises(ValueError, match="queries or grid_size"):
        hub.open(frame_size=(64, 64), grid_size=0)
    with pytest.raises(ValueError, match="queries"):
        hub.open(frame_size=(64, 64), queries=torch.zeros(2, 5, 3))
    with pytest.raises(ValueError, match="CUDA"):                          # the model is on the CPU
        hub.open(frame_size=(64, 64), grid_size=3)
    for call in (lambda: hub.push(0, torch.zeros(1, 8, 3, 64, 64)), lambda: hub.close(0)):
        with pytest.raises(KeyError):
            call()
    # a stream registered by hand (open() itself needs a GPU) to reach push()'s checks
    state = hub.pool.open(torch.zeros(4, dtype=torch.int32), torch.zeros(4, 2))
    hub._streams[7] = dict(state=state, hw=(64, 64), out=(4, (1.0, 1.0)))
    for bad in (torch.zeros(8, 3, 64, 64), torch.zeros(2, 8, 3, 64, 64), torch.zeros(1, 8, 3, 64, 48),
                torch.zeros(1, 8, 4, 64, 64)):
        with pytest.raises(ValueError, match="takes chunks"):
            hub.push(7, bad)
    for T in (0, 9):
        with pytest.raises(ValueError, match="window_len"):
            hub.push(7, torch.zeros(1, T, 3, 64, 64))
    hub.push(7, torch.zeros(1, 8, 3, 64, 64))
    with pytest.raises(ValueError, match="already has a chunk"):
        hub.push(7, torch.zeros(1, 8, 3, 64, 64))
    state.ind, state.length = 4, 7                                          # after a 7-frame chunk at window start 0
    hub._pending.clear()
    with pytest.raises(ValueError, match="ended"):
        hub.push(7, torch.zeros(1, 8, 3, 64, 64))
    hub.close(7)
    with pytest.raises(KeyError):
        hub.push(7, torch.zeros(1, 8, 3, 64, 64))


def test_online_window_abi_rejects_bad_arguments():
    """ct3_online_window_begin / _end are exported and return CT3_EINVAL (CT3_ENOSPC for a small workspace) before any
    launch."""
    lib = engine.lib()
    for name in ("ct3_online_window_begin", "ct3_online_window_end"):
        assert name in engine.EXPORTED_SYMBOLS and hasattr(lib, name)
    p = ctypes.c_void_p(1 << 20)

    def entry(**kw):
        e = engine.OnlineStream(p.value, p.value, p.value, 64, 0, None, None, 0, 16, 10, 0, 0, 10, 1.0, 1.0)
        for k, v in kw.items():
            setattr(e, k, v)
        return e

    def begin(entries, S=16, step=8, stride=4, T_pyr=16, N=10, ws=4096, q=p):
        arr = (engine.OnlineStream * len(entries))(*entries)
        return lib.ct3_online_window_begin(arr, len(entries), S, step, stride, T_pyr, q, p, N, p, p, p, p, p, p, p, ws,
                                           None)

    def end(entries, S=16, stride=4, N=10, ws=4096):
        arr = (engine.OnlineStream * len(entries))(*entries)
        return lib.ct3_online_window_end(arr, len(entries), S, stride, p, p, p, N, ctypes.c_float(0.6), p, ws, None)

    assert begin([entry()], q=None) == -1 and b"null" in lib.ct3_last_error()
    assert begin([entry()], ws=8) == -3
    assert begin([entry()], S=1) == -1 and begin([entry()], step=16) == -1 and begin([entry()], stride=0) == -1
    assert begin([entry(n=0)]) == -1 and b"tile" in lib.ct3_last_error()
    assert begin([entry(), entry(first=10)], N=15) == -1                    # tracks past N
    assert begin([entry(n=5), entry(n=5, first=4)]) == -1                   # overlapping streams
    assert begin([entry(T=0)]) == -1 and begin([entry(T=17)]) == -1
    assert begin([entry(ind=-1)]) == -1 and begin([entry(ind=1 << 30)]) == -1
    assert begin([entry(frame0=1)]) == -1 and b"T_pyr" in lib.ct3_last_error()
    assert begin([entry(ind=8, len=15)]) == -1 and b"overlap" in lib.ct3_last_error()
    assert begin([entry(ind=8, len=16, coords=None)]) == -1 and b"null" in lib.ct3_last_error()
    assert begin([entry(len=65)]) == -1
    assert end([entry(ind=50, len=50)]) == -1 and b"ind + T" in lib.ct3_last_error()
    assert end([entry(ind=8, len=7)]) == -1 and b"before its window" in lib.ct3_last_error()
    assert end([entry(tracks=p.value)]) == -1 and b"visibility" in lib.ct3_last_error()
    assert end([entry(tracks=p.value, visibility=p.value, n_keep=11)]) == -1
    assert end([entry(vis=None)]) == -1
    with pytest.raises(engine.EngineError):                                 # the wrapper takes CUDA tensors only
        engine.online_stream((torch.zeros(4, 3, 2), torch.zeros(4, 3), torch.zeros(4, 3)), 0, 0, 4, 0, 0)
