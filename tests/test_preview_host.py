"""CPU tests of online stream previews (`OnlineStreams.push(sid, chunk, preview=True)`): the argument checks of push,
which raise before any device work, and the ABI of the `preview` field of ct3_online_stream with the rejections
ct3_online_window_end / _end_scores return before any launch."""
import ctypes

import pytest
import torch

from cotracker_b200 import engine

S, STEP = 16, 8


def _hub():
    from cotracker_b200.predictor import CoTrackerOnlinePredictor
    from cotracker_b200.streams import OnlineStreams
    return OnlineStreams(CoTrackerOnlinePredictor(checkpoint=None, window_len=S))


def _register(hub, sid, ind=0, length=0, n=4):
    """A stream registered by hand (open() itself needs a GPU), at window start ind with length frames."""
    state = hub.pool.open(torch.zeros(n, dtype=torch.int32), torch.zeros(n, 2))
    state.ind, state.length = ind, length
    hub._streams[sid] = dict(state=state, hw=(64, 64), out=(n, (1.0, 1.0)), ids=list(range(n)), next_id=n)
    return state


def _chunk(T):
    return torch.zeros(1, T, 3, 64, 64, dtype=torch.uint8)


@pytest.mark.parametrize("bad", [1, 0, None, "yes", 1.0, torch.tensor(True)])
def test_preview_must_be_a_bool(bad):
    hub = _hub()
    _register(hub, 0)
    with pytest.raises(ValueError, match="preview must be a bool"):
        hub.push(0, _chunk(4), preview=bad)
    assert hub._pending == {} and hub._previews == set()


def test_a_preview_must_add_a_frame():
    """A preview holds frames [ind, f] with f >= length: T > length - ind.  Before the first step any T in [1, S]."""
    hub = _hub()
    _register(hub, 0)
    for T in (1, 9, S):
        hub.push(0, _chunk(T), preview=True)
        assert hub._previews == {0}
        hub.close(0)
        assert hub._previews == set() and hub._pending == {}
        _register(hub, 0)
    _register(hub, 1, ind=STEP, length=S)                  # after one window: frames [8, 16) are held
    for T in (1, STEP):
        with pytest.raises(ValueError, match="must add a frame after frame 15"):
            hub.push(1, _chunk(T), preview=True)
        assert 1 not in hub._pending and hub._previews == set()
    hub.push(1, _chunk(STEP), preview=False)               # the same chunk may still end the stream
    hub._pending.clear()
    for T in (STEP + 1, S - 1, S):
        hub.push(1, _chunk(T), preview=True)
        assert hub._previews == {1} and hub._pending[1].shape[1] == T
        hub._pending.clear()
        hub._previews.clear()


def test_a_preview_passes_the_checks_of_any_chunk():
    hub = _hub()
    _register(hub, 0, ind=2 * STEP, length=2 * STEP + 4)   # its last chunk was short: the stream has ended
    with pytest.raises(ValueError, match="has ended"):
        hub.push(0, _chunk(S), preview=True)
    _register(hub, 1, ind=STEP, length=S)
    for T in (0, S + 1):
        with pytest.raises(ValueError, match="1 to window_len"):
            hub.push(1, _chunk(T), preview=True)
    with pytest.raises(ValueError, match="takes chunks"):
        hub.push(1, torch.zeros(1, S, 3, 32, 64), preview=True)
    hub.push(1, _chunk(S), preview=True)
    with pytest.raises(ValueError, match="already has a chunk"):
        hub.push(1, _chunk(S), preview=True)
    with pytest.raises(ValueError, match="already has a chunk"):
        hub.push(1, _chunk(S))
    assert hub._previews == {1}


def test_snapshot_rejects_a_pending_preview():
    hub = _hub()
    _register(hub, 0)
    hub.push(0, _chunk(3), preview=True)
    with pytest.raises(ValueError, match="between steps"):
        hub.snapshot(0)


def test_preview_is_the_last_field_of_the_stream_entry():
    assert ctypes.sizeof(engine.OnlineStream) == 104
    e = engine.OnlineStream()
    assert e.preview == 0
    e.preview = 1
    assert e.pad == 1 and bytes(e)[-4:] == (1).to_bytes(4, "little")
    with pytest.raises(engine.EngineError, match="track count"):
        engine.online_stream(None, 0, 0, 4, 0, 0, preview=True)
    e = engine.online_stream(None, 0, 0, 4, 0, 0, preview=True, n=7)
    assert (e.coords, e.vis, e.conf, e.cap, e.len, e.ring, e.n, e.preview) == (None, None, None, 0, 0, 0, 7, 1)


def test_preview_abi_rejections_before_any_launch():
    lib = engine.lib()
    p = ctypes.c_void_p(1 << 20)

    def entry(**kw):
        e = engine.OnlineStream(p.value, p.value, p.value, 64, 16, p.value, p.value, 8, 16, 10, 0, 0, 10, 1.0, 1.0)
        for k, v in kw.items():
            setattr(e, k, v)
        return e

    def end(e):
        arr = (engine.OnlineStream * 1)(e)
        return lib.ct3_online_window_end(arr, 1, S, 4, p, p, p, 10, ctypes.c_float(0.6), p, 4096, None)

    def end_scores(e):
        arr = (engine.OnlineStream * 1)(e)
        sc = (engine.OnlineScores * 1)(engine.OnlineScores(None, None))
        return lib.ct3_online_window_end_scores(arr, 1, S, 4, p, p, p, 10, ctypes.c_float(0.6), sc, p, 4096, None)

    for call in (end, end_scores):
        for bad in (2, -1, 1 << 20):
            assert call(entry(preview=bad)) == -1 and b"preview must be 0 or 1" in lib.ct3_last_error()
        assert call(entry(preview=1, tracks=None)) == -1 and b"preview entry needs an output" in lib.ct3_last_error()
        # a missing history is accepted for a preview at ind = 0 only, with cap = len = ring = 0
        bare = dict(coords=None, vis=None, conf=None, cap=0, len=0)
        assert call(entry(preview=0, ind=0, **bare)) == -1 and b"history is null" in lib.ct3_last_error()
        assert call(entry(preview=1, ind=8, **bare)) == -1 and b"history" in lib.ct3_last_error()
        assert call(entry(preview=1, ind=0, **dict(bare, cap=64))) == -1 and b"null" in lib.ct3_last_error()
        assert call(entry(preview=1, ind=0, **dict(bare, vis=p.value))) == -1 and b"null" in lib.ct3_last_error()
        assert call(entry(preview=1, ind=0, ring=1, **bare)) == -1 and b"at least S" in lib.ct3_last_error()
        # the other checks hold for a preview as for any entry
        assert call(entry(preview=1, len=4)) == -1 and b"before its window" in lib.ct3_last_error()
        assert call(entry(preview=1, out_first=24)) == -1 and b"out_first" in lib.ct3_last_error()
