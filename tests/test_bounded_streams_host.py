"""CPU tests of bounded online streams (`OnlineStreams.open(history=h)`): the argument checks, the frame count a result
covers, the frame limit reported before any work, the ring's size, and the ring-mode ABI rejections
ct3_online_window_begin / _end return before any launch."""
import ctypes

import pytest
import torch

from cotracker_b200 import engine
from cotracker_b200.model import StreamPool, StreamState


def _hub(window_len=8):
    from cotracker_b200.predictor import CoTrackerOnlinePredictor
    from cotracker_b200.streams import OnlineStreams
    return OnlineStreams(CoTrackerOnlinePredictor(checkpoint=None, window_len=window_len))


def _register(hub, sid, history=None, n=4):
    """A stream registered by hand (open() itself needs a GPU)."""
    state = hub.pool.open(torch.zeros(n, dtype=torch.int32), torch.zeros(n, 2), history=history)
    hub._streams[sid] = dict(state=state, hw=(64, 64), out=(n, (1.0, 1.0)))
    return state


@pytest.mark.parametrize("bad", [0, -3, 2.0, 1.5, "8", True, False, [4], torch.tensor(4)])
def test_open_rejects_a_bad_history_before_any_allocation(bad):
    hub = _hub()
    with pytest.raises(ValueError, match="history"):
        hub.open(frame_size=(64, 64), grid_size=3, history=bad)
    assert hub.pool.streams == [] and hub.pool.support is None and hub._streams == {}


def test_open_accepts_a_valid_history_up_to_the_device_check():
    hub = _hub()
    for ok in (None, 1, 16, 10 ** 6):
        with pytest.raises(ValueError, match="CUDA"):                      # the model is on the CPU
            hub.open(frame_size=(64, 64), grid_size=3, history=ok)


def test_length_follows_the_stream():
    hub = _hub()
    state = _register(hub, 3, history=5)
    assert hub.length(3) == 0 and state.history == 5
    state.ind, state.length = 4, 8                                          # after one full 8-frame window
    assert hub.length(3) == 8
    state.ind, state.length = 400, 404
    assert hub.length(3) == 404
    hub.close(3)
    with pytest.raises(KeyError):
        hub.length(3)


def test_ring_is_allocated_once_and_holds_what_a_window_reads():
    S, step = 16, 8
    for h in (1, 5, 8, 16, 23, 200):
        s = StreamState(3, 0, history=h)
        cap = s.ring_frames(S, step)
        assert cap >= S and cap >= h
        # the window at ind reads [ind + T - L, ind) while the ring holds [ind + S - step - cap, ind + S - step)
        for T in range(1, S + 1):
            L = min(h, 1000 + T)
            assert 1000 + T - L >= 1000 + S - step - cap
        s.reserve(cap, "cpu")
        buf = s.hist[0]
        s.reserve(cap, "cpu")
        assert s.hist[0] is buf and buf.shape == (cap, 3, 2)
    assert StreamState(3, 0).history is None


def test_frame_limit_is_reported_by_push_before_any_work():
    hub = _hub()
    S, step = 8, 4
    state = _register(hub, 7, history=16)
    lim = engine.STREAM_FRAME_LIMIT
    assert lim == 1 << 30
    state.ind, state.length = lim - S, lim - S + S - step                  # the last window that fits
    hub.push(7, torch.zeros(1, S, 3, 64, 64))
    hub._pending.clear()
    state.ind, state.length = lim - S + step, lim - S + step + S - step    # one window further
    with pytest.raises(ValueError, match="frame limit"):
        hub.push(7, torch.zeros(1, S, 3, 64, 64))
    assert 7 not in hub._pending
    unbounded = _register(hub, 8)                                           # the limit holds for every stream
    unbounded.ind, unbounded.length = state.ind, state.length
    with pytest.raises(ValueError, match="frame limit"):
        hub.push(8, torch.zeros(1, S, 3, 64, 64))


def test_struct_layout_appends_the_ring_fields():
    fields = [f for f, _ in engine.OnlineStream._fields_]
    assert fields[-3:] == ["out_first", "ring", "pad"] and len(fields) == 18
    assert ctypes.sizeof(engine.OnlineStream) == 104 and ctypes.sizeof(engine.OnlineStream) % 8 == 0
    assert engine.OnlineStream.out_first.offset == 88


def test_ring_abi_rejections_before_any_launch():
    lib = engine.lib()
    p = ctypes.c_void_p(1 << 20)

    def entry(**kw):
        e = engine.OnlineStream(p.value, p.value, p.value, 64, 0, None, None, 0, 16, 10, 0, 0, 10, 1.0, 1.0)
        for k, v in kw.items():
            setattr(e, k, v)
        return e

    def begin(entries, S=16, step=8, ws=4096):
        arr = (engine.OnlineStream * len(entries))(*entries)
        return lib.ct3_online_window_begin(arr, len(entries), S, step, 4, 16, p, p, 10, p, p, p, p, p, p, p, ws, None)

    def end(entries, S=16, ws=4096):
        arr = (engine.OnlineStream * len(entries))(*entries)
        return lib.ct3_online_window_end(arr, len(entries), S, 4, p, p, p, 10, ctypes.c_float(0.6), p, ws, None)

    def err():
        return lib.ct3_last_error()

    out = dict(tracks=p.value, visibility=p.value)
    # a ring shorter than the window
    assert begin([entry(ring=1, cap=15)]) == -1 and b"at least S" in err()
    assert end([entry(ring=1, cap=15)]) == -1 and b"at least S" in err()
    assert begin([entry(ring=2)]) == -1 and b"ring" in err()
    # an overlap frame the ring no longer holds: frames [len - cap, len) = [84, 100)
    assert begin([entry(ring=1, cap=16, ind=80, len=100)]) == -1 and b"no longer holds" in err()
    # an output longer than the ring: a frame read would share its row with a frame written
    assert end([entry(ring=1, cap=16, ind=80, len=88, T=16, out_first=79, **out)]) == -1 and b"fit in the ring" in err()
    # an output frame before the window the ring no longer holds: frames [len - cap, len) = [72, 88)
    assert end([entry(ring=1, cap=20, ind=80, len=88, T=4, out_first=67, **out)]) == -1 and b"no longer holds" in err()
    # out_first outside [0, ind + T), either mode
    for ring in (0, 1):
        assert end([entry(ring=ring, cap=64, ind=8, len=16, out_first=24, **out)]) == -1 and b"out_first" in err()
        assert end([entry(ring=ring, cap=64, ind=8, len=16, out_first=-1, **out)]) == -1 and b"out_first" in err()
    # the ring may hold fewer frames than the stream has; a plain history may not
    assert end([entry(ring=0, cap=90, ind=80, len=88)]) == -1 and b"ind + T" in err()
    assert begin([entry(ring=0, cap=16, ind=80, len=88)]) == -1 and b"len <= cap" in err()


def test_positional_entries_keep_the_plain_history_checks():
    """An entry built positionally with the 15 original fields has out_first = ring = 0: the plain history checks and
    their messages, unchanged."""
    lib = engine.lib()
    p = ctypes.c_void_p(1 << 20)
    e = engine.OnlineStream(p.value, p.value, p.value, 64, 0, None, None, 0, 16, 10, 0, 0, 10, 1.0, 1.0)
    assert (e.out_first, e.ring, e.pad) == (0, 0, 0)

    def one(**kw):
        x = engine.OnlineStream.from_buffer_copy(e)
        for k, v in kw.items():
            setattr(x, k, v)
        return (engine.OnlineStream * 1)(x)

    assert lib.ct3_online_window_begin(one(len=65), 1, 16, 8, 4, 16, p, p, 10, p, p, p, p, p, p, p, 4096, None) == -1
    assert b"len <= cap" in lib.ct3_last_error()
    assert lib.ct3_online_window_end(one(ind=50, len=50), 1, 16, 4, p, p, p, 10, ctypes.c_float(0.6), p, 4096,
                                     None) == -1
    assert b"ind + T" in lib.ct3_last_error()


def test_engine_entry_carries_out_first_and_ring():
    with pytest.raises(engine.EngineError):                                 # the wrapper takes CUDA tensors only
        engine.online_stream((torch.zeros(4, 3, 2), torch.zeros(4, 3), torch.zeros(4, 3)), 0, 0, 4, 0, 0,
                             out_first=2, ring=True)


def test_pool_open_passes_the_bound():
    pool = StreamPool()
    a = pool.open(torch.zeros(3, dtype=torch.int32), torch.zeros(3, 2), history=9)
    b = pool.open(torch.zeros(2, dtype=torch.int32), torch.zeros(2, 2))
    assert (a.history, b.history) == (9, None) and (b.first, b.n) == (3, 2)
