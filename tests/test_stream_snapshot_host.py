"""CPU tests of stream snapshots (`OnlineStreams.snapshot` / `restore`): the pool and history surgery of
`StreamPool.export` / `restore` on CPU tensors (plain, wrapped-ring and edited streams), every rejection of
`restore` before any state changes, the stream states `check_snapshot` accepts, the weights fingerprint, and a
`torch.save` / `torch.load(weights_only=True)` round trip."""
import io

import pytest
import torch

from cotracker_b200.streams import SNAPSHOT_FORMAT, check_snapshot

S, STEP, STRIDE = 16, 8, 4


def _hub():
    from cotracker_b200.predictor import CoTrackerOnlinePredictor
    from cotracker_b200.streams import OnlineStreams
    return OnlineStreams(CoTrackerOnlinePredictor(checkpoint=None, window_len=S))


def _register(hub, sid, n, n_keep, history=None, length=0, seed=0):
    """A stream registered by hand on CPU tensors (open() itself needs a GPU), with a filled history of `length`
    frames and filled support features."""
    g = torch.Generator().manual_seed(seed)
    state = hub.pool.open(torch.randint(0, 40, (n,), generator=g, dtype=torch.int32), torch.rand(n, 2, generator=g) * 90,
                          history=history)
    hub.pool.support[:, :, state.first:] = torch.randn(4, 49, n, 128, generator=g)
    if length:
        state.reserve(length if history is None else state.ring_frames(S, STEP), "cpu")
        for h in state.hist:
            h.copy_(torch.randn(h.shape, generator=g) * 50)
        state.ind, state.length = length - (S - STEP), length
    hub._streams[sid] = dict(state=state, hw=(96, 128), out=(n_keep, (0.5, 0.25)), ids=list(range(n_keep)),
                             next_id=n_keep)
    return state


def _hub_state(hub):
    pool = hub.pool
    return ([t.clone() for t in (pool.support, pool.qframes, pool.qcoords)],
            [(s.first, s.n, s.ind, s.length, s.history, None if s.hist is None else [h.clone() for h in s.hist])
             for s in pool.streams],
            {k: (v["hw"], v["out"], list(v["ids"]), v["next_id"]) for k, v in hub._streams.items()}, hub._next_id)


def _same(a, b):
    (ta, sa, da, ia), (tb, sb, db, ib) = a, b
    assert all(torch.equal(x, y) for x, y in zip(ta, tb)) and (da, ia) == (db, ib) and len(sa) == len(sb)
    for x, y in zip(sa, sb):
        assert x[:5] == y[:5] and (x[5] is None) == (y[5] is None)
        assert x[5] is None or all(torch.equal(p, q) for p, q in zip(x[5], y[5]))


def _three(history, edit=False):
    """Three streams; the middle one has 4 user tracks and a 36-point support grid, 48 frames of history (a ring of
    `history` wraps: 48 > 16 rows at history 5), and optionally a retire of user columns 0 and 2 plus an add of 3."""
    hub = _hub()
    states = [_register(hub, 0, 7, 7, length=32, seed=3), _register(hub, 1, 40, 4, history=history, length=48, seed=4),
              _register(hub, 2, 5, 5, history=9, length=24, seed=5)]
    if edit:
        hub.pool.edit(states[1], [1, 3] + list(range(4, 40)), 2, torch.tensor([48, 50, 70], dtype=torch.int32),
                      torch.tensor([[1.25, 2.5], [10.0, 0.0], [127.75, 95.5]]), STRIDE)
        hub._streams[1].update(out=(5, (0.5, 0.25)), ids=[1, 3, 4, 5, 6], next_id=7)
    return hub, states


@pytest.mark.parametrize("history,edit", [(None, False), (5, False), (None, True), (30, True)])
def test_export_close_restore_round_trip(history, edit):
    hub, (s0, s1, s2) = _three(history, edit)
    pool = hub.pool
    a, b = s1.first, s1.first + s1.n
    sup, qf, qc = pool.support[:, :, a:b].clone(), pool.qframes[a:b].clone(), pool.qcoords[a:b].clone()
    hist = [h.clone() for h in s1.hist]
    others = [(t.clone(), u.clone()) for t, u in ((pool.support[:, :, :a], pool.support[:, :, b:]),
                                                   (pool.qframes[:a], pool.qframes[b:]))]
    snap = pool.export(s1)
    assert snap["n"] == s1.n == (41 if edit else 40) and (snap["ind"], snap["length"]) == (40, 48)
    assert all(not t.is_cuda for t in [snap["support"], snap["qframes"], snap["qcoords"], *snap["hist"]])
    pool.close(s1)
    assert (s0.first, s2.first) == (0, 7)
    r = pool.restore(snap, "cpu")
    assert pool.streams == [s0, s2, r] and (s0.first, s2.first, r.first) == (0, 7, 12)
    assert (r.n, r.ind, r.length, r.history) == (s1.n, 40, 48, history)
    assert torch.equal(pool.support[:, :, 12:], sup) and torch.equal(pool.qframes[12:], qf)
    assert torch.equal(pool.qcoords[12:], qc)
    assert torch.equal(pool.support[:, :, :a], others[0][0]) and torch.equal(pool.support[:, :, a:12], others[0][1])
    assert torch.equal(pool.qframes[:a], others[1][0]) and torch.equal(pool.qframes[a:12], others[1][1])
    rows = r.ring_frames(S, STEP) if history is not None else 48       # the whole ring; frames so far
    assert r.hist[1].shape[0] == rows and all(h.is_contiguous() for h in r.hist)
    for x, y in zip(r.hist, hist):
        assert torch.equal(x, y[:rows])
    # the restored state owns its tensors: a second restore of the same snapshot is an independent stream
    r2 = pool.restore(snap, "cpu")
    r.hist[0].add_(1.0)
    pool.support[:, :, 12:12 + r.n] = 0.0
    assert torch.equal(r2.hist[0], hist[0][:rows]) and torch.equal(pool.support[:, :, r2.first:], sup)
    assert torch.equal(snap["hist"][0], hist[0][:rows]) and torch.equal(snap["support"], sup)


def test_hub_snapshot_holds_the_stream_and_the_model():
    hub, (s0, s1, s2) = _three(5, edit=True)
    snap = hub.snapshot(1)
    assert snap["format"] == SNAPSHOT_FORMAT and snap["model"] == hub.model_identity()
    assert snap["model"]["window_len"] == S and snap["model"]["stride"] == STRIDE
    assert (snap["frame_size"], snap["n_keep"], snap["ids"], snap["next_id"]) == ([96, 128], 5, [1, 3, 4, 5, 6], 7)
    assert snap["history"] == 5 and snap["hist"][0].shape == (16, 41, 2)
    check_snapshot(snap, hub.model_identity())
    check_snapshot(hub.snapshot(0), hub.model_identity())
    for k in (7, -1):
        with pytest.raises(KeyError):
            hub.snapshot(k)
    hub._pending[2] = torch.zeros(1, S, 3, 96, 128)
    with pytest.raises(ValueError, match="between steps"):
        hub.snapshot(2)


def test_snapshot_round_trips_through_torch_save_with_weights_only():
    hub, _ = _three(None, edit=True)
    for sid in (0, 1, 2):
        snap = hub.snapshot(sid)
        buf = io.BytesIO()
        torch.save(snap, buf)
        buf.seek(0)
        back = torch.load(buf, weights_only=True)
        assert back.keys() == snap.keys()
        for k, v in snap.items():
            if k == "hist":
                assert all(torch.equal(x, y) for x, y in zip(back[k], v))
            elif torch.is_tensor(v):
                assert torch.equal(back[k], v) and back[k].dtype == v.dtype
            else:
                assert back[k] == v, k
        check_snapshot(back, hub.model_identity())


def test_fingerprint_follows_the_weights_and_is_cached():
    hub = _hub()
    m = hub.model
    fp = m.weights_fingerprint()
    assert isinstance(fp, str) and len(fp) == 64 and m.weights_fingerprint() is fp     # cached, not recomputed
    w = next(m.parameters())
    old = w.view(-1)[0].item()
    with torch.no_grad():
        w.view(-1)[0] = old + 1.0
    assert m.weights_fingerprint() != fp
    with torch.no_grad():
        w.view(-1)[0] = old
    assert m.weights_fingerprint() == fp                                    # the same weights, the same fingerprint
    m.time_emb.mul_(2.0)                                                    # buffers count too
    assert m.weights_fingerprint() != fp


def _bad(snap, **kw):
    bad = dict(snap)
    for k, v in kw.items():
        if v is KeyError:
            del bad[k]
        else:
            bad[k] = v
    return bad


def _rejections(snap, ident):
    """(snapshot, message) for every rejection; `snap` is a snapshot of a ring stream (history 5) of 41 tracks,
    n_keep 5, at ind 40, length 48."""
    n = snap["n"]
    hist = snap["hist"]
    model = lambda **kw: dict(ident, **kw)                                   # noqa: E731
    cases = [
        ("not a dict", [snap], "is a dict"),
        ("format", _bad(snap, format=2), "unknown snapshot format 2"),
        ("format True", _bad(snap, format=True), "unknown snapshot format"),
        ("no format", _bad(snap, format=KeyError), "unknown snapshot format None"),
        ("missing", _bad(snap, hist=KeyError), "misses the fields \\['hist'\\]"),
        ("model type", _bad(snap, model=None), "model must be a dict"),
        ("window_len", _bad(snap, model=model(window_len=8)), "window_len"),
        ("interp_shape", _bad(snap, model=model(interp_shape=[192, 256])), "interp_shape"),
        ("stride", _bad(snap, model=model(stride=8)), "stride"),
        ("weights", _bad(snap, model=model(weights="0" * 64)), "weights"),
        ("n type", _bad(snap, n=float(n)), "n must be an int"),
        ("ind bool", _bad(snap, ind=True), "ind must be an int"),
        ("length tensor", _bad(snap, length=torch.tensor(48)), "length must be an int"),
        ("frame_size", _bad(snap, frame_size=[96]), "frame_size"),
        ("frame_size small", _bad(snap, frame_size=[1, 128]), "frame_size"),
        ("history", _bad(snap, history=0), "history"),
        ("history type", _bad(snap, history=5.0), "history"),
        ("ids type", _bad(snap, ids=[1, 3, 4, 5, 6.0]), "ids must be a list of ints"),
        ("ids length", _bad(snap, ids=[1, 3, 4, 5]), "n_keep = 5 distinct ids"),
        ("ids duplicate", _bad(snap, ids=[1, 3, 4, 5, 5]), "distinct"),
        ("ids past next_id", _bad(snap, ids=[1, 3, 4, 5, 7]), "next_id = 7"),
        ("n_keep", _bad(snap, n_keep=n + 1), "n_keep"),
        ("n_keep 0", _bad(snap, n_keep=0, ids=[]), "n_keep"),
        ("support n", _bad(snap, support=snap["support"][:, :, 1:]), "support"),
        ("support dtype", _bad(snap, support=snap["support"].double()), "support"),
        ("support type", _bad(snap, support=snap["support"].numpy()), "support"),
        ("qframes n", _bad(snap, qframes=snap["qframes"][1:]), "qframes"),
        ("qframes dtype", _bad(snap, qframes=snap["qframes"].long()), "qframes"),
        ("qframes range", _bad(snap, qframes=snap["qframes"].clone().fill_(2 ** 30 + 1)), "past"),
        ("qcoords", _bad(snap, qcoords=snap["qcoords"][:, :1]), "qcoords"),
        ("n", _bad(snap, n=n - 1), "support"),
        ("ind negative", _bad(snap, ind=-8, length=0), ">= 0"),
        ("length negative", _bad(snap, length=-1), ">= 0"),
        ("ind off the step", _bad(snap, ind=36), "no stream reaches"),
        ("length past the chunk", _bad(snap, length=49), "no stream reaches"),
        ("length before the window", _bad(snap, length=32), "no stream reaches"),
        ("length without a window", _bad(snap, ind=0), "no stream reaches"),
        ("frame limit", _bad(snap, ind=2 ** 30, length=2 ** 30), "frame limit"),
        ("hist type", _bad(snap, hist=hist[0]), "hist must be"),
        ("hist arity", _bad(snap, hist=hist[:2]), "hist must be"),
        ("ring rows", _bad(snap, hist=[h[:15] for h in hist]), "ring of 16 frames"),
        ("ring coords", _bad(snap, hist=[hist[0][:, :, :1], hist[1], hist[2]]), "hist coords"),
        ("conf dtype", _bad(snap, hist=[hist[0], hist[1], hist[2].half()]), "hist conf"),
        ("conf n", _bad(snap, hist=[hist[0], hist[1], hist[2][:, 1:]]), "hist conf"),
        ("not advanced", _bad(snap, ind=0, length=0), "has no history"),
        ("unbounded rows", _bad(snap, history=None, hist=[h[:15] for h in hist], ind=24, length=32), "holds 32"),
    ]
    return cases


def test_every_rejection_happens_before_any_state_change():
    hub, _ = _three(5, edit=True)
    snap = hub.snapshot(1)
    ident = hub.model_identity()
    before = _hub_state(hub)
    cases = _rejections(snap, ident)
    assert len({name for name, _, _ in cases}) == len(cases)
    for name, bad, match in cases:
        with pytest.raises(ValueError, match=match):
            check_snapshot(bad, ident)
        with pytest.raises(ValueError, match=match):
            hub.restore(bad)
        _same(before, _hub_state(hub))
    # a valid snapshot passes every check; this hub's model is on the CPU, so restore() stops at the device
    with pytest.raises(ValueError, match="CUDA"):
        hub.restore(snap)
    _same(before, _hub_state(hub))


def test_the_states_a_stream_reaches_are_accepted():
    """Window starts and lengths after k windows of chunks of 1..S frames; the last one short (an ended stream)."""
    hub = _hub()
    ident = hub.model_identity()
    _register(hub, 0, 3, 3)
    snap = hub.snapshot(0)
    assert snap["hist"] is None and (snap["ind"], snap["length"]) == (0, 0)
    check_snapshot(snap, ident)
    for ind, length in ((8, 1), (8, 16), (16, 9), (16, 24), (40, 35), (2 ** 30 - 8, 2 ** 30 - 5),
                        (2 ** 30 - 8, 2 ** 30)):
        hist = [torch.zeros(16, 3, 2), torch.zeros(16, 3), torch.zeros(16, 3)]
        check_snapshot(dict(snap, ind=ind, length=length, history=1, hist=hist), ident)
    for ind, length in ((8, 0), (8, 17), (16, 8), (2 ** 30, 2 ** 30)):
        with pytest.raises(ValueError):
            check_snapshot(dict(snap, ind=ind, length=length, history=1,
                                hist=[torch.zeros(16, 3, 2), torch.zeros(16, 3), torch.zeros(16, 3)]), ident)
    # an unbounded history may hold more rows than frames (its buffers double); restore keeps [0, length)
    check_snapshot(dict(snap, ind=16, length=20, hist=[torch.zeros(32, 3, 2), torch.zeros(32, 3),
                                                     torch.zeros(32, 3)]), ident)
