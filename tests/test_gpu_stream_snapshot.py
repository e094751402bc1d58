"""GPU tests of stream snapshots (`OnlineStreams.snapshot` / `restore`).  A stream snapshotted after k steps, closed
and restored into a second hub that already holds streams of other frame sizes continues `torch.equal` to a hub that
never snapshotted it: results, track ids, length and the ids later `add_tracks` calls return, for unbounded, bounded
(before and after the ring wraps), support-grid and edited streams.  Also: a snapshot does not perturb its source;
a snapshot restored twice gives two exact copies; a `torch.save` / `torch.load(weights_only=True)` round trip; a
forced one-stream-per-pass split; the first step after a restore encodes the stream's whole chunk and later steps
reuse the cache; an ended stream stays ended; other weights are refused; snapshot + close frees the stream's device
memory; and a restore onto a second device when there is one."""
import io

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
S, STEP, STEPS = 16, 8, 8
H, W = 96, 128


def _predictor(seed=53, dev=DEV):
    from cotracker_b200.predictor import CoTrackerOnlinePredictor
    from cotracker_b200.synthetic import seeded_state_dict
    p = CoTrackerOnlinePredictor(checkpoint=None, window_len=S)
    p.model.load_state_dict(seeded_state_dict(seed, offline=False, window_len=S, head_gain=10.0, vis_gain=100.0))
    return p.to(dev)


def _video(T, h, w, seed, dev=DEV):
    from cotracker_b200.synthetic import texture_video
    return texture_video(T, h, w, seed=seed, shift=(1 + seed % 3, 2)).to(dev)


def _queries(n, t0, t1, seed, h=H, w=W, dev=DEV):
    """[1,n,3] queries with frames in [t0, t1)."""
    g = torch.Generator().manual_seed(seed)
    t = torch.randint(t0, t1, (n,), generator=g).float()
    return torch.stack([t, torch.rand(n, generator=g) * (w - 1), torch.rand(n, generator=g) * (h - 1)], -1)[None].to(dev)


def _specs(dev=DEV):
    """The tested streams: their video, open() arguments and edits {k: [("add", queries) | ("retire", ids)]} made in
    the gap before step k.  Adds in gaps 0, 2, 5 and 6, retires in gaps 3 and 5: before and after a snapshot at k = 1
    or 4.  Bounds 1, 5 and 16 give rings of 16, 16 and 24 frames, which wrap from k = 2, 2 and 3 on."""
    def edits():
        return {0: [("add", _queries(2, 0, 8, 10, dev=dev))], 2: [("add", _queries(3, 24, 40, 11, dev=dev))],
                3: [("retire", [1, 4, 26])],
                5: [("retire", [0]), ("add", _queries(2, 48, 56, 13, dev=dev))],
                6: [("add", _queries(1, 56, 64, 14, dev=dev))]}
    specs = dict(unbounded=dict(kw=dict(grid_size=4)),
                 h1=dict(kw=dict(grid_size=4, history=1)),
                 h5=dict(kw=dict(grid_size=4, history=5)),
                 h16=dict(kw=dict(grid_size=4, history=16)),
                 grid=dict(kw=dict(queries=_queries(6, 0, 30, 12, dev=dev), add_support_grid=True)),
                 edits=dict(kw=dict(grid_size=5), edits=edits()),
                 edits_h5=dict(kw=dict(grid_size=5, history=5), edits=edits()))
    for k, (name, sp) in enumerate(specs.items()):
        sp.update(video=_video(STEP * STEPS + S, H, W, 60 + k, dev), edits=sp.get("edits", {}))
    return specs


NAMES = ("unbounded", "h1", "h5", "h16", "grid", "edits", "edits_h5")


@pytest.fixture(scope="module")
def p():
    return _predictor()


@pytest.fixture(scope="module")
def specs():
    return _specs()


def _solo(p, spec):
    """The stream of `spec` alone on a hub that never snapshots it: per step (tracks, visibility, track_ids, length,
    ids of that gap's add_tracks)."""
    from cotracker_b200.streams import OnlineStreams
    hub = OnlineStreams(p)
    sid = hub.open(frame_size=(H, W), **spec["kw"])
    return [_advance(hub, [sid], spec, k)[0] for k in range(STEPS)]


@pytest.fixture(scope="module")
def ref(p, specs):
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = _solo(p, specs[name])
        return cache[name]
    return get


class _Others:
    """Streams of other frame sizes on a hub: one pushes at every step, one bounded at history 5 at every other."""

    def __init__(self, hub, seed):
        from cotracker_b200 import ingest
        dev = ingest.model_device(hub.model)
        self.hub, self.calls, self.pos = hub, 0, [0, 0]
        self.video = [_video(STEP * 24 + S, 80, 96, seed, dev), _video(STEP * 24 + S, 64, 80, seed + 1, dev)]
        self.sids = [hub.open(frame_size=(80, 96), grid_size=3),
                     hub.open(frame_size=(64, 80), queries=_queries(5, 0, 20, seed, 64, 80, dev), history=5)]

    def push(self) -> int:
        """Push the chunks of this step.  -> the new frames they bring to the encoder (all cached by now)."""
        pushing = [0] if self.calls % 2 else [0, 1]
        self.calls += 1
        for i in pushing:
            o = STEP * self.pos[i]
            self.hub.push(self.sids[i], self.video[i][:, o:o + S])
            self.pos[i] += 1
        return STEP * len(pushing)


def _edit(hub, sid, spec, k):
    """The edits of the gap before step k.  -> the ids add_tracks returned."""
    added = []
    for op, arg in spec["edits"].get(k, ()):
        if op == "add":
            added += hub.add_tracks(sid, arg)
        else:
            hub.retire_tracks(sid, arg)
    return added


def _step(hub, sids, spec, k, added, others=None):
    for sid in sids:
        hub.push(sid, spec["video"][:, STEP * k:STEP * k + S])
    if others is not None:
        others.push()
    out = hub.step()
    return [(*out[sid], hub.track_ids(sid), hub.length(sid), a) for sid, a in zip(sids, added)]


def _advance(hub, sids, spec, k, others=None):
    """Step k of the copies `sids` of the stream of `spec`: the gap's edits, the chunk, one `step()` of the hub.
    -> per copy (tracks, visibility, track_ids, length, ids of the gap's add_tracks)."""
    return _step(hub, sids, spec, k, [_edit(hub, sid, spec, k) for sid in sids], others)


def _moved(p, spec, k, q=None, through=None, copies=1, dst_spec=None):
    """The stream of `spec` for k steps on a hub shared with other streams, then snapshotted, closed, passed through
    `through`, and restored `copies` times into a second hub on q's model (default p's) that already holds advanced
    streams of other frame sizes, and advanced there to step STEPS with the inputs of `dst_spec` (default `spec`).
    -> per copy, the results of every step as `_solo` gives them."""
    from cotracker_b200.streams import OnlineStreams
    src = OnlineStreams(p)
    others = _Others(src, 30)
    sid = src.open(frame_size=(H, W), **spec["kw"])
    before = [_advance(src, [sid], spec, j, others)[0] for j in range(k)]
    snap = src.snapshot(sid)
    src.close(sid)
    if through is not None:
        snap = through(snap)
    dst = OnlineStreams(q or p)
    dst_others = _Others(dst, 40)
    for _ in range(2):
        dst_others.push()
        dst.step()
    rids = [dst.restore(snap) for _ in range(copies)]
    after = [_advance(dst, rids, dst_spec or spec, j, dst_others) for j in range(k, STEPS)]
    return [before + [a[c] for a in after] for c in range(copies)]


def _equal(a, b):
    assert len(a) == len(b)
    for k, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x[0], y[0]) and torch.equal(x[1], y[1]), k
        assert x[2:] == y[2:], (k, x[2:], y[2:])


def _save_load(snap):
    buf = io.BytesIO()
    torch.save(snap, buf)
    buf.seek(0)
    return torch.load(buf, weights_only=True)


@pytest.mark.parametrize("k", [0, 1, 4])
@pytest.mark.parametrize("name", NAMES)
def test_restored_stream_continues_bit_for_bit(p, specs, ref, name, k):
    (got,) = _moved(p, specs[name], k)
    _equal(got, ref(name))


def test_snapshot_does_not_perturb_the_source(p, specs, ref):
    """Snapshots before and after every gap's edits, of a stream that runs on."""
    from cotracker_b200.streams import OnlineStreams
    for name in ("edits_h5", "grid", "unbounded"):
        spec = specs[name]
        hub = OnlineStreams(p)
        others = _Others(hub, 50)
        sid = hub.open(frame_size=(H, W), **spec["kw"])
        res = []
        for k in range(STEPS):
            hub.snapshot(sid)
            added = _edit(hub, sid, spec, k)
            hub.snapshot(sid)
            res.append(_step(hub, [sid], spec, k, [added], others)[0])
        hub.snapshot(sid)
        _equal(res, ref(name))


def test_a_snapshot_restored_twice_gives_two_exact_copies(p, specs, ref):
    for name, k in (("edits_h5", 3), ("grid", 1)):
        a, b = _moved(p, specs[name], k, copies=2)
        _equal(a, ref(name))
        _equal(b, ref(name))


def test_restore_after_a_torch_save_round_trip(p, specs, ref):
    for name, k in (("edits", 4), ("h16", 4), ("h1", 0)):
        (got,) = _moved(p, specs[name], k, through=_save_load)
        _equal(got, ref(name))


def test_restored_stream_under_a_forced_one_stream_per_pass_split(p, specs, ref, monkeypatch):
    import cotracker_b200.model as M
    for name in NAMES:
        ref(name)
    passes = []
    planner = M.plan_clip_passes
    monkeypatch.setattr(M, "pass_budget_bytes", lambda *a, **k: 1)
    monkeypatch.setattr(M, "plan_clip_passes", lambda *a, **k: passes.append(planner(*a, **k)) or passes[-1])
    for name, k in (("edits_h5", 4), ("grid", 1), ("unbounded", 2)):
        (got,) = _moved(p, specs[name], k)
        _equal(got, ref(name))
    assert passes and all(b1 - b0 == 1 for pl in passes for b0, b1 in pl)


def test_first_step_after_restore_encodes_the_whole_chunk(p, specs, ref, monkeypatch):
    """The encoder gets the restored stream's whole chunk, 16 frames, at its first step after the restore, and its 8
    new frames after that.  The stream is alone on its hub here: the overlap check compares float64 frame sums, which
    need not repeat bit for bit when the set of streams that advance together changes, and then a stream's overlap is
    encoded again (with the same result); alone, the count shows the cache at work."""
    from cotracker_b200.streams import OnlineStreams
    spec, k = specs["edits"], 2
    want = ref("edits")
    log = []
    encode = p.model._encode
    monkeypatch.setattr(p.model, "_encode", lambda video, chunk: log.append(video.shape[0]) or encode(video, chunk))
    src = OnlineStreams(p)
    sid = src.open(frame_size=(H, W), **spec["kw"])
    got = [_advance(src, [sid], spec, j)[0] for j in range(k)]
    snap = src.snapshot(sid)
    src.close(sid)
    dst = OnlineStreams(p)
    rid = dst.restore(snap)
    n = len(log)
    got += [_advance(dst, [rid], spec, j)[0] for j in range(k, STEPS)]
    _equal(got, want)
    assert log[:n] == [S, STEP] and log[n:] == [S] + [STEP] * (STEPS - k - 1), log


def test_an_ended_stream_stays_ended(p, specs, ref):
    from cotracker_b200.streams import OnlineStreams
    spec = specs["h5"]
    hub = OnlineStreams(p)
    sid = hub.open(frame_size=(H, W), **spec["kw"])
    for k in range(3):
        _advance(hub, [sid], spec, k)
    hub.push(sid, spec["video"][:, STEP * 3:STEP * 3 + 5])                  # a short last chunk
    hub.step()
    with pytest.raises(ValueError, match="ended") as ended:
        hub.push(sid, spec["video"][:, STEP * 4:STEP * 4 + S])
    snap = _save_load(hub.snapshot(sid))
    length = hub.length(sid)
    hub.close(sid)
    dst = OnlineStreams(p)
    rid = dst.restore(snap)
    assert dst.length(rid) == length == STEP * 3 + 5
    with pytest.raises(ValueError, match="ended") as again:
        dst.push(rid, spec["video"][:, STEP * 4:STEP * 4 + S])
    assert str(again.value).split(": ", 1)[1] == str(ended.value).split(": ", 1)[1]


def test_restore_onto_other_weights_is_refused(p, specs):
    from cotracker_b200.streams import OnlineStreams
    spec = specs["unbounded"]
    hub = OnlineStreams(p)
    sid = hub.open(frame_size=(H, W), **spec["kw"])
    _advance(hub, [sid], spec, 0)
    snap = hub.snapshot(sid)
    dst = OnlineStreams(_predictor(seed=54))
    other = dst.open(frame_size=(H, W), grid_size=3)
    pool = [t.clone() for t in (dst.pool.support, dst.pool.qframes, dst.pool.qcoords)]
    with pytest.raises(ValueError, match="weights"):
        dst.restore(snap)
    assert list(dst._streams) == [other] and len(dst.pool.streams) == 1
    assert all(torch.equal(x, y) for x, y in zip(pool, (dst.pool.support, dst.pool.qframes, dst.pool.qcoords)))
    assert OnlineStreams(_predictor()).restore(snap) == 0                  # the same weights in another model


def test_snapshot_and_close_free_the_stream_and_restore_continues(p, specs, ref):
    """Offload: device memory returns to its level from before the stream opened, up to any growth of the
    workspaces the model keeps for its passes; a later restore continues exactly."""
    from cotracker_b200.streams import OnlineStreams
    name, k = "edits", 3
    want = [tuple(x.cpu() if torch.is_tensor(x) else x for x in r) for r in ref(name)]   # also warms the workspaces
    spec = specs[name]
    model = p.model

    def kept():
        return model._ws.buf.numel() + model._enc_ws.numel()

    torch.cuda.synchronize()
    base, kept0 = torch.cuda.memory_allocated(), kept()
    hub = OnlineStreams(p)
    sid = hub.open(frame_size=(H, W), **spec["kw"])
    got = []
    for j in range(k):
        got.append(tuple(x.cpu() if torch.is_tensor(x) else x for x in _advance(hub, [sid], spec, j)[0]))
    torch.cuda.synchronize()
    held = torch.cuda.memory_allocated() - base
    st = hub.pool.streams[0]
    own = (hub.pool.support.numel() + st.enc[2].numel() + sum(h.numel() for h in st.hist)) * 4
    del st                                                                  # the hub's references only
    snap = hub.snapshot(sid)
    hub.close(sid)
    torch.cuda.synchronize()
    assert held >= own > 0                                                  # support, encoder cache and history
    assert torch.cuda.memory_allocated() - base <= kept() - kept0, (torch.cuda.memory_allocated(), base, held)
    rid = hub.restore(snap)
    for j in range(k, STEPS):
        got.append(tuple(x.cpu() if torch.is_tensor(x) else x for x in _advance(hub, [rid], spec, j)[0]))
    _equal(got, want)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs a second CUDA device")
def test_restore_onto_a_second_device(p, specs):
    q = _predictor(dev="cuda:1")
    specs1 = _specs("cuda:1")
    for name, k in (("edits_h5", 4), ("grid", 1)):
        want = _solo(q, specs1[name])
        (got,) = _moved(p, specs[name], k, q=q, dst_spec=specs1[name])
        # the steps before the snapshot ran on cuda:0 and the rest on cuda:1; compare on the host
        _equal([tuple(x.cpu() if torch.is_tensor(x) else x for x in r) for r in got],
               [tuple(x.cpu() if torch.is_tensor(x) else x for x in r) for r in want])
