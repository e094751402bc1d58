"""CPU tests of track edits in online streams (`OnlineStreams.add_tracks` / `retire_tracks` / `track_ids`): every
rejection happens before any state changes, the pool and history surgery of `StreamPool.edit` on CPU tensors (plain and
ring histories), the ids a stream reports, and the in-repo oracle with the same surgery against the reference golden
`online_track_edits.npz` (oracle/make_track_edit_golden.py)."""
import pytest
import torch

from cases import O, compare, load_golden
from cotracker_b200.model import StreamPool
from oracle import make_track_edit_golden as G

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


def _snapshot(hub):
    pool = hub.pool
    return ([t.clone() for t in (pool.support, pool.qframes, pool.qcoords)],
            [(s.first, s.n, None if s.hist is None else [h.clone() for h in s.hist]) for s in pool.streams],
            {k: (v["out"], list(v["ids"]), v["next_id"]) for k, v in hub._streams.items()})


def _same(a, b):
    (ta, sa, da), (tb, sb, db) = a, b
    assert all(torch.equal(x, y) for x, y in zip(ta, tb)) and da == db
    for (fa, na, ha), (fb, nb, hb) in zip(sa, sb):
        assert (fa, na) == (fb, nb) and (ha is None) == (hb is None)
        assert ha is None or all(torch.equal(x, y) for x, y in zip(ha, hb))


def test_every_rejection_happens_before_any_state_change():
    hub = _hub()
    _register(hub, 0, 5, 5, length=24)
    _register(hub, 1, 42, 6, history=5, length=40, seed=1)                # 6 user tracks and a 36-point support grid
    _register(hub, 2, 3, 3, seed=2)                                         # not advanced yet
    before = _snapshot(hub)
    q = torch.tensor([[[40.0, 3.0, 4.0], [39.0, 5.0, 6.0]]])
    with pytest.raises(ValueError, match="query frames must be >= 40"):     # 39 is below the stream's length
        hub.add_tracks(1, q)
    with pytest.raises(ValueError, match=">= 24"):
        hub.add_tracks(0, torch.tensor([[[23.5, 1.0, 1.0]]]))
    with pytest.raises(ValueError, match=">= 0"):
        hub.add_tracks(2, torch.tensor([[[-1.0, 1.0, 1.0]]]))
    with pytest.raises(ValueError, match=">= 24"):
        hub.add_tracks(0, torch.tensor([[[float("nan"), 1.0, 1.0]]]))
    for bad in (torch.zeros(2, 1, 3) + 50, torch.zeros(1, 0, 3), torch.zeros(1, 2, 2) + 50, torch.zeros(3) + 50):
        with pytest.raises(ValueError, match=r"\[1,m,3\]"):
            hub.add_tracks(0, bad)
    for call in (lambda: hub.add_tracks(7, q), lambda: hub.retire_tracks(7, [0]), lambda: hub.track_ids(7)):
        with pytest.raises(KeyError):
            call()
    for ids, match in (([6], "no track 6"), ([10], "no track 10"), ([41], "no track"), ([-1], "no track"),
                       ([0, 2, 0], "duplicates"), ([True], "no track"), ([1.0], "no track"),
                       ([0, 1, 2, 3, 4, 5], "close it")):
        with pytest.raises(ValueError, match=match):                         # 6..41: support-grid columns
            hub.retire_tracks(1, ids)
    with pytest.raises(ValueError, match="close it"):
        hub.retire_tracks(2, torch.tensor([2, 0, 1]))
    _same(before, _snapshot(hub))
    hub.retire_tracks(1, [4])
    with pytest.raises(ValueError, match="no track 4"):                     # already retired
        hub.retire_tracks(1, [4])


def _pool_of_three(history):
    hub = _hub()
    states = [_register(hub, 0, 7, 7, length=32, seed=3), _register(hub, 1, 40, 4, history=history, length=48, seed=4),
              _register(hub, 2, 5, 5, history=9, length=24, seed=5)]
    return hub, states


@pytest.mark.parametrize("history", [None, 1, 30])
def test_pool_and_history_surgery(history):
    """Edit the middle stream: 4 user tracks and 36 support-grid points; retire user columns 0 and 2, add 3."""
    hub, (s0, s1, s2) = _pool_of_three(history)
    pool = hub.pool
    sup, qf, qc = pool.support.clone(), pool.qframes.clone(), pool.qcoords.clone()
    hist = [[h.clone() for h in s.hist] for s in (s0, s1, s2)]
    a, b = s1.first, s1.first + s1.n
    cap = s1.hist[1].shape[0]
    new_qf = torch.tensor([48, 50, 70], dtype=torch.int32)
    new_qc = torch.tensor([[1.25, 2.5], [10.0, 0.0], [127.75, 95.5]])
    keep = [1, 3] + list(range(4, 40))
    pool.edit(s1, keep, 2, new_qf, new_qc, STRIDE)
    assert (s0.first, s0.n, s1.first, s1.n, s2.first, s2.n) == (0, 7, 7, 41, 48, 5)
    assert pool.support.shape == (4, 49, 53, 128)
    # other streams: rows and histories intact, the following one shifted
    for (x, y) in ((pool.support[:, :, :a], sup[:, :, :a]), (pool.support[:, :, 48:], sup[:, :, b:]),
                   (pool.qframes[:a], qf[:a]), (pool.qframes[48:], qf[b:]), (pool.qcoords[48:], qc[b:])):
        assert torch.equal(x, y)
    for s, h in ((s0, hist[0]), (s2, hist[2])):
        assert all(torch.equal(x, y) for x, y in zip(s.hist, h))
    # the edited stream: kept columns bit-equal, new ones in place 2..4 with the placeholder
    cols = [0, 1] + list(range(5, 41))
    src = torch.tensor(keep) + a
    assert torch.equal(pool.support[:, :, a + torch.tensor(cols)], sup[:, :, src])
    assert torch.equal(pool.qframes[a + torch.tensor(cols)], qf[src])
    assert torch.equal(pool.qcoords[a + torch.tensor(cols)], qc[src])
    assert not pool.support[:, :, a + 2:a + 5].any()
    assert torch.equal(pool.qframes[a + 2:a + 5], new_qf) and torch.equal(pool.qcoords[a + 2:a + 5], new_qc)
    assert s1.hist[1].shape[0] == cap and s1.hist[0].shape == (cap, 41, 2)
    for x, y in zip(s1.hist, hist[1]):
        assert torch.equal(x[:, cols], y[:, keep])
    rows = cap if history is not None else s1.length                        # every row a ring holds; frames so far
    assert torch.equal(s1.hist[0][:rows, 2:5], (new_qc * STRIDE)[None].expand(rows, 3, 2))
    assert not s1.hist[1][:rows, 2:5].any() and not s1.hist[2][:rows, 2:5].any()
    assert all(h.is_contiguous() for h in s1.hist) and pool.qframes.is_contiguous()
    # retire-only, add-only, and a stream not advanced yet (no history)
    pool.edit(s0, [6, 0], 2, new_qf[:0], new_qc[:0], STRIDE)
    assert (s0.n, s1.first, s2.first) == (2, 2, 43) and torch.equal(pool.qframes[:2], qf[torch.tensor([6, 0])])
    fresh = pool.open(torch.zeros(2, dtype=torch.int32), torch.zeros(2, 2))
    pool.edit(fresh, [0, 1], 2, new_qf, new_qc, STRIDE)
    assert fresh.hist is None and fresh.n == 5 and pool.qframes.shape[0] == 53


def test_track_ids_follow_edits():
    hub = _hub()
    state = _register(hub, 3, 40, 4, length=24)                             # 4 user tracks and a support grid
    qf = hub.pool.qframes.clone()
    assert hub.track_ids(3) == [0, 1, 2, 3]
    q = torch.tensor([[[24.0, 10.0, 20.0], [30.0, 0.0, 95.0]]])
    assert hub.add_tracks(3, q) == [4, 5]
    assert hub.track_ids(3) == [0, 1, 2, 3, 4, 5] and hub._streams[3]["out"][0] == 6 and state.n == 42
    assert hub.pool.qframes[4:6].tolist() == [24, 30] and torch.equal(hub.pool.qframes[6:], qf[4:])
    # frame pixels of a 96x128 stream -> model resolution 384x512 -> feature-grid units
    want = q[0, :, 1:] * torch.tensor([511 / 127, 383 / 95]) / STRIDE
    assert torch.equal(hub.pool.qcoords[4:6], want)
    hub.retire_tracks(3, [1, 4])
    assert hub.track_ids(3) == [0, 2, 3, 5] and hub._streams[3]["out"][0] == 4 and state.n == 40
    assert hub.add_tracks(3, torch.tensor([[[24.0, 1.0, 1.0]]])) == [6]      # ids are never reused
    hub.retire_tracks(3, [0, 2, 3, 5])
    assert hub.track_ids(3) == [6] and hub.pool.qframes[0].item() == 24
    ids = hub.track_ids(3)
    ids.append(99)                                                          # a copy
    assert hub.track_ids(3) == [6]


def _scaled(adds, H, W):
    return G.scale_queries(G.edit_queries(adds), H, W, G.CASE["interp_shape"])


def _edit_oracle(st, ids, next_id, retire, adds, H, W):
    """The edit of the oracle's online predictor state, as oracle/make_track_edit_golden.py edits the reference's."""
    q = _scaled(adds, H, W) if adds else torch.zeros(1, 0, 3)
    m = q.shape[1]
    keep, at, ids, next_id = G.plan_edit(ids, st.queries.shape[1], retire, m, next_id)
    st.queries, st.N = G.columns(st.queries, 1, keep, at, q), at + m
    ms = st.model
    if ms.coords is not None:
        ms.support = [G.columns(s, 1, keep, at, s.new_zeros(s.shape[0], m, s.shape[2])) for s in ms.support]
        T = ms.coords.shape[0]
        ms.coords = G.columns(ms.coords, 1, keep, at, (q[0, :, 1:3] / O.STRIDE * O.STRIDE)[None].expand(T, m, 2))
        ms.vis = G.columns(ms.vis, 1, keep, at, torch.zeros(T, m))
        ms.conf = G.columns(ms.conf, 1, keep, at, torch.zeros(T, m))
    return ids, next_id


def test_oracle_with_the_same_surgery_meets_the_reference_golden():
    sd, streams = G.case_inputs()
    golden = load_golden(G.NAME)
    got = {}
    with torch.no_grad():
        for s, (video, kw) in streams.items():
            st = O.OnlinePredictorState()
            H, W = video.shape[3:]
            O.predict_online(sd, st, video[:, :1], is_first_step=True, window_len=S, **kw)
            ids, next_id = list(range(st.N)), st.N
            for k in range(G.CASE["steps"]):
                if k in G.EDITS[s]:
                    ids, next_id = _edit_oracle(st, ids, next_id, *G.EDITS[s][k], H, W)
                tr, vi = O.predict_online(sd, st, video[:, STEP * k:STEP * k + S], window_len=S,
                                          add_support_grid=kw["add_support_grid"])
                got[f"tracks{k}_{s}"], got[f"visibility{k}_{s}"] = tr, vi
                assert tr.shape[2] == len(ids)
    assert set(got) == {k for k in golden if not k.startswith("prob_")}
    print(compare(got, golden, tol_px=1e-3))
    # the fixture shows what the contract says: an added track reads as its query point, not visible, before the
    # window it was added at (stream a, added at length 24: window start 16), and comes from the model from there on
    tr, vi = golden["tracks2_a"], golden["visibility2_a"]
    q = _scaled(G.EDITS["a"][2][1], 160, 224)[0]
    pt = q[:, 1:] * torch.tensor([223 / 511, 159 / 383])
    assert torch.equal(tr[0, :16, 18:22], pt[None].expand(16, 4, 2)) and not vi[0, :16, 18:22].any()
    assert all(not torch.equal(tr[0, t, 18:20], pt[:2]) for t in range(16, 32))
