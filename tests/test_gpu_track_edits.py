"""GPU tests of track edits in online streams (`OnlineStreams.add_tracks` / `retire_tracks`): the hub meets the
reference golden of oracle/make_track_edit_golden.py; edits before the first step equal opening with the edited
queries, and an add undone in the same gap equals no edit, bit for bit; an edited stream's results do not depend on
the other streams or on how a step is split into passes; the frames before the next window keep their values across
an edit and added tracks read as their query point there; a bounded stream with edits is the tail of the unbounded
one; and a bounded stream that keeps replacing its tracks stops raising the device memory peak."""
import pytest
import torch

from cases import compare, load_golden
from oracle import make_track_edit_golden as G

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
S, STEP = 16, 8


def _predictor(sd=None):
    from cotracker_b200.predictor import CoTrackerOnlinePredictor
    from cotracker_b200.synthetic import seeded_state_dict
    p = CoTrackerOnlinePredictor(checkpoint=None, window_len=S)
    p.model.load_state_dict(sd or seeded_state_dict(53, offline=False, window_len=S, head_gain=10.0, vis_gain=100.0))
    return p.to(DEV)


def _video(T, h, w, seed):
    from cotracker_b200.synthetic import texture_video
    return texture_video(T, h, w, seed=seed, shift=(1 + seed % 3, 2)).to(DEV)


def _queries(n, t0, t1, h, w, seed):
    """[1,n,3] queries with frames in [t0, t1)."""
    g = torch.Generator().manual_seed(seed)
    t = torch.randint(t0, t1, (n,), generator=g).float()
    return torch.stack([t, torch.rand(n, generator=g) * (w - 1), torch.rand(n, generator=g) * (h - 1)], -1)[None].to(DEV)


def _spec(video, edits=None, open_at=0, close_after=None, skip=(), **kw):
    """A stream of a run: its frames, open() arguments, and edits {step: [("add", queries) | ("retire", ids)]} made
    in the gap before that step."""
    return dict(video=video, kw=kw, edits=edits or {}, open_at=open_at, close_after=close_after, skip=set(skip))


def _run(p, specs, steps):
    """-> {name: {step: (tracks, visibility, track_ids, length)}} of the steps that advanced each stream."""
    from cotracker_b200.streams import OnlineStreams
    hub = OnlineStreams(p)
    sid, pos, res = {}, {}, {n: {} for n in specs}
    for k in range(steps):
        for n, sp in specs.items():
            if sp["open_at"] == k:
                sid[n], pos[n] = hub.open(frame_size=tuple(sp["video"].shape[3:]), **sp["kw"]), 0
            if n not in sid:
                continue
            for op, arg in sp["edits"].get(k, ()):
                if op == "add":
                    hub.add_tracks(sid[n], arg)
                else:
                    hub.retire_tracks(sid[n], arg)
            if k not in sp["skip"]:
                hub.push(sid[n], sp["video"][:, STEP * pos[n]:STEP * pos[n] + S])
                pos[n] += 1
        out = hub.step()
        for n in list(sid):
            if sid[n] in out:
                tr, vi = out[sid[n]]
                assert tr.shape[2] == vi.shape[2] == len(hub.track_ids(sid[n]))
                res[n][k] = (tr, vi, hub.track_ids(sid[n]), hub.length(sid[n]))
            if specs[n]["close_after"] == k:
                hub.close(sid.pop(n))
    return res


def _equal(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert torch.equal(a[k][0], b[k][0]) and torch.equal(a[k][1], b[k][1]) and a[k][2:] == b[k][2:], k


def test_hub_meets_the_reference_golden():
    sd, streams = G.case_inputs()
    specs = {}
    for s, (video, kw) in streams.items():
        kw = {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in kw.items()}
        edits = {k: ([("retire", r)] if r else []) + ([("add", G.edit_queries(a))] if a else [])
                 for k, (r, a) in G.EDITS[s].items()}
        specs[s] = _spec(video.to(DEV), edits, **kw)
    specs["other"] = _spec(_video(80, 80, 96, 9), {1: [("add", _queries(3, 16, 40, 80, 96, 1))]}, grid_size=3)
    res = _run(_predictor(sd), specs, G.CASE["steps"])
    golden = load_golden(G.NAME)
    got = {}
    for s in streams:
        for k, (tr, vi, _, _) in res[s].items():
            got[f"tracks{k}_{s}"], got[f"visibility{k}_{s}"] = tr.cpu(), vi.cpu()
    assert set(got) == {k for k in golden if not k.startswith("prob_")}
    print(compare(got, golden, tol_px=1e-3))
    assert res["a"][5][2] == [2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 20, 22, 23]
    assert res["b"][5][2] == [2, 3, 4, 5, 6, 8]


def test_edits_before_the_first_step_and_an_undone_add_are_bitwise_no_ops():
    """Adding before the first step equals opening with the concatenated queries (also with the support grid),
    retiring before it equals opening without those tracks, and an add retired in the same gap equals no edit."""
    v = [_video(6 * STEP + S, 96, 128, 60 + k) for k in range(4)]
    q1, q2 = _queries(6, 0, 40, 96, 128, 1), _queries(3, 0, 40, 96, 128, 2)
    q3 = _queries(7, 0, 30, 96, 128, 3)
    late = _queries(2, 24, 60, 96, 128, 4)                                   # query frames >= length 24 at step 2
    edited = dict(e=_spec(v[0], {0: [("add", q2)]}, queries=q1),
                  s=_spec(v[1], {0: [("add", q2)]}, queries=q1, add_support_grid=True),
                  r=_spec(v[2], {0: [("retire", [1, 4])]}, queries=q3),
                  n=_spec(v[3], {2: [("add", late), ("retire", [16, 17])]}, grid_size=4))
    plain = dict(e=_spec(v[0], queries=torch.cat([q1, q2], 1)),
                 s=_spec(v[1], queries=torch.cat([q1, q2], 1), add_support_grid=True),
                 r=_spec(v[2], queries=q3[:, [0, 2, 3, 5, 6]]),
                 n=_spec(v[3], grid_size=4))
    p = _predictor()
    got, want = _run(p, edited, 6), _run(p, plain, 6)
    for n in "esr":
        for k in want[n]:
            want[n][k] = want[n][k][:2] + (got[n][k][2],) + want[n][k][3:]   # the ids differ where columns do not
        _equal(got[n], want[n])
    _equal(got["n"], want["n"])
    assert got["e"][0][2] == list(range(9)) and got["r"][0][2] == [0, 2, 3, 5, 6]


def _edited(video, h=None):
    """A grid stream with an add before the first step, adds entering one and two windows later, a retire of
    entered and of not yet entered tracks, and a retire and an add in one gap."""
    H, W = video.shape[3:]
    return _spec(video, {0: [("add", _queries(2, 0, 8, H, W, 10))],
                         2: [("add", _queries(4, 24, 40, H, W, 11)), ("add", _queries(1, 50, 56, H, W, 12))],
                         3: [("retire", [3, 25, 22])],
                         4: [("retire", [0, 31]), ("add", _queries(3, 40, 48, H, W, 13))],
                         6: [("retire", [1, 2, 4, 5]), ("add", _queries(2, 56, 70, H, W, 14))]},
                 grid_size=5, history=h)


def _crowded(v):
    H, W = 80, 96
    return dict(e=_edited(v[0]),
                f=_spec(v[1], {2: [("add", _queries(5, 24, 33, H, W, 20))], 3: [("retire", [1, 9, 13])],
                               4: [("retire", [0]), ("add", _queries(2, 40, 41, H, W, 21))]},
                        queries=_queries(9, 0, 20, H, W, 22), add_support_grid=True),
                c=_spec(v[2], grid_size=3, close_after=1),
                d=_spec(v[3], {4: [("add", _queries(2, 24, 40, H, W, 23))], 5: [("retire", [0])]}, open_at=2,
                        skip=(5,), grid_size=4),
                b=_spec(v[4], {3: [("retire", [0, 1])]}, grid_size=3, history=5))


def test_edited_stream_is_independent_of_other_streams_and_of_the_pass_split(monkeypatch):
    import cotracker_b200.model as M
    steps = 8
    v = [_video(STEP * steps + S, 96, 128, 70)] + [_video(STEP * steps + S, 80, 96, 71 + k) for k in range(4)]
    p = _predictor()
    alone = _run(p, dict(e=_edited(v[0])), steps)["e"]
    crowded = _run(p, _crowded(v), steps)
    passes = []
    planner = M.plan_clip_passes
    monkeypatch.setattr(M, "pass_budget_bytes", lambda *a, **k: 1)
    monkeypatch.setattr(M, "plan_clip_passes", lambda *a, **k: passes.append(planner(*a, **k)) or passes[-1])
    split = _run(p, _crowded(v), steps)
    assert passes and all(b1 - b0 == 1 for pl in passes for b0, b1 in pl)   # one stream per pass
    _equal(alone, crowded["e"])
    _equal(alone, split["e"])
    for n in crowded:
        _equal(crowded[n], split[n])


def _scaled_point(q, H, W):
    """Where the hub reports a track before its first window: its query point through the model's resolution and
    feature grid and back to the frame."""
    iw, ih = 512, 384
    m = q[0, :, 1:] * q.new_tensor([(iw - 1) / (W - 1), (ih - 1) / (H - 1)])
    return (m / 4 * 4) * q.new_tensor([(W - 1) / (iw - 1), (H - 1) / (ih - 1)])


def test_frames_before_the_next_window_survive_an_edit():
    """In an unbounded stream, across each edit: kept tracks' frames before the next window start equal the previous
    result bit for bit, and added tracks read as their scaled query point, not visible."""
    steps = 8
    video = _video(STEP * steps + S, 96, 128, 80)
    spec = _edited(video)
    res = _run(_predictor(), dict(e=spec), steps)["e"]
    checked = n_added = 0
    for k, ops in spec["edits"].items():
        if k == 0:
            continue
        tr0, vi0, ids0, length0 = res[k - 1]
        tr, vi, ids, _ = res[k]
        ind = length0 - (S - STEP)                                          # the window start of step k
        new = [i for i in ids if i not in ids0]                            # ids in the order of the adds
        pts = [_scaled_point(arg, 96, 128) for op, arg in ops if op == "add"]
        added = dict(zip(new, torch.cat(pts))) if pts else {}
        assert len(added) == len(new)
        n_added += len(added)
        for c, i in enumerate(ids):
            if i in added:
                assert torch.equal(tr[0, :ind, c], added[i][None].expand(ind, 2)) and not vi[0, :ind, c].any()
            else:
                c0 = ids0.index(i)
                assert torch.equal(tr[0, :ind, c], tr0[0, :ind, c0]) and torch.equal(vi[0, :ind, c], vi0[0, :ind, c0])
            checked += 1
    assert checked > 60 and n_added == 10


def test_bounded_stream_with_edits_is_the_tail_of_the_unbounded_one():
    steps = 9
    video = _video(STEP * steps + S, 96, 128, 90)
    bounds = (1, 5, 8, 20, 100)
    specs = dict(full=_edited(video), **{f"h{h}": _edited(video, h) for h in bounds})
    res = _run(_predictor(), specs, steps)
    for k, (ftr, fvi, ids, length) in res["full"].items():
        for h in bounds:
            tr, vi, hids, hlen = res[f"h{h}"][k]
            L = min(h, length)
            assert (hids, hlen) == (ids, length) and tr.shape[1] == L
            assert torch.equal(tr, ftr[:, -L:]) and torch.equal(vi, fvi[:, -L:])


def test_churn_in_a_bounded_stream_stops_raising_the_memory_peak():
    """A bounded stream that retires its 20 oldest tracks and adds 20 every step, at a constant 200."""
    from cotracker_b200.streams import OnlineStreams
    hub = OnlineStreams(_predictor())
    base = _video(64, 64, 80, 100)
    loop = torch.cat([base, base[:, :S]], 1)                                 # frame f + 64 repeats frame f
    sid = hub.open(frame_size=(64, 80), queries=_queries(200, 0, 8, 64, 80, 101), history=12)
    seen = {}
    for i in range(1, 61):
        length = hub.length(sid)
        if i > 1:
            hub.retire_tracks(sid, hub.track_ids(sid)[:20])
            q = _queries(20, length, length + 24, 64, 80, 200 + i)
            hub.add_tracks(sid, q)
        hub.push(sid, loop[:, (STEP * (i - 1)) % 64:(STEP * (i - 1)) % 64 + S])
        out = hub.step()
        assert out[sid][0].shape[1:3] == (min(12, STEP * i + STEP), 200)
        del out
        if i == 10:
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
        if i in (20, 60):
            torch.cuda.synchronize()
            seen[i] = (torch.cuda.max_memory_allocated(), torch.cuda.memory_allocated())
    assert hub.track_ids(sid)[0] == 200 + 20 * 59 - 200 and len(hub.track_ids(sid)) == 200
    assert seen[20] == seen[60], seen
