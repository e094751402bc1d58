"""GPU tests of online stream previews (`OnlineStreams.push(sid, chunk, preview=True)`).  The hub meets the reference
golden of oracle/make_preview_golden.py (a deep copy of the reference predictor called on the chunk [w, f]).  A preview
equals forking the stream (snapshot, restore into a second hub) and pushing the chunk there without the flag, for every
T a stream allows, before and after the first step, unbounded and bounded, with the support grid and after track
edits.  Previews change nothing: the commits of a hub with previews between them equal those of a hub without, and the
snapshot and the pool's support after a preview step equal those before it.  Streams that preview, commit or wait share
a step and give their own results, in one pass or in passes forced apart.  Each camera frame reaches the encoder once;
a frame replaced after a preview is encoded again.  And ct3_online_window_end / _end_scores with preview = 1 give the
outputs of preview = 0 and leave the history byte for byte."""
import pytest
import torch

from cases import compare, load_golden
from oracle import make_preview_golden as G

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
S, STEP = 16, 8
H, W = 96, 128


def _predictor(sd=None):
    from cotracker_b200.predictor import CoTrackerOnlinePredictor
    from cotracker_b200.synthetic import seeded_state_dict
    p = CoTrackerOnlinePredictor(checkpoint=None, window_len=S)
    p.model.load_state_dict(sd or seeded_state_dict(53, offline=False, window_len=S, head_gain=10.0, vis_gain=100.0))
    return p.to(DEV)


@pytest.fixture(scope="module")
def p():
    return _predictor()


def _video(T, seed, h=H, w=W):
    from cotracker_b200.synthetic import texture_video
    return texture_video(T, h, w, seed=seed, shift=(1 + seed % 3, 2)).to(DEV)


def _queries(n, t0, t1, seed, h=H, w=W):
    """[1,n,3] queries with frames in [t0, t1)."""
    g = torch.Generator().manual_seed(seed)
    t = torch.randint(t0, t1, (n,), generator=g).float()
    return torch.stack([t, torch.rand(n, generator=g) * (w - 1), torch.rand(n, generator=g) * (h - 1)], -1)[None].to(DEV)


def _hub(p):
    from cotracker_b200.streams import OnlineStreams
    return OnlineStreams(p)


def _start(length):
    """The window start of a stream of `length` frames: a chunk of frames [start, f] previews frame f."""
    return max(0, length - (S - STEP))


def _flat(r):
    return (r[0], r[1]) + ((r[2].visibility, r[2].confidence) if len(r) == 3 else ())


def _same(a, b, what):
    fa, fb = _flat(a), _flat(b)
    assert len(fa) == len(fb), what
    for x, y in zip(fa, fb):
        assert x.shape == y.shape and torch.equal(x, y), what


def _snap_equal(a, b, what):
    assert a.keys() == b.keys(), what
    for k in a:
        x, y = a[k], b[k]
        if k == "hist" and x is not None:
            assert len(x) == len(y) and all(torch.equal(u, v) for u, v in zip(x, y)), (what, k)
        elif torch.is_tensor(x):
            assert x.dtype == y.dtype and torch.equal(x, y), (what, k)
        else:
            assert x == y, (what, k)


def _edit(hub, sid, edits):
    for op, arg in edits:
        if op == "add":
            hub.add_tracks(sid, arg)
        else:
            hub.retire_tracks(sid, arg)


def test_hub_meets_the_reference_golden():
    sd, video, queries = G.case_inputs()
    golden = load_golden(G.NAME)
    hub = _hub(_predictor(sd))
    video = video.to(DEV)
    other = hub.open(frame_size=(80, 96), grid_size=3)          # an unrelated stream sharing every step
    ov = _video(G.CASE["T"], 7, 80, 96)
    sid = hub.open(frame_size=tuple(video.shape[3:]), queries=queries.to(DEV))
    got, worst = {}, 0.0
    for kind, x in G.PLAN:
        length = hub.length(sid)
        if kind == "c":
            hub.push(sid, video[:, STEP * x:STEP * x + S])
        else:
            hub.push(sid, video[:, _start(length):x + 1], preview=True)
        olen = hub.length(other)
        if olen + STEP <= G.CASE["T"] - S:
            hub.push(other, ov[:, _start(olen):_start(olen) + S])
        tr, vi, sc = hub.step(return_scores=True)[sid]
        name = G.entry_name(kind, x)
        assert tr.shape[1] == (x + 1 if kind == "p" else STEP * x + S) and hub.length(sid) == (
            length if kind == "p" else STEP * x + S)
        got[f"tracks_{name}"], got[f"visibility_{name}"] = tr.cpu(), vi.cpu()
        n = tr.shape[2]
        for mine, key in ((sc.visibility, "prob_vis_"), (sc.confidence, "prob_conf_")):
            worst = max(worst, float((mine.cpu() - golden[key + name][..., :n]).abs().max()))
    assert set(got) == {k for k in golden if not k.startswith("prob_")}
    print(compare(got, golden, tol_px=1e-3), f"max |P - P_ref| = {worst:.2e}")
    assert worst <= 2e-4


def _fork_configs():
    return dict(grid=dict(kw=dict(grid_size=4), video=_video(48, 31), edits={}),
                h5=dict(kw=dict(grid_size=4, history=5), video=_video(48, 32), edits={}),
                sgrid=dict(kw=dict(queries=_queries(6, 0, 40, 12), add_support_grid=True), video=_video(48, 33),
                           edits={}),
                edits=dict(kw=dict(grid_size=3), video=_video(48, 34),
                           edits={0: [("add", _queries(2, 0, 20, 4))], 2: [("add", _queries(3, 24, 40, 5))],
                                  3: [("retire", [1, 10])]}))


def test_a_preview_equals_a_fork_that_steps(p):
    """For every T a stream allows at lengths 0, 16, 24 and 32: the preview's result is torch.equal to that of the
    stream restored from its snapshot into a second hub and pushed the chunk without the flag, and the stream's
    snapshot after the preview step equals the one before."""
    cfg = _fork_configs()
    hub = _hub(p)
    sids = {n: hub.open(frame_size=(H, W), **c["kw"]) for n, c in cfg.items()}
    for k in range(4):
        for n, c in cfg.items():
            _edit(hub, sids[n], c["edits"].get(k, ()))
        snaps = {n: hub.snapshot(sids[n]) for n in cfg}
        length = hub.length(sids["grid"])
        w = _start(length)
        for T in range(length - w + 1, S + 1):
            for n, c in cfg.items():
                hub.push(sids[n], c["video"][:, w:w + T], preview=True)
            got = hub.step(return_scores=True)
            twin = _hub(p)
            tids = {n: twin.restore(snaps[n]) for n in cfg}
            for n, c in cfg.items():
                twin.push(tids[n], c["video"][:, w:w + T])
            want = twin.step(return_scores=True)
            for n in cfg:
                _same(got[sids[n]], want[tids[n]], (n, k, T))
                assert got[sids[n]][0].shape[1] == (min(5, w + T) if n == "h5" else w + T)
                _snap_equal(hub.snapshot(sids[n]), snaps[n], (n, k, T))
            assert not hub._pending and not hub._previews
        for n, c in cfg.items():
            hub.push(sids[n], c["video"][:, STEP * k:STEP * k + S])
        hub.step()


def test_previews_change_nothing(p):
    """A preview at every frame (two at some), a commit every 8 frames: each commit equals that of a hub fed the
    commits only; after each preview step the snapshots and the whole pool's support are as before it."""
    specs = dict(a=dict(kw=dict(queries=torch.cat([_queries(8, 0, 1, 21), _queries(8, 4, 44, 22)], 1))),
                 b=dict(kw=dict(queries=_queries(6, 0, 40, 23), add_support_grid=True, history=5)),
                 c=dict(kw=dict(grid_size=3)))
    for k, sp in enumerate(specs.values()):
        sp["video"] = _video(56, 40 + k)
    P, Q = _hub(p), _hub(p)
    ps = {n: P.open(frame_size=(H, W), **sp["kw"]) for n, sp in specs.items()}
    qs = {n: Q.open(frame_size=(H, W), **sp["kw"]) for n, sp in specs.items()}
    commits = 0
    for f in range(56):
        w = _start(P.length(ps["a"]))
        if f + 1 == w + S:
            for n, sp in specs.items():
                P.push(ps[n], sp["video"][:, w:f + 1])
                Q.push(qs[n], sp["video"][:, w:f + 1])
            got, want = P.step(return_scores=True), Q.step(return_scores=True)
            for n in specs:
                _same(got[ps[n]], want[qs[n]], (n, f))
            commits += 1
            continue
        for again in range(2 if f % 5 == 2 and f > P.length(ps["a"]) else 1):   # then also frame f - 1 again
            before = {n: P.snapshot(ps[n]) for n in specs}
            support = P.pool.support.clone()
            for n in "ab":
                P.push(ps[n], specs[n]["video"][:, w:f + 1 - again], preview=True)
            out = P.step()
            assert set(out) == {ps["a"], ps["b"]}
            assert torch.equal(P.pool.support.view(torch.int32), support.view(torch.int32)), f
            for n in specs:
                _snap_equal(P.snapshot(ps[n]), before[n], (n, f))
    assert commits == 6


@pytest.mark.parametrize("split", [False, True])
def test_previews_commits_and_idle_streams_share_a_step(p, split, monkeypatch):
    """In one step: a stream previews after two windows, one previews before its first, one commits and one does not
    push.  Each result equals that stream's own, alone on a hub restored from its snapshot; the streams that did not
    commit keep their snapshots.  With split=True every stream gets its own pass."""
    import cotracker_b200.model as M
    specs = dict(pre=dict(kw=dict(grid_size=4), hw=(H, W), T=12),
                 first=dict(kw=dict(queries=_queries(5, 0, 12, 3, 80, 96), add_support_grid=True), hw=(80, 96), T=5,
                            late=True),
                 com=dict(kw=dict(grid_size=5, history=6), hw=(80, 96), T=S),
                 idle=dict(kw=dict(grid_size=3), hw=(H, W), T=None))
    for k, sp in enumerate(specs.values()):
        sp["video"] = _video(40, 50 + k, *sp["hw"])
    if split:
        passes, plan = [], M.plan_clip_passes
        monkeypatch.setattr(M, "pass_budget_bytes", lambda *a, **k: 1)
        monkeypatch.setattr(M, "plan_clip_passes", lambda *a, **k: passes.append(plan(*a, **k)) or passes[-1])
    hub = _hub(p)
    sids = {n: hub.open(frame_size=sp["hw"], **sp["kw"]) for n, sp in specs.items()}
    for k in range(2):
        for n, sp in specs.items():
            if not sp.get("late"):
                hub.push(sids[n], sp["video"][:, STEP * k:STEP * k + S])
        hub.step()
    snaps = {n: hub.snapshot(sids[n]) for n in specs}
    chunks = {}
    for n, sp in specs.items():
        if sp["T"] is not None:
            w = _start(hub.length(sids[n]))
            chunks[n] = sp["video"][:, w:w + sp["T"]]
            hub.push(sids[n], chunks[n], preview=n != "com")
    got = hub.step(return_scores=True)
    assert set(got) == {sids[n] for n in chunks}
    if split:
        assert passes and len(passes[-1]) == 3
    monkeypatch.undo()
    for n, chunk in chunks.items():
        solo = _hub(p)
        t = solo.restore(snaps[n])
        solo.push(t, chunk)
        _same(got[sids[n]], solo.step(return_scores=True)[t], n)
    for n in ("pre", "first", "idle"):
        _snap_equal(hub.snapshot(sids[n]), snaps[n], n)
    assert hub.length(sids["com"]) == 3 * STEP + S - STEP


def test_each_frame_is_encoded_once(p, monkeypatch):
    """A preview at every frame and a commit every 8 frames: each frame of the stream reaches the encoder once (the
    padding of a short preview none).  A previewed frame replaced by another is encoded again, and the results still
    equal a fork's and, at the commits, a hub's without previews."""
    log = []
    encode = p.model._encode
    monkeypatch.setattr(p.model, "_encode", lambda video, chunk: log.append(video.shape[0]) or encode(video, chunk))
    video, other = _video(48, 61), _video(48, 62)
    P, Q = _hub(p), _hub(p)
    sid, qid = P.open(frame_size=(H, W), grid_size=4), Q.open(frame_size=(H, W), grid_size=4)
    per_step = []

    def step(hub):
        n0 = sum(log)
        out = hub.step(return_scores=True)
        return out, sum(log) - n0

    for f in range(48):
        w = _start(P.length(sid))
        if f + 1 == w + S:
            P.push(sid, video[:, w:f + 1])
            Q.push(qid, video[:, w:f + 1])
            got, n = step(P)
            want, _ = step(Q)
            _same(got[sid], want[qid], f)
        else:
            P.push(sid, video[:, w:f + 1], preview=True)
            got, n = step(P)
        per_step.append(n)
    assert sum(per_step) == 48 and all(n == 1 for n in per_step), per_step
    # after the commit at f = 47 (window start 40), on a stream restored from a snapshot: previews of 48..50, then 50
    # with frame 49 replaced, then 50 with the real frame 49 again, then 51
    snap = P.snapshot(sid)
    F = _hub(p)
    fid = F.restore(snap)
    clip = torch.cat([video, _video(16, 63)], 1)
    w = _start(F.length(fid))
    assert w == 40
    counts = []
    for f, swap in ((48, False), (49, False), (50, False), (50, True), (50, False), (51, False)):
        chunk = clip[:, w:f + 1].clone()
        if swap:
            chunk[:, 49 - w] = other[:, 9]
        F.push(fid, chunk, preview=True)
        got, n = step(F)
        counts.append(n)
        fork = _hub(p)
        t = fork.restore(snap)
        fork.push(t, chunk)
        _same(got[fid], fork.step(return_scores=True)[t], (f, swap))
    # the first preview after the restore encodes the overlap too; then one frame each, the swapped frame and the real
    # one again once each
    assert counts == [S - STEP + 1, 1, 1, 1, 1, 1], counts


def test_window_end_preview_leaves_the_history_and_matches(p):
    """ct3_online_window_end and _end_scores with preview = 1 against preview = 0 on copies: the outputs (tracks,
    visibility, scores) are torch.equal, and the previewed histories byte-identical before and after.  Three streams:
    a plain history with an output from before the window, a ring, and a stream at ind = 0 whose preview entry has no
    history at all."""
    from cotracker_b200 import engine
    g = torch.Generator(device=DEV).manual_seed(5)
    # (n, n_keep, ring, cap, length, ind, T, out_first)
    cfg = [(5, 4, False, 40, 24, 16, 12, 3), (7, 7, True, 24, 40, 32, 16, 28), (3, 2, False, 16, 0, 0, 9, 0)]
    N = sum(c[0] for c in cfg)
    coords = torch.randn(S, N, 2, device=DEV, generator=g) * 30
    vis = torch.randn(S, N, device=DEV, generator=g) * 4
    conf = torch.randn(S, N, device=DEV, generator=g) * 4
    hists = [tuple(torch.randn(cap, n, *s, device=DEV, generator=g) * 20 for s in ((2,), (), ()))
             for n, _, _, cap, _, _, _, _ in cfg]
    for scores in (False, True):
        res = {}
        for preview in (0, 1):
            entries, outs, probs, first = [], [], [], 0
            hist = [tuple(t.clone() for t in h) for h in hists]
            for k, ((n, n_keep, ring, cap, length, ind, T, out_first), h) in enumerate(zip(cfg, hist)):
                rows = ind + T - out_first
                out = (torch.full((rows, n_keep, 2), -7.0, device=DEV),
                       torch.full((rows, n_keep), 3, dtype=torch.uint8, device=DEV))
                outs.append(out)
                probs.append((torch.full((rows, n_keep), -1.0, device=DEV), torch.full((rows, n_keep), -1.0,
                                                                                       device=DEV)))
                bare = preview and ind == 0
                entries.append(engine.online_stream(None if bare else h, length, ind, T, first, 0, out, n_keep,
                                                    (0.75, 1.25), out_first=out_first, ring=ring,
                                                    preview=bool(preview), n=n))
                first += n
            engine.online_window_end(entries, S, 4, coords, vis, conf, scores=probs if scores else None)
            torch.cuda.synchronize()
            res[preview] = (outs, probs, hist)
            if preview:
                for h, h0 in zip(hist, hists):
                    for a, b in zip(h, h0):
                        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
            else:
                assert not torch.equal(hist[0][1], hists[0][1])        # a commit writes its window
        for k in range(len(cfg)):
            for a, b in zip(res[0][0][k], res[1][0][k]):
                assert torch.equal(a, b), (scores, k)
            if scores:
                for a, b in zip(res[0][1][k], res[1][1][k]):
                    assert torch.equal(a, b) and bool((a >= 0).all()), (scores, k)
