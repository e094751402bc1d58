"""GPU tests of the probability outputs (`return_scores=True`):

- tracks and visibility are `torch.equal` with and without the flag, in every predictor mode and on a hub;
- the scores are `torch.equal` to ATen's sigmoid of the model's outputs passed through the predictor's backward merge,
  support-grid drop and frame selection (offline), or to the sigmoid of the stream's history (online);
- they agree with the bool: offline `visibility == (P_vis > 0.9)` off the query cells, online
  `visibility == (P_vis * P_conf > 0.6)` everywhere;
- they stay within a measured bound of the unmodified reference's probabilities stored in the predictor goldens;
- streams: bounded and unbounded streams of one hub each equal their own online predictor, added tracks read 0.5
  before their first window, and scores continue bit for bit across snapshot / close / restore."""
import pytest
import torch

from cases import CASES, case_inputs, load_golden, predictor_kwargs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
S = 16
# |scores - reference probabilities| over the predictor goldens that store them, measured on an H100 80GB HBM3 at
# 700 W: at most 1.11e-4 (c4_online_grid50's P_vis * P_conf), 7.9e-5 offline (the stress cases; 1.1e-6 at unit gains)
REFERENCE_TOL = 2e-4


def _offline(offline=True, seed=43):
    from cotracker_b200.predictor import CoTrackerPredictor
    from cotracker_b200.synthetic import seeded_state_dict
    W = 60 if offline else S
    p = CoTrackerPredictor(checkpoint=None, offline=offline, window_len=W)
    p.model.load_state_dict(seeded_state_dict(seed, offline=offline, window_len=W, head_gain=10.0, vis_gain=100.0))
    return p.to(DEV)


def _online(seed=47):
    from cotracker_b200.predictor import CoTrackerOnlinePredictor
    from cotracker_b200.synthetic import seeded_state_dict
    p = CoTrackerOnlinePredictor(checkpoint=None, window_len=S)
    p.model.load_state_dict(seeded_state_dict(seed, offline=False, window_len=S, head_gain=10.0, vis_gain=100.0))
    return p.to(DEV)


def _batch(B, T, N, h, w, seed=100):
    from cotracker_b200.synthetic import random_queries, texture_video
    video = torch.cat([texture_video(T, h, w, seed=seed + b, shift=(1 + b, 2)) for b in range(B)]).to(DEV)
    queries = torch.cat([random_queries(N, T, h, w, seed=seed + 50 + b) for b in range(B)]).to(DEV)
    return video, queries


# ---- offline: the merged, sliced model outputs ------------------------------------------------------------------
def _record_groups(monkeypatch, model):
    """Record every query group a predictor call tracks: (queries [B,n,3] at model resolution, reversed, clip id,
    (tracks, P_vis, P_conf)) -- the model's outputs, ATen sigmoids of its logits -- in call order."""
    import cotracker_b200.predictor as P
    rec = []
    track_groups = P._EncodedClip.track_groups

    def groups(self, gs, flags, scores=False):
        out = track_groups(self, gs, flags, scores)
        rec.extend((q, r, 0, o) for q, r, o in zip(gs, flags, out))
        return out

    monkeypatch.setattr(P._EncodedClip, "track_groups", groups)
    if hasattr(model, "_track_ragged"):   # list calls: the offline model only
        track_ragged = type(model)._track_ragged

        def ragged(self, pyr, H, W, gs, iters, scores=False):
            out = track_ragged(self, pyr, H, W, gs, iters, scores)
            rec.extend((q, r, f0, o) for (q, f0, _, r), o in zip(gs, out))
            return out

        monkeypatch.setattr(type(model), "_track_ragged", ragged)
    return rec


def _merge(fwd, bwd, qt):
    """The predictor's merge of probabilities [B,T,N]: the backward pass (reversed-clip time) where t < query frame."""
    if bwd is None:
        return fwd
    before = torch.arange(fwd.shape[1], device=fwd.device)[None, :, None] < qt[:, None, :]
    return torch.where(before, bwd.flip(1), fwd)


def _expected(rec, clip=0):
    """(P_vis, P_conf, query frames) of the recorded groups of one clip, merged and concatenated along N."""
    groups = [g for g in rec if g[2] == clip]
    vis, conf, qt = [], [], []
    for k, (q, rev, _, out) in enumerate(groups):
        if rev:
            continue
        bwd = groups[k + 1][3] if k + 1 < len(groups) and groups[k + 1][1] else None
        vis.append(_merge(out[1], None if bwd is None else bwd[1], q[:, :, 0]))
        conf.append(_merge(out[2], None if bwd is None else bwd[2], q[:, :, 0]))
        qt.append(q[:, :, 0])
    return torch.cat(vis, 2), torch.cat(conf, 2), torch.cat(qt, 1)


def _check_offline(tr, vi, sc, rec, clip=0):
    n = vi.shape[2]
    assert sc.visibility.dtype == sc.confidence.dtype == torch.float32
    assert sc.visibility.shape == sc.confidence.shape == vi.shape and sc.visibility.device == vi.device
    want_v, want_c, qt = _expected(rec, clip)
    assert torch.equal(sc.visibility, want_v[:, :, :n]) and torch.equal(sc.confidence, want_c[:, :, :n])
    pinned = torch.arange(vi.shape[1], device=DEV)[None, :, None] == qt[:, None, :n].long()
    assert bool(vi[pinned].all())
    assert torch.equal(vi[~pinned], (sc.visibility > 0.9)[~pinned])
    return int(pinned.sum())


MODES = {
    "queries": dict(queries=True),
    "queries_backward": dict(queries=True, backward_tracking=True),
    "grid": dict(grid_size=5),
    "grid_query_frame_backward": dict(grid_size=4, grid_query_frame=7, backward_tracking=True),
    "segm_mask": dict(grid_size=6, segm_mask=True),
    "batch3_queries_backward": dict(B=3, queries=True, backward_tracking=True),
    "batch3_grid": dict(B=3, grid_size=4),
}


@pytest.mark.parametrize("offline", [True, False])
@pytest.mark.parametrize("mode", list(MODES))
def test_offline_scores_are_the_merged_model_outputs(mode, offline, monkeypatch):
    p = _offline(offline)
    kw = dict(MODES[mode])
    B = kw.pop("B", 1)
    use_q = kw.pop("queries", False)
    T, h, w = 21, 144, 192
    video, queries = _batch(B, T, 7, h, w)
    if use_q:
        kw["queries"] = queries
    if kw.pop("segm_mask", False):
        from oracle.make_golden import box_mask
        kw["segm_mask"] = box_mask(h, w).to(DEV)
    rec = _record_groups(monkeypatch, p.model)
    with torch.no_grad():
        base = p(video, **kw)
        off = p(video, **kw, return_scores=False)
        rec.clear()
        tr, vi, sc = p(video, **kw, return_scores=True)
    assert len(base) == len(off) == 2
    for got in (base, off):
        assert torch.equal(got[0], tr) and torch.equal(got[1], vi)
    assert _check_offline(tr, vi, sc, rec) > 0


@pytest.mark.parametrize("backward", [False, True])
def test_dense_scores_are_the_merged_model_outputs(backward, monkeypatch):
    p = _offline(seed=93)
    video, _ = _batch(1, 8, 1, 96, 160)            # grid step 2: 4 offsets of 48 x 80 tracks
    gq = 5 if backward else 0
    rec = _record_groups(monkeypatch, p.model)
    with torch.no_grad():
        base = p(video, grid_query_frame=gq, backward_tracking=backward)
        rec.clear()
        tr, vi, sc = p(video, grid_query_frame=gq, backward_tracking=backward, return_scores=True)
    assert torch.equal(base[0], tr) and torch.equal(base[1], vi) and vi.shape == (1, 8, 48 * 80 * 4)
    assert len([g for g in rec if not g[1]]) == 4
    _check_offline(tr, vi, sc, rec)


@pytest.mark.parametrize("backward", [False, True])
def test_list_call_scores_are_the_merged_model_outputs(backward, monkeypatch):
    """Three ragged clips (lengths, sizes and query counts differ) in one call; a support grid on every clip."""
    from cotracker_b200.synthetic import random_queries, texture_video
    p = _offline(seed=47)
    shapes = [(9, 96, 128, 5), (17, 144, 192, 8), (12, 80, 112, 3)]
    clips = [texture_video(T, h, w, seed=10 + k, shift=(1 + k, 2)).to(DEV) for k, (T, h, w, _) in enumerate(shapes)]
    qs = [random_queries(n, T, h, w, seed=20 + k).to(DEV) for k, (T, h, w, n) in enumerate(shapes)]
    rec = _record_groups(monkeypatch, p.model)
    with torch.no_grad():
        base = p(clips, queries=qs, backward_tracking=backward)
        rec.clear()
        tr, vi, sc = p(clips, queries=qs, backward_tracking=backward, return_scores=True)
    assert isinstance(sc, list) and len(sc) == 3
    first = 0
    for b, (T, *_, n) in enumerate(shapes):
        assert torch.equal(base[0][b], tr[b]) and torch.equal(base[1][b], vi[b]) and vi[b].shape == (1, T, n)
        _check_offline(tr[b], vi[b], sc[b], rec, clip=first)
        first += T


# ---- online ------------------------------------------------------------------------------------------------------
def _sigmoid_rows(hist, frames, n_keep, cap=None):
    """ATen sigmoid of history logits [cap,n] at stream frames `frames` (ring rows f mod cap when cap is given)."""
    rows = frames if cap is None else frames % cap
    return torch.sigmoid(hist[rows.to(hist.device)][:, :n_keep])


@pytest.mark.parametrize("support", [False, True])
def test_online_predictor_scores_are_the_sigmoid_of_its_history(support):
    """B = 2 streams in lockstep: scores are sigmoid of the history logits, the bool is their product > 0.6, and
    tracks and visibility do not change with the flag."""
    p, q_ = _online(), _online()
    video, queries = _batch(2, 48, 6, 128, 160)
    first = dict(queries=queries, add_support_grid=True) if support else dict(grid_size=4)
    for pr in (p, q_):
        pr(video_chunk=video[:, :S], is_first_step=True, **first)
    with torch.no_grad():
        for k in range(5):
            chunk = video[:, 8 * k:8 * k + S]
            tr0, vi0 = q_(video_chunk=chunk, add_support_grid=support)
            tr, vi, sc = p(video_chunk=chunk, add_support_grid=support, return_scores=True)
            assert torch.equal(tr, tr0) and torch.equal(vi, vi0)
            n = vi.shape[2]
            assert sc.visibility.shape == sc.confidence.shape == vi.shape
            assert torch.equal(vi, sc.visibility * sc.confidence > 0.6)
            for b, st in enumerate(p.model._online_streams):
                f = torch.arange(st.length)
                assert torch.equal(sc.visibility[b], _sigmoid_rows(st.hist[1], f, n))
                assert torch.equal(sc.confidence[b], _sigmoid_rows(st.hist[2], f, n))


def test_hub_streams_equal_their_own_predictors():
    """Mixed bounded and unbounded streams on one hub (with a twin hub stepped without scores): each stream's scores
    equal its own CoTrackerOnlinePredictor(return_scores=True), a bounded stream's are the last L frames of those,
    the bool is the product > 0.6 and equals the twin's, and the scores are the sigmoid of the (ring) history."""
    from cotracker_b200.streams import OnlineStreams
    from cotracker_b200.synthetic import random_queries, texture_video
    shared = _online()
    hub, twin = OnlineStreams(shared), OnlineStreams(_online())
    F = 8 * 7 + S
    specs = {   # name: (frame size, open arguments, bound)
        "a": ((96, 128), dict(grid_size=4), None),
        "b": ((144, 192), dict(queries=random_queries(5, 40, 144, 192, seed=7).to(DEV), add_support_grid=True), 5),
        "c": ((80, 112), dict(grid_size=3, grid_query_frame=2), 13),
        "d": ((96, 96), dict(queries=random_queries(4, 30, 96, 96, seed=8).to(DEV)), None),
    }
    videos = {k: texture_video(F, *hw, seed=3 + i, shift=(1 + i, 2)).to(DEV) for i, (k, (hw, _, _)) in
              enumerate(specs.items())}
    ids = {k: (hub.open(frame_size=hw, history=h, **kw), twin.open(frame_size=hw, history=h, **kw))
           for k, (hw, kw, h) in specs.items()}
    own = {k: _online() for k in specs}
    for k, (hw, kw, _) in specs.items():
        own[k](video_chunk=videos[k][:, :S], is_first_step=True, **kw)
    with torch.no_grad():
        for step in range(6):
            live = [k for k in specs if not (k == "d" and step == 2)]       # d skips a step
            for k in live:
                ind = own[k].model.online_ind                                # the stream's window start
                chunk = videos[k][:, ind:ind + S]
                hub.push(ids[k][0], chunk)
                twin.push(ids[k][1], chunk)
            out, out0 = hub.step(return_scores=True), twin.step()
            for k in live:
                sup = specs[k][1].get("add_support_grid", False)
                ind = own[k].model.online_ind
                ftr, fvi, fsc = own[k](video_chunk=videos[k][:, ind:ind + S], add_support_grid=sup,
                                       return_scores=True)
                tr, vi, sc = out[ids[k][0]]
                assert torch.equal(tr, out0[ids[k][1]][0]) and torch.equal(vi, out0[ids[k][1]][1])
                assert torch.equal(vi, sc.visibility * sc.confidence > 0.6)
                L = fvi.shape[1] if specs[k][2] is None else min(specs[k][2], fvi.shape[1])
                assert vi.shape[1] == L
                assert torch.equal(tr, ftr[:, -L:]) and torch.equal(vi, fvi[:, -L:])
                assert torch.equal(sc.visibility, fsc.visibility[:, -L:])
                assert torch.equal(sc.confidence, fsc.confidence[:, -L:])
                st = hub._streams[ids[k][0]]["state"]
                f = torch.arange(st.length - L, st.length)
                cap = None if st.history is None else st.hist[1].shape[0]
                assert torch.equal(sc.visibility[0], _sigmoid_rows(st.hist[1], f, vi.shape[2], cap))
                assert torch.equal(sc.confidence[0], _sigmoid_rows(st.hist[2], f, vi.shape[2], cap))


def test_edited_streams_and_snapshots():
    """Added tracks read 0.5 before their first window; after retire / add, snapshot -> close -> restore on a fresh
    hub continues the scores bit for bit."""
    from cotracker_b200.streams import OnlineStreams
    from cotracker_b200.synthetic import texture_video
    p = _online()
    video = texture_video(8 * 8 + S, 112, 144, seed=9, shift=(2, 1)).to(DEV)
    hubs = [OnlineStreams(p), OnlineStreams(p)]
    for history in (None, 12):
        sids = [h.open(frame_size=(112, 144), grid_size=4, add_support_grid=True, history=history) for h in hubs]

        def step(k, pairs):
            pairs = list(pairs)
            for h, s in pairs:
                h.push(s, video[:, 8 * k:8 * k + S])
            return [h.step(return_scores=True)[s] for h, s in pairs]

        with torch.no_grad():
            for k in range(2):
                step(k, zip(hubs, sids))
            length = hubs[0].length(sids[0])
            new = torch.tensor([[[length + 1.0, 30.0, 40.0], [length + 9.0, 70.0, 20.0]]], device=DEV)
            for h, s in zip(hubs, sids):
                h.retire_tracks(s, [1, 5])
                added = h.add_tracks(s, new)
            cols = [hubs[0].track_ids(sids[0]).index(i) for i in added]
            a, b = step(2, zip(hubs, sids))
            ind = 16                                   # the third window starts at frame 16
            first = length + 8 - a[1].shape[1]          # the result's first stream frame
            split = max(ind - first, 0)                # result frames before the window: none for the bound of 12
            for sc in (a[2].visibility, a[2].confidence):
                assert bool((sc[:, :split, cols] == 0.5).all())
            assert not bool((a[2].visibility[:, split:, cols[0]] == 0.5).all())   # query frame 25: in the window
            assert all(torch.equal(x, y) for x, y in zip(a[:2] + tuple(a[2]), b[:2] + tuple(b[2])))
            snap = hubs[1].snapshot(sids[1])
            hubs[1].close(sids[1])
            fresh = OnlineStreams(p)
            r = fresh.restore(snap)
            for k in range(3, 6):
                x, y = step(k, [(hubs[0], sids[0]), (fresh, r)])
                assert torch.equal(x[0], y[0]) and torch.equal(x[1], y[1])
                assert torch.equal(x[2].visibility, y[2].visibility) and torch.equal(x[2].confidence, y[2].confidence)
            hubs[0].close(sids[0])


# ---- against the reference ---------------------------------------------------------------------------------------
# the predictor goldens that store the reference's probabilities next to its bools
OFFLINE_GOLDENS = ["pred_segm_mask", "pred_backward", "pred_grid_query_frame", "c1_apple_grid10",
                   "c1_apple_grid10_stress", "c2_grid30", "c2_grid30_stress", "headline_grid80", "headline_grid80_stress"]
ONLINE_GOLDENS = ["pred_online_support_grid", "c4_online_grid50"]


def _report(name, dev):
    """The measured deviation, on stdout (pytest -s)."""
    print(f"{name}: max |scores - reference| = {dev:.3e}")


@pytest.mark.parametrize("name", OFFLINE_GOLDENS)
def test_offline_scores_match_the_reference_probabilities(name):
    from cotracker_b200.predictor import CoTrackerPredictor
    cfg = CASES[name]
    sd, video, queries = case_inputs(cfg)
    want = load_golden(name)
    p = CoTrackerPredictor(checkpoint=None, window_len=cfg["window_len"])
    p.model.load_state_dict(sd)
    p = p.to(DEV)
    video = video.to(DEV)
    kw = predictor_kwargs(cfg, video, None if queries is None else queries.to(DEV))
    with torch.no_grad():
        tr, vi, sc = p(video, **kw, return_scores=True)
    B, T, n = vi.shape
    ref = want["prob_vis"][..., :n]
    if "prob_vis_inv" in want:
        qt = queries[:, :, 0] if queries is not None else torch.full((B, n), float(cfg.get("grid_query_frame", 0)))
        ref = torch.where(torch.arange(T)[None, :, None] < qt[:, None, :], want["prob_vis_inv"][..., :n], ref)
    dev = float((sc.visibility.cpu() - ref).abs().max())
    _report(name, dev)
    assert dev <= REFERENCE_TOL, f"{name}: {dev:.3e}"


@pytest.mark.parametrize("name", ONLINE_GOLDENS)
def test_online_scores_match_the_reference_probabilities(name):
    from cotracker_b200.predictor import CoTrackerOnlinePredictor
    cfg = CASES[name]
    sd, video, queries = case_inputs(cfg)
    want = load_golden(name)
    p = CoTrackerOnlinePredictor(checkpoint=None, window_len=cfg["window_len"])
    p.model.load_state_dict(sd)
    p = p.to(DEV)
    video = video.to(DEV)
    kw = predictor_kwargs(cfg, video, None if queries is None else queries.to(DEV))
    sup = cfg.get("add_support_grid", False)
    dev = 0.0
    with torch.no_grad():
        p(video_chunk=video, is_first_step=True, **kw)
        for k, ind in enumerate(range(0, video.shape[1] - p.step, p.step)):
            tr, vi, sc = p(video_chunk=video[:, ind:ind + 2 * p.step], add_support_grid=sup, return_scores=True)
            prod = (sc.visibility * sc.confidence).cpu()
            dev = max(dev, float((prod - want[f"prob_visconf{k}"][..., :vi.shape[2]]).abs().max()))
    _report(name, dev)
    assert dev <= REFERENCE_TOL, f"{name}: {dev:.3e}"
