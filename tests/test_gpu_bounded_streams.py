"""GPU tests of bounded online streams (`OnlineStreams.open(history=h)`): at every step a bounded stream's result is
`torch.equal` to the last L = min(h, frames so far) frames of the same stream opened without a bound, whatever the other
streams do and however the step is split into passes; the reference golden tracked as a bounded stream meets its bound;
the ring-mode window kernels equal torch expressions on the ring bit for bit; and a bounded hub's device memory stops
growing."""
import pytest
import torch

from cases import CASES, case_inputs, compare, load_golden, predictor_kwargs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
S = 16


def _predictor(seed=47):
    from cotracker_b200.predictor import CoTrackerOnlinePredictor
    from cotracker_b200.synthetic import seeded_state_dict
    p = CoTrackerOnlinePredictor(checkpoint=None, window_len=S)
    p.model.load_state_dict(seeded_state_dict(seed, offline=False, window_len=S, head_gain=10.0, vis_gain=100.0))
    return p.to(DEV)


def _video(T, h, w, seed):
    from cotracker_b200.synthetic import texture_video
    return texture_video(T, h, w, seed=seed, shift=(1 + seed % 3, 2))


def _dev_chunks(video):
    v = video.to(DEV)
    return lambda k: v[:, 8 * k:8 * k + S]


def _host_u8_hwc_chunks(video):
    hwc = video.to(torch.uint8).permute(0, 1, 3, 4, 2).contiguous()    # a decoder's [1,T,H,W,3] buffer
    return lambda k: hwc[:, 8 * k:8 * k + S].permute(0, 1, 4, 2, 3)


class _Pair:
    """One stream opened on both hubs: bounded (history=h) on one, unbounded on the other, fed the same chunks
    (h = None: unbounded on both)."""

    def __init__(self, bounded, full, h, chunk_of, frame_size, **first):
        self.h, self.chunk_of, self.k = h, chunk_of, 0
        self.b = bounded.open(frame_size=frame_size, history=h, **first)
        self.f = full.open(frame_size=frame_size, **first)

    def push(self, bounded, full):
        c = self.chunk_of(self.k)
        self.k += 1
        bounded.push(self.b, c)
        full.push(self.f, c)

    def check(self, bounded, full, ob, of):
        (tr, vi), (ftr, fvi) = ob[self.b], of[self.f]
        L = ftr.shape[1] if self.h is None else min(self.h, ftr.shape[1])
        assert bounded.length(self.b) == full.length(self.f) == ftr.shape[1]
        assert tr.shape == (1, L) + tuple(ftr.shape[2:]) and vi.dtype == torch.bool
        assert torch.equal(tr, ftr[:, -L:]) and torch.equal(vi, fvi[:, -L:])


def _run(plan, steps, split=False):
    """plan(i) -> (pairs to open as {name: kwargs}, names to advance, names to close); checks every step."""
    from cotracker_b200.streams import OnlineStreams
    p = _predictor()
    bounded, full = OnlineStreams(p), OnlineStreams(p)
    pairs, n_checked, outs = {}, 0, []
    for i in range(steps):
        opens, adv, closes = plan(i)
        for name, kw in opens.items():
            pairs[name] = _Pair(bounded, full, **kw)
        for name in adv:
            pairs[name].push(bounded, full)
        ob, of = bounded.step(), full.step()
        assert set(ob) == {pairs[n].b for n in adv}
        for name in adv:
            pairs[name].check(bounded, full, ob, of)
            n_checked += 1
        outs.append({n: ob[pairs[n].b] for n in adv})
        for name in closes:
            pr = pairs.pop(name)
            bounded.close(pr.b)
            full.close(pr.f)
    return n_checked, outs


def test_bounded_streams_equal_the_tail_of_unbounded_ones():
    """Six bounds over 16 steps (every ring shorter than its stream wraps several times): staggered opens, a stream that
    skips steps, one that closes and reopens, mixed frame sizes, host uint8 and device float chunks, query frames that
    enter in later windows and a support grid."""
    from cotracker_b200.synthetic import random_queries
    F = 8 * 17 + S
    va, vb, vc = _video(F, 96, 128, 1), _video(F, 144, 192, 2), _video(F, 80, 112, 3)
    vd, ve, vf = _video(F, 96, 96, 4), _video(F, 64, 80, 5), _video(F, 96, 128, 6)
    qb = random_queries(7, 60, 144, 192, seed=5).to(DEV)                    # query frames up to 59: later windows
    qe = random_queries(5, 40, 64, 80, seed=6).to(DEV)

    def plan(i):
        opens = {}
        if i == 0:
            opens["a"] = dict(h=1, chunk_of=_dev_chunks(va), frame_size=(96, 128), grid_size=4, grid_query_frame=2)
            opens["d"] = dict(h=16, chunk_of=_host_u8_hwc_chunks(vd), frame_size=(96, 96), grid_size=3)
            opens["f"] = dict(h=200, chunk_of=_dev_chunks(vf), frame_size=(96, 128), grid_size=3)
        if i == 1:
            opens["c"] = dict(h=8, chunk_of=_dev_chunks(vc), frame_size=(80, 112), grid_size=3)
        if i == 2:
            opens["b"] = dict(h=5, chunk_of=_host_u8_hwc_chunks(vb), frame_size=(144, 192), queries=qb,
                              add_support_grid=True)
        if i == 3:
            opens["e"] = dict(h=23, chunk_of=_dev_chunks(ve), frame_size=(64, 80), queries=qe)
        if i == 9:                                                          # d reopens in the compacted pool
            opens["d"] = dict(h=16, chunk_of=_dev_chunks(vd), frame_size=(96, 96), grid_size=4)
        opened = dict(a=0, b=2, c=1, d=0, e=3, f=0)
        live = [n for n in "abcdef" if opened[n] <= i and not (n == "d" and 7 <= i <= 8)]
        adv = [n for n in live if not (n == "c" and i in (4, 5, 10))]      # c skips three steps
        return opens, adv, ["d"] if i == 6 else []

    n, _ = _run(plan, 16)
    assert n >= 70


def test_bounded_stream_ending_on_a_short_chunk():
    """One bounded stream ends on an 11-frame chunk, another on a 3-frame one (shorter than the overlap)."""
    va, vb = _video(72, 96, 128, 11).to(DEV), _video(72, 96, 128, 12).to(DEV)

    def chunks(v, last, T):
        return lambda k: v[:, 8 * k:8 * k + (S if k < last else T)]

    def plan(i):
        opens = {}
        if i == 0:
            opens = dict(a=dict(h=5, chunk_of=chunks(va, 3, 11), frame_size=(96, 128), grid_size=4),
                         b=dict(h=13, chunk_of=chunks(vb, 4, 3), frame_size=(96, 128), grid_size=3))
        return opens, (["a", "b"] if i < 4 else ["b"]), []

    n, _ = _run(plan, 5)
    assert n == 9


def _mixed(split, monkeypatch):
    import cotracker_b200.model as M
    passes = []
    if split:
        planner = M.plan_clip_passes
        monkeypatch.setattr(M, "pass_budget_bytes", lambda *a, **k: 1)
        monkeypatch.setattr(M, "plan_clip_passes", lambda *a, **k: passes.append(planner(*a, **k)) or passes[-1])
    vids = [_video(8 * 7 + S, 96, 128, 20 + k).to(DEV) for k in range(4)]
    hs = [None, 3, 40, 9]

    def plan(i):
        opens = {}
        if i == 0:
            opens = {str(k): dict(h=h, chunk_of=(lambda v: lambda k: v[:, 8 * k:8 * k + S])(v), frame_size=(96, 128),
                                  grid_size=3 + k) for k, (h, v) in enumerate(zip(hs, vids))}
        return opens, ["0", "1", "2", "3"], []

    return _run(plan, 6)[1], passes


def test_bounded_and_unbounded_streams_in_one_pass_and_split(monkeypatch):
    """Bounded and unbounded streams advance together in one pass; forcing one stream per pass changes no bit."""
    want, passes = _mixed(False, monkeypatch)
    assert not passes
    got, passes = _mixed(True, monkeypatch)
    assert passes and all(len(p) == 4 for p in passes)                       # one stream per pass
    for g, w in zip(got, want):
        assert g.keys() == w.keys()
        for k in g:
            assert torch.equal(g[k][0], w[k][0]) and torch.equal(g[k][1], w[k][1])


@pytest.mark.parametrize("h", [1, 5, 16, 24, 200])
def test_predictor_online_golden_as_a_bounded_stream(h):
    """The reference golden `predictor_online` as a bounded stream between two others: for h >= its length it meets
    the golden's bound, for smaller h it equals the golden's last h frames."""
    from cotracker_b200.streams import OnlineStreams
    name = "predictor_online"
    cfg = CASES[name]
    sd, video, queries = case_inputs(cfg)
    assert cfg["window_len"] == S
    p = _predictor()
    p.model.load_state_dict(sd)
    hub = OnlineStreams(p)
    H, W = video.shape[3:]
    other = _video(video.shape[1] + 16, 80, 96, 31).to(DEV)
    first = {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in predictor_kwargs(cfg, video, queries).items()}
    o1 = hub.open(frame_size=(80, 96), grid_size=5, history=7)
    step = S // 2
    hub.push(o1, other[:, :S])
    hub.step()
    g = hub.open(frame_size=(H, W), history=h, **first)
    o2 = hub.open(frame_size=(80, 96), grid_size=3)
    v = video.to(DEV)
    golden = load_golden(name)
    got, want = {}, {}
    for k, ind in enumerate(range(0, video.shape[1] - step, step)):
        hub.push(g, v[:, ind:ind + 2 * step])
        hub.push(o1, other[:, step * (k + 1):step * (k + 1) + S])
        if k % 2 == 0:
            hub.push(o2, other[:, ind:ind + S])
        res = hub.step()
        n = golden[f"tracks{k}"].shape[1]
        assert hub.length(g) == n and res[g][0].shape[1] == min(h, n)
        for key in (f"tracks{k}", f"visibility{k}"):
            want[key] = golden[key][:, -min(h, n):]
        got[f"tracks{k}"], got[f"visibility{k}"] = res[g][0].cpu(), res[g][1].cpu()
    print(compare(got, want, tol_px=1e-3, tol_logit=1e-3))


# ---- ring-mode ct3_online_window_begin / _end against torch expressions on the ring ----------------------------------
def _logical(ring, first_frame, length):
    """Frames [first_frame, length) of a ring history as a plain [frames, ...] tensor."""
    cap = ring.shape[0]
    rows = torch.arange(first_frame, length, device=ring.device) % cap
    return ring[rows]


@pytest.mark.parametrize("K", [1, 3, 7])
def test_ring_window_kernels_bitwise_equal_torch(K):
    from cotracker_b200 import engine
    g = torch.Generator().manual_seed(100 + K)
    S_, step, stride = 16, 8, 4
    overlap = S_ - step
    streams, first = [], 0
    for k in range(K):
        n = int(torch.randint(1, 40, (1,), generator=g))
        ring = k % 4 != 3                                                   # every fourth entry: a plain history
        T = S_ if k % 3 else int(torch.randint(1, S_ + 1, (1,), generator=g))
        if ring:
            cap = S_ + int(torch.randint(0, 30, (1,), generator=g))
            ind = 8 * int(torch.randint(cap // 8 + 1, cap // 8 + 20, (1,), generator=g))   # ind > cap: wrapped
        else:
            ind = 8 * int(torch.randint(1, 8, (1,), generator=g))
            cap = ind + S_ + 3
        length = ind + overlap
        held = length - cap if ring else 0
        L_max = min(cap if ring else ind + T, ind + T - held)
        L = int(torch.randint(1, L_max + 1, (1,), generator=g))
        if k == 0:
            L = min(L_max, max(L, T + 3))                                   # output frames before the window
        hist = ((torch.rand(cap, n, 2, generator=g) * 500 - 20).to(DEV), (torch.randn(cap, n, generator=g) * 8).to(DEV),
                (torch.randn(cap, n, generator=g) * 8).to(DEV))
        n_keep = max(1, n - (36 if n > 36 else k % 2))
        streams.append(dict(n=n, ind=ind, T=T, length=length, hist=hist, first=first, frame0=k * S_, n_keep=n_keep,
                            ring=ring, out_first=ind + T - L, scale=((1280 - 1) / (512 - 1), (720 - 1) / (384 - 1))))
        first += n
    N = first
    assert any(s["ring"] and s["ind"] > s["hist"][1].shape[0] and s["out_first"] > 0 for s in streams)
    qf = torch.randint(-3, 400, (N,), generator=g).to(DEV)
    qc = (torch.rand(N, 2, generator=g) * 120).to(DEV)

    def entry(s, out=None):
        return engine.online_stream(s["hist"], s["length"], s["ind"], s["T"], s["first"], s["frame0"], out,
                                    s["n_keep"] if out else 0, s["scale"], out_first=s["out_first"] if out else 0,
                                    ring=s["ring"])

    got = engine.online_window_begin([entry(s) for s in streams], S_, step, stride, K * S_, qf.to(torch.int32), qc)
    for s in streams:
        a, b, ind = s["first"], s["first"] + s["n"], s["ind"]
        f, n = qf[a:b], s["n"]
        prev = [_logical(h, ind, ind + overlap) for h in s["hist"]]
        rows = torch.clamp(torch.arange(S_, device=DEV), max=overlap - 1)
        carry = (f < ind + overlap)[None, :]
        want = ((f < ind + S_).to(torch.uint8), ((f >= ind + step) & (f < ind + S_)).to(torch.uint8),
                ((f - ind).clamp(0, S_ - 1) + s["frame0"]).to(torch.int32),
                torch.where(carry[..., None], prev[0][rows] / stride, qc[a:b][None].expand(S_, n, 2)),
                torch.where(carry, prev[1][rows], torch.zeros(S_, n, device=DEV)),
                torch.where(carry, prev[2][rows], torch.zeros(S_, n, device=DEV)))
        for x, y in zip(got, want):
            assert torch.equal(x[..., a:b, :] if x.dim() == 3 else (x[:, a:b] if x.dim() == 2 else x[a:b]), y)

    coords = (torch.rand(S_, N, 2, generator=g) * 130).to(DEV)
    vis = (torch.randn(S_, N, generator=g) * 6).to(DEV)
    conf = (torch.randn(S_, N, generator=g) * 6).to(DEV)
    before = [tuple(h.clone() for h in s["hist"]) for s in streams]
    outs = []
    for s in streams:
        L = s["ind"] + s["T"] - s["out_first"]
        outs.append((torch.empty(L, s["n_keep"], 2, device=DEV), torch.empty(L, s["n_keep"], dtype=torch.bool,
                                                                            device=DEV)))
    engine.online_window_end([entry(s, o) for s, o in zip(streams, outs)], S_, stride, coords, vis, conf)
    for s, h0, (tr, vi) in zip(streams, before, outs):
        a, b, ind, T, cap = s["first"], s["first"] + s["n"], s["ind"], s["T"], s["hist"][1].shape[0]
        want = [h.clone() for h in h0]
        rows = (torch.arange(ind, ind + T, device=DEV) % cap) if s["ring"] else torch.arange(ind, ind + T, device=DEV)
        want[0][rows] = (coords * float(stride))[:T, a:b]
        want[1][rows] = vis[:T, a:b]
        want[2][rows] = conf[:T, a:b]
        for x, y in zip(s["hist"], want):
            assert torch.equal(x, y)
        span = [_logical(w, s["out_first"], ind + T) if s["ring"] else w[s["out_first"]:ind + T] for w in want]
        tracks = span[0][:, :s["n_keep"]] * span[0].new_tensor(s["scale"])
        visible = (torch.sigmoid(span[1]) * torch.sigmoid(span[2]))[:, :s["n_keep"]] > 0.6
        assert torch.equal(tr, tracks) and torch.equal(vi, visible)


def test_bounded_hub_memory_stops_growing():
    """With its results dropped, a bounded hub holds the same device memory after step 80 as after step 20."""
    from cotracker_b200.streams import OnlineStreams
    hub = OnlineStreams(_predictor())
    base = [_video(64, 64, 80, 40 + k).to(DEV) for k in range(2)]
    loops = [torch.cat([v, v[:, :S]], 1) for v in base]                     # frame f + 64 repeats frame f
    ids = [hub.open(frame_size=(64, 80), grid_size=4, history=h) for h in (5, 30)]
    seen = {}
    for i in range(1, 81):
        for sid, v in zip(ids, loops):
            hub.push(sid, v[:, (8 * (i - 1)) % 64:(8 * (i - 1)) % 64 + S])
        out = hub.step()
        assert [o[0].shape[1] for o in out.values()] == [min(5, 8 * i + 8), min(30, 8 * i + 8)]
        del out
        if i in (20, 80):
            torch.cuda.synchronize()
            seen[i] = torch.cuda.memory_allocated()
    assert hub.length(ids[0]) == 8 * 80 + 8
    assert seen[20] == seen[80], seen
