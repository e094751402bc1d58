"""GPU tests of independent online streams (cotracker_b200.streams.OnlineStreams): every result of a stream is
bit-identical to a fresh CoTrackerOnlinePredictor on the same model fed that stream's chunks, whatever the other streams
do; a reference golden tracked as one stream among others meets its bound; ct3_online_window_begin / _end equal the
torch expressions they replace bit for bit."""
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


class _Stream:
    """A stream of the hub and its reference: a fresh predictor on the same model, fed the same chunks."""

    def __init__(self, hub, video, chunk_of, **first):
        self.video, self.chunk_of, self.first = video, chunk_of, first
        self.ref = _predictor()
        self.ref.model.load_state_dict(hub.model.state_dict())
        self.id = hub.open(frame_size=tuple(video.shape[3:]), **first)
        self.ref(video_chunk=chunk_of(video, 0), is_first_step=True, **first)
        self.k = 0

    def chunk(self):
        c = self.chunk_of(self.video, self.k)
        self.k += 1
        return c

    def check(self, got, chunk):
        want = self.ref(video_chunk=chunk, add_support_grid=self.first.get("add_support_grid", False))
        assert got[0].shape == want[0].shape and got[1].shape == want[1].shape, (got[0].shape, want[0].shape)
        assert got[1].dtype == torch.bool
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


def _dev_chunks(video):
    v = video.to(DEV)
    return lambda _, k: v[:, 8 * k:8 * k + S]


def _host_u8_hwc_chunks(video):
    hwc = video.to(torch.uint8).permute(0, 1, 3, 4, 2).contiguous()    # a decoder's [1,T,H,W,3] buffer
    return lambda _, k: hwc[:, 8 * k:8 * k + S].permute(0, 1, 4, 2, 3)


def _run(hub, plan, streams, steps):
    """plan(step) -> (streams to open as {name: kwargs}, names to advance, names to close); checks every result."""
    n_checked = 0
    for i in range(steps):
        opens, adv, closes = plan(i)
        for name, kw in opens.items():
            streams[name] = _Stream(hub, **kw)
        chunks = {}
        for name in adv:
            chunks[name] = streams[name].chunk()
            hub.push(streams[name].id, chunks[name])
        out = hub.step()
        assert set(out) == {streams[n].id for n in adv}
        for name in adv:
            streams[name].check(out[streams[name].id], chunks[name])
            n_checked += 1
        for name in closes:
            hub.close(streams.pop(name).id)
    return n_checked


def test_staggered_skipping_closing_mixed_streams():
    """Staggered starts (b opens three steps after a), a stream that skips steps, close then open in the compacted
    pool, mixed frame sizes, host uint8 channels-last and device float chunks, grid / queries / support grid, and query
    frames that enter in later windows."""
    from cotracker_b200.streams import OnlineStreams
    from cotracker_b200.synthetic import random_queries
    hub = OnlineStreams(_predictor())
    va, vb, vc, vd = _video(88, 96, 128, 1), _video(88, 144, 192, 2), _video(88, 80, 112, 3), _video(88, 96, 96, 4)
    qb = random_queries(7, 40, 144, 192, seed=5).to(DEV)                    # query frames up to 39: later windows
    qd = random_queries(5, 30, 96, 96, seed=6).to(DEV)

    def plan(i):
        opens = {}
        if i == 0:
            opens["a"] = dict(video=va, chunk_of=_dev_chunks(va), grid_size=4, grid_query_frame=2)
        if i == 3:
            opens["b"] = dict(video=vb, chunk_of=_host_u8_hwc_chunks(vb), queries=qb, add_support_grid=True)
            opens["c"] = dict(video=vc, chunk_of=_dev_chunks(vc), grid_size=3)
        if i == 6:
            opens["d"] = dict(video=vd, chunk_of=_host_u8_hwc_chunks(vd), queries=qd)
        adv = [n for n in "abcd" if n in streams or n in opens]
        if i in (4, 5):
            adv.remove("c")                                                  # c skips two steps
        return opens, adv, ["a"] if i == 5 else []                          # a closes; d opens in the compacted pool

    streams = {}
    assert _run(hub, plan, streams, 9) >= 18


def test_short_last_chunk_and_reencoded_overlap():
    """One stream ends with T < window_len while another runs on; a chunk whose overlap frames differ from the previous
    chunk's (only that stream is re-encoded)."""
    from cotracker_b200.streams import OnlineStreams
    hub = OnlineStreams(_predictor())
    va, vb = _video(60, 96, 128, 11), _video(60, 96, 128, 12).to(DEV)
    vb_alt = vb.clone()
    vb_alt[:, 16:24] += 3.0                                                 # frames chunk 2 shares with chunk 1

    def b_chunks(_, k):
        return (vb_alt if k == 2 else vb)[:, 8 * k:8 * k + S]

    def a_chunks(v, k):
        return v[:, 8 * k:8 * k + (S if k < 3 else 11)].to(DEV)            # chunk 3 holds 11 frames

    def plan(i):
        opens = {}
        if i == 0:
            opens = dict(a=dict(video=va, chunk_of=a_chunks, grid_size=4),
                         b=dict(video=vb, chunk_of=b_chunks, grid_size=5, grid_query_frame=1))
        return opens, ["a", "b"] if i < 4 else ["b"], []

    streams = {}
    _run(hub, plan, streams, 6)
    with pytest.raises(ValueError, match="ended"):                           # nothing follows a short chunk
        hub.push(streams["a"].id, va[:, :S])


def test_forced_pass_split_is_bit_identical(monkeypatch):
    import cotracker_b200.model as M
    from cotracker_b200.streams import OnlineStreams

    def run(split):
        hub = OnlineStreams(_predictor())
        vids = [_video(40, 96, 128, 20 + k).to(DEV) for k in range(3)]
        ids = [hub.open(frame_size=(96, 128), grid_size=3 + k) for k in range(3)]
        outs = []
        for step in range(3):
            for i, v in zip(ids, vids):
                hub.push(i, v[:, 8 * step:8 * step + S])
            outs.append(hub.step())
        return outs

    want = run(False)
    passes = []
    plan = M.plan_clip_passes
    monkeypatch.setattr(M, "pass_budget_bytes", lambda *a, **k: 1)
    monkeypatch.setattr(M, "plan_clip_passes", lambda *a, **k: passes.append(plan(*a, **k)) or passes[-1])
    got = run(True)
    assert passes and all(len(p) == 3 for p in passes)                       # one stream per pass
    for g, w in zip(got, want):
        assert g.keys() == w.keys()
        for k in g:
            assert torch.equal(g[k][0], w[k][0]) and torch.equal(g[k][1], w[k][1])


def test_predictor_online_golden_as_one_of_three_streams():
    """The reference golden `predictor_online` as the middle stream, opened a step after an unrelated one."""
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
    o1 = hub.open(frame_size=(80, 96), grid_size=5)
    out = {}
    step = S // 2
    hub.push(o1, other[:, :S])
    hub.step()
    g = hub.open(frame_size=(H, W), **first)
    o2 = hub.open(frame_size=(80, 96), grid_size=3)
    v = video.to(DEV)
    for k, ind in enumerate(range(0, video.shape[1] - step, step)):
        hub.push(g, v[:, ind:ind + 2 * step])
        hub.push(o1, other[:, step * (k + 1):step * (k + 1) + S])
        if k % 2 == 0:
            hub.push(o2, other[:, ind:ind + S])
        res = hub.step()
        out[f"tracks{k}"], out[f"visibility{k}"] = res[g][0].cpu(), res[g][1].cpu()
    print(compare(out, load_golden(name), tol_px=1e-3, tol_logit=1e-3))


# ---- ct3_online_window_begin / _end against the torch expressions ---------------------------------------------------
def _torch_begin(s, qf, qc, S_, step, stride):
    """The per-window torch expressions of the streaming model for one stream (qf int64 [n], qc [n,2])."""
    ind, hist, n = s["ind"], s["hist"], qf.shape[0]
    left = 0 if ind == 0 else ind + step
    entering = ((qf >= left) & (qf < ind + S_)).to(torch.uint8)
    valid = (qf < ind + S_).to(torch.uint8)
    rel = ((qf - ind).clamp(0, S_ - 1) + s["frame0"]).to(torch.int32)
    coords_init = qc[None].expand(S_, n, 2).contiguous()
    vis_init = torch.zeros(S_, n, device=DEV)
    conf_init = torch.zeros(S_, n, device=DEV)
    if ind > 0:
        overlap = S_ - step
        carry = (qf < ind + overlap)[None, :]
        prev_c = hist[0][ind:ind + overlap] / stride
        prev_c = torch.cat([prev_c, prev_c[-1:].expand(step, -1, -1)], 0)
        prev_v = torch.cat([hist[1][ind:ind + overlap], hist[1][ind + overlap - 1:ind + overlap].expand(step, -1)], 0)
        prev_q = torch.cat([hist[2][ind:ind + overlap], hist[2][ind + overlap - 1:ind + overlap].expand(step, -1)], 0)
        coords_init = torch.where(carry[..., None], prev_c, coords_init)
        vis_init = torch.where(carry, prev_v, vis_init)
        conf_init = torch.where(carry, prev_q, conf_init)
    return valid, entering, rel, coords_init, vis_init, conf_init


@pytest.mark.parametrize("K", [1, 3, 7])
def test_online_window_kernels_bitwise_equal_torch(K):
    from cotracker_b200 import engine
    g = torch.Generator().manual_seed(K)
    S_, step, stride = 16, 8, 4
    streams, first = [], 0
    for k in range(K):
        n = int(torch.randint(1, 40, (1,), generator=g))
        ind = [0, 8, 24, 56][k % 4]
        T = S_ if k % 3 else int(torch.randint(1, S_ + 1, (1,), generator=g))
        length = 0 if ind == 0 else ind + S_ - step
        cap = ind + S_ + 5
        hist = ((torch.rand(cap, n, 2, generator=g) * 500 - 20).to(DEV), (torch.randn(cap, n, generator=g) * 8).to(DEV),
                (torch.randn(cap, n, generator=g) * 8).to(DEV))
        n_keep = max(1, n - (36 if n > 36 else k % 2))
        streams.append(dict(n=n, ind=ind, T=T, length=length, hist=hist, first=first, frame0=k * S_, n_keep=n_keep,
                            scale=((1280 - 1) / (512 - 1), (720 - 1) / (384 - 1))))
        first += n
    N = first
    qf = torch.randint(-3, 80, (N,), generator=g).to(DEV)
    qc = (torch.rand(N, 2, generator=g) * 120).to(DEV)
    entries = [engine.online_stream(s["hist"], s["length"], s["ind"], s["T"], s["first"], s["frame0"]) for s in streams]
    got = engine.online_window_begin(entries, S_, step, stride, K * S_, qf.to(torch.int32), qc)
    for s in streams:
        a, b = s["first"], s["first"] + s["n"]
        want = _torch_begin(s, qf[a:b], qc[a:b], S_, step, stride)
        for x, y in zip(got, want):
            assert torch.equal(x[..., a:b, :] if x.dim() == 3 else (x[:, a:b] if x.dim() == 2 else x[a:b]), y)

    coords = (torch.rand(S_, N, 2, generator=g) * 130).to(DEV)
    vis = (torch.randn(S_, N, generator=g) * 6).to(DEV)
    conf = (torch.randn(S_, N, generator=g) * 6).to(DEV)
    vis[0, :3] = 0.0                                                        # sigmoid(0)^2 = 0.25: well below 0.6
    before = [tuple(h.clone() for h in s["hist"]) for s in streams]
    outs = []
    for s in streams:
        rows = s["ind"] + s["T"]
        outs.append((torch.empty(rows, s["n_keep"], 2, device=DEV), torch.empty(rows, s["n_keep"], dtype=torch.bool,
                                                                               device=DEV)))
    entries = [engine.online_stream(s["hist"], s["length"], s["ind"], s["T"], s["first"], s["frame0"], o, s["n_keep"],
                                    s["scale"]) for s, o in zip(streams, outs)]
    engine.online_window_end(entries, S_, stride, coords, vis, conf)
    for s, h0, (tr, vi) in zip(streams, before, outs):
        a, b, ind, T = s["first"], s["first"] + s["n"], s["ind"], s["T"]
        want = [h.clone() for h in h0]
        want[0][ind:ind + T] = (coords * float(stride))[:T, a:b]
        want[1][ind:ind + T] = vis[:T, a:b]
        want[2][ind:ind + T] = conf[:T, a:b]
        for x, y in zip(s["hist"], want):
            assert torch.equal(x, y)
        rows = ind + T
        tracks = want[0][:rows, :s["n_keep"]] * want[0].new_tensor(s["scale"])
        visible = (torch.sigmoid(want[1][:rows]) * torch.sigmoid(want[2][:rows]))[:, :s["n_keep"]] > 0.6
        assert torch.equal(tr, tracks) and torch.equal(vi, visible)
        assert 0 < int(vi.sum()) < vi.numel() or vi.numel() < 8
