"""GPU tests of corner detection: ct3_detect_corners is bit-identical to the float64 restatement of
tests/corner_cases.py (responses, corners, counts) over frame sizes, block sizes, quality levels, minimum distances,
caps, ties, degenerate frames, exclusion discs, batching and frame strides; detect_corners gives the same queries for
every input form; OnlineStreams.seed_corners equals detect + add_tracks by hand, stays within its cap in a bounded
stream with flat memory, and a seeded stream snapshots and restores bit for bit."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import corner_cases as C
from cotracker_b200 import YUVClip, corners, detect_corners, engine

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
S, STEP = 16, 8


def _apple(idx=(0, 25, 49)):
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    v = np.load(os.path.join(root, "tests", "golden", "apple_frames_120x216.npz"))["frames"]
    x = torch.from_numpy(v[list(idx)]).permute(0, 3, 1, 2).float()
    return (2 * (F.interpolate(x, (384, 512), mode="bilinear", align_corners=True) / 255) - 1).contiguous()


def _run(frames, par, exclude=None):
    """frames [K,3,H,W] on the device, par: K CornerParams -> (corners, counts, responses [K,H,W] fp64) on the host."""
    K, _, H, W = frames.shape
    ws = torch.empty(engine.corners_workspace_bytes(K, H, W), dtype=torch.uint8, device=DEV)
    found, counts = engine.detect_corners(frames, par, exclude, workspace=ws)
    lam = ws[:K * H * W * 8].view(torch.float64).view(K, H, W)
    return found.cpu(), counts.cpu(), lam.cpu()


def _check(frame, par, excl=None):
    """One frame on the device against the oracle with the same parameters: corners, count and responses equal."""
    f = frame.to(DEV)[None]
    ex = None if excl is None else (torch.as_tensor(excl, dtype=torch.float32, device=DEV)[None], [len(excl)])
    found, counts, lam = _run(f, [par], ex)
    want, want_lam = C.corners(frame.cpu().numpy(), par.max_corners, par.quality_level, par.min_distance,
                               par.block_size, excl, par.exclude_radius)
    assert torch.equal(lam[0], torch.from_numpy(want_lam))
    n = int(counts[0])
    assert n == len(want)
    assert torch.equal(found[0, :n], torch.from_numpy(want).float())
    assert not found[0, n:].any()
    return want


@pytest.mark.parametrize("block", [3, 5, 7])
def test_apple_frames_equal_oracle(block):
    for f in _apple():
        for q, md, m in ((0.01, 10, 300), (0.001, 0, 50), (0.3, 37, 10 ** 5), (0.01, 1, 1), (0.001, 0.5, 1000)):
            _check(f, corners.params(m, q, md, block))


@pytest.mark.parametrize("hw", [(97, 131), (7, 9), (16, 32), (33, 65), (384, 512)])
def test_odd_sizes_equal_oracle(hw):
    f = C.textured_frame(*hw, seed=hw[0])
    for block in (3, 5, 7):
        for q, md, m in ((1e-3, 0, 10 ** 5), (0.01, 10, 50), (0.3, 1, 10 ** 5), (0.01, 37, 10 ** 5), (1e-3, 0.5, 1)):
            _check(f, corners.params(m, q, md, block))


def test_ties_pin_the_order():
    for period, md in ((8, 0), (8, 10), (5, 3), (6, 1.5)):
        want = _check(C.checkerboard(384, 512, period), corners.params(10 ** 5, 0.01, md, 3))
        assert len(want) > (300 if md <= 3 else 100)
    stripes = C.checkerboard(96, 128, 4)
    stripes[:, ::7] = 0.3                       # broken plateaus of equal values in both directions
    _check(stripes, corners.params(10 ** 5, 1e-3, 0, 5))


def test_degenerate_frames():
    flat = torch.full((3, 40, 56), 0.25)
    assert len(_check(flat, corners.params(10))) == 0
    one = flat.clone()
    one[:, 17, 30] = 1.0
    assert _check(one, corners.params(10, 0.01, 10)).tolist() == [[30, 17]]


def test_exclusion_discs():
    f = C.textured_frame(192, 256, seed=7)
    full = _check(f, corners.params(500, 0.001, 5))
    pts = [[float(x) + 0.25, float(y) - 0.5] for x, y in full[::3]]
    for r in (0.0, 4.0, 12.5):
        got = _check(f, corners.params(500, 0.001, 5, 3, r), pts)
        if r == 0:
            assert np.array_equal(got, full)
        else:
            assert len(set(map(tuple, got.tolist())) & set(map(tuple, full[::3].tolist()))) == 0


def test_batch_equals_single_frames_and_strides():
    frames = torch.stack([C.textured_frame(120, 160, seed=s) for s in range(4)] + [C.checkerboard(120, 160, 6)])
    pars = [corners.params(300, 0.01, 10, 3), corners.params(7, 0.3, 0, 5), corners.params(1000, 1e-3, 2.5, 7, 3),
            corners.params(50, 0.05, 37, 3, 9), corners.params(2000, 0.01, 0.5, 5)]
    E = 12
    g = torch.Generator().manual_seed(0)
    pts = torch.rand(5, E, 2, generator=g) * torch.tensor([159.0, 119.0])
    cnt = [0, 12, 5, 3, 1]
    dev = frames.to(DEV)
    found, counts, lam = _run(dev, pars, (pts.to(DEV), cnt))
    M = found.shape[1]
    assert M == 2000
    for k in range(5):
        one, c1, l1 = _run(dev[k:k + 1], [pars[k]], (pts[k:k + 1, :max(cnt[k], 1)].to(DEV), [cnt[k]]))
        assert torch.equal(counts[k:k + 1], c1) and torch.equal(lam[k], l1[0])
        assert torch.equal(found[k, :one.shape[1]], one[0]) and not found[k, one.shape[1]:].any()
    # a frame-strided view (every other frame of a clip) equals its contiguous copy
    clip = torch.stack([C.textured_frame(64, 96, seed=s) for s in range(6)]).to(DEV)
    view = clip[::2]
    assert view.stride(0) == 6 * 64 * 96
    a, b = _run(view, corners.params(100)), _run(view.contiguous(), corners.params(100))
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    same = clip[:1].expand(3, -1, -1, -1)       # frame stride 0
    c = _run(same, corners.params(100))
    assert all(torch.equal(c[i][k], c[i][0]) for i in range(3) for k in range(3))


def test_public_function_inputs_agree():
    from cotracker_b200.synthetic import texture_video
    from yuv_cases import yuv_video
    u8 = texture_video(5, 120, 216, seed=4)[0].to(torch.uint8)[None]        # [1,T,3,H,W]
    ref = detect_corners(u8.float().to(DEV), 200, frame=2)
    assert ref.shape[0] == 1 and ref.shape[2] == 3 and ref.shape[1] > 20
    assert bool((ref[0, :, 0] == 2).all())
    for v in (u8, u8.to(DEV), u8.float(), u8.permute(0, 1, 3, 4, 2).contiguous().permute(0, 1, 4, 2, 3).to(DEV)):
        assert torch.equal(detect_corners(v, 200, frame=2), ref)
    # NV12 against the RGB float device clip of the same frames
    nv12 = yuv_video("nv12", 2, 4, 96, 128, seed=1)
    from yuv_cases import yuv_to_rgb
    rgb = yuv_to_rgb("nv12", nv12).float().to(DEV)
    got = detect_corners(YUVClip(nv12, "nv12"), 150, frame=3, min_distance=5)
    assert isinstance(got, list) and len(got) == 2
    for b in range(2):
        assert torch.equal(got[b], detect_corners(rgb[b:b + 1], 150, frame=3, min_distance=5))
    assert torch.equal(detect_corners(YUVClip(nv12, "nv12").to(DEV), 150, frame=3, min_distance=5)[1], got[1])
    # B = 3 list form equals three B = 1 calls, with per-clip exclusions in frame pixels
    clips = torch.cat([texture_video(3, 120, 216, seed=s) for s in (5, 6, 7)]).to(DEV)
    ex = [torch.tensor([[50.0, 40.0], [100.0, 60.0]]), torch.zeros(0, 2), torch.tensor([[10.0, 10.0]])]
    many = detect_corners(clips, 100, frame=1, exclude=ex, exclude_radius=20, block_size=5)
    for b in range(3):
        assert torch.equal(many[b], detect_corners(clips[b:b + 1], 100, frame=1, exclude=[ex[b]], exclude_radius=20,
                                                   block_size=5))
    # the points are the oracle's on the prepared frame, in frame pixels
    from cotracker_b200 import ingest
    f = ingest.prepare_video(u8[:, 2:3], (384, 512), DEV)[0].cpu()
    want, _ = C.corners(f.numpy(), 200)
    xy = torch.from_numpy(want).float() * torch.tensor([215 / 511, 119 / 383])
    assert torch.equal(ref[0, :, 1:].cpu(), xy)


def _predictor():
    from cotracker_b200.predictor import CoTrackerOnlinePredictor
    from cotracker_b200.synthetic import seeded_state_dict
    p = CoTrackerOnlinePredictor(checkpoint=None, window_len=S)
    p.model.load_state_dict(seeded_state_dict(53, offline=False, window_len=S, head_gain=10.0, vis_gain=100.0))
    return p.to(DEV)


def _by_hand(hub, sid, max_tracks, md):
    """seed_corners' work through the public pieces: detect on the chunk's first new frame, excluding discs around the
    stream's own tracks at the last frame (model resolution), then add_tracks."""
    from cotracker_b200 import ingest
    s = hub._streams[sid]
    st, chunk = s["state"], hub._pending[sid]
    frame = ingest.prepare_video(chunk[:, st.length - st.ind:st.length - st.ind + 1], (384, 512), DEV)
    n_keep, scale = s["out"]
    ex = None
    if st.length:
        c = st.hist[0]
        row = (st.length - 1) % c.shape[0] if st.history is not None else st.length - 1
        ex = (c[row, :n_keep][None].contiguous(), [n_keep])
    found, counts = engine.detect_corners(frame, corners.params(max_tracks, 0.01, md, 3, md), ex)
    n = int(counts[0])
    if n == 0:
        return []
    xy = (found[0, :n] * found.new_tensor(scale)).double()
    return hub.add_tracks(sid, torch.cat([xy.new_full((n, 1), float(st.length)), xy], 1)[None])


def test_seed_corners_equals_detect_and_add_by_hand():
    from cotracker_b200.streams import OnlineStreams
    from cotracker_b200.synthetic import texture_video
    p = _predictor()
    video = texture_video(40, 96, 128, seed=2, shift=(2, 1)).to(DEV)
    hubs = [OnlineStreams(p), OnlineStreams(p)]
    sids = [h.open(frame_size=(96, 128), grid_size=3, history=h_) for h in hubs for h_ in (None, 8)]
    for k in range(4):
        for h, pair in zip(hubs, (sids[:2], sids[2:])):
            for sid in pair:
                h.push(sid, video[:, STEP * k:STEP * k + S])
        for a, b in zip(sids[:2], sids[2:]):
            assert hubs[0].length(a) == hubs[1].length(b)
            ids = hubs[0].seed_corners(a, 12, min_distance=8)
            assert ids == _by_hand(hubs[1], b, 12, 8)
            assert len(ids) <= 12
        out = [h.step() for h in hubs]
        for a, b in zip(sids[:2], sids[2:]):
            assert hubs[0].track_ids(a) == hubs[1].track_ids(b)
            assert all(torch.equal(x, y) for x, y in zip(out[0][a], out[1][b]))
    assert len(hubs[0].track_ids(sids[0])) > 9


def test_bounded_stream_reseeded_every_step():
    from cotracker_b200.streams import OnlineStreams
    from cotracker_b200.synthetic import texture_video
    p = _predictor()
    video = texture_video(8 * 21 + S, 96, 128, seed=3, shift=(3, 1)).to(DEV)
    hub = OnlineStreams(p)
    sid = hub.open(frame_size=(96, 128), grid_size=2, history=8)
    mem = []
    for k in range(20):
        hub.push(sid, video[:, STEP * k:STEP * k + S])
        new = hub.seed_corners(sid, 6, min_distance=6)
        assert len(new) <= 6
        ids = hub.track_ids(sid)
        if len(ids) > 24:                      # a service retires what it no longer needs
            hub.retire_tracks(sid, ids[:len(ids) - 24])
        out = hub.step()[sid]
        assert out[0].shape[1] == min(8, hub.length(sid))
        torch.cuda.synchronize()
        mem.append(torch.cuda.memory_allocated(DEV))
    assert max(mem[10:]) <= max(mem[:10]) + (1 << 20), mem


def test_snapshot_after_seed_continues_bit_for_bit():
    from cotracker_b200.streams import OnlineStreams
    from cotracker_b200.synthetic import texture_video
    p = _predictor()
    video = texture_video(48, 96, 128, seed=5).to(DEV)
    hub = OnlineStreams(p)
    sid = hub.open(frame_size=(96, 128), grid_size=3, history=8)
    for k in range(2):
        hub.push(sid, video[:, STEP * k:STEP * k + S])
        assert hub.seed_corners(sid, 10, min_distance=6)
        hub.step()
    snap = hub.snapshot(sid)
    other = OnlineStreams(p)
    sid2 = other.restore(snap)
    for k in range(2, 4):
        hub.push(sid, video[:, STEP * k:STEP * k + S])
        other.push(sid2, video[:, STEP * k:STEP * k + S])
        assert hub.seed_corners(sid, 5, min_distance=6) == other.seed_corners(sid2, 5, min_distance=6)
        a, b = hub.step()[sid], other.step()[sid2]
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_seed_corners_with_no_corner_leaves_the_stream():
    from cotracker_b200.streams import OnlineStreams
    p = _predictor()
    hub = OnlineStreams(p)
    sid = hub.open(frame_size=(96, 128), grid_size=2)
    hub.push(sid, torch.full((1, S, 3, 96, 128), 90.0, device=DEV))
    before = (hub.track_ids(sid), hub.pool.qcoords.clone())
    assert hub.seed_corners(sid, 10) == []
    assert hub.track_ids(sid) == before[0] and torch.equal(hub.pool.qcoords, before[1])
    hub.step()
