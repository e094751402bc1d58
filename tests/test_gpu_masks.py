"""GPU tests of region masks: ct3_detect_corners_masked is bit-identical to the float64 restatement of
tests/mask_cases.py (responses, corners, counts) on empty, full, one-pixel and plateau-cutting masks, a candidate
suppressed from outside its mask, exclusion discs and batches of frames with different masks; a full mask gives what
ct3_detect_corners gives; ct3_prepare_masks is torch.equal to ATen's nearest resize for every dtype, odd ratios and
strided input; detect_corners(mask=) takes every mask form; a stream opened with a grid and a mask, the online predictor
started with one, seed_grid and seed_corners(mask=) are torch.equal to the same points given as queries, and a stream
seeded this way snapshots and restores bit for bit."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import corner_cases as C
import mask_cases as M
from cotracker_b200 import corners, detect_corners, engine

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
S, STEP = 16, 8
HW = (384, 512)          # the model resolution: frame pixels are model pixels, the query scale is exactly 1


def _apple(idx=(0, 25)):
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    v = np.load(os.path.join(root, "tests", "golden", "apple_frames_120x216.npz"))["frames"]
    x = torch.from_numpy(v[list(idx)]).permute(0, 3, 1, 2).float()
    return (2 * (F.interpolate(x, HW, mode="bilinear", align_corners=True) / 255) - 1).contiguous()


def _run(frames, par, region=None, exclude=None):
    """frames [K,3,H,W] and region [K,H,W] uint8 on the device -> (corners, counts, responses) on the host."""
    K, _, H, W = frames.shape
    ws = torch.empty(engine.corners_workspace_bytes(K, H, W), dtype=torch.uint8, device=DEV)
    found, counts = engine.detect_corners(frames, par, exclude, workspace=ws, mask=region)
    lam = ws[:K * H * W * 8].view(torch.float64).view(K, H, W)
    return found.cpu(), counts.cpu(), lam.cpu()


def _check(frame, region, par, excl=None):
    """One frame and its region on the device against the restatement: responses, corners and count equal."""
    ex = None if excl is None else (torch.as_tensor(excl, dtype=torch.float32, device=DEV)[None], [len(excl)])
    reg = torch.as_tensor(np.ascontiguousarray(region), dtype=torch.uint8, device=DEV)[None]
    found, counts, lam = _run(frame.to(DEV)[None], [par], reg, ex)
    want, want_lam = M.corners_masked(frame.cpu().numpy(), region, par.max_corners, par.quality_level,
                                      par.min_distance, par.block_size, excl, par.exclude_radius)
    assert torch.equal(lam[0], torch.from_numpy(want_lam))
    n = int(counts[0])
    assert n == len(want)
    assert torch.equal(found[0, :n], torch.from_numpy(want).float())
    assert not found[0, n:].any()
    return want, want_lam


def test_mask_edge_cases_equal_restatement():
    for f in list(_apple()) + [C.textured_frame(97, 131, seed=3)]:
        H, W = f.shape[1:]
        lam = C.response(C.gray(f.numpy()), 3)
        full = np.ones((H, W), np.uint8)
        for par in (corners.params(300, 0.01, 10), corners.params(10 ** 5, 0.3, 0, 5), corners.params(50, 1e-3, 3.5, 7)):
            assert len(_check(f, np.zeros((H, W), np.uint8), par)[0]) == 0
            got, _ = _check(f, full, par)
            plain = _run(f.to(DEV)[None], [par])                           # ct3_detect_corners
            assert np.array_equal(got, C.corners(f.numpy(), par.max_corners, par.quality_level, par.min_distance,
                                                 par.block_size)[0])
            n = int(plain[1][0])
            assert n == len(got) and torch.equal(plain[0][0, :n], torch.from_numpy(got).float())
            for region in (M.disc(H, W, H // 2, W // 3, min(H, W) // 3), M.box(H, W, 5, H - 20, W // 2, W - 1),
                           M.without_global_max(lam, min(H, W) // 4)):
                _check(f, region, par)
        # the global maximum left out: corners weaker than q times it come back
        q = 0.3
        got, lb = _check(f, M.without_global_max(lam, min(H, W) // 4), corners.params(10 ** 5, q, 0))
        assert len(got) and lb[got[:, 1], got[:, 0]].min() < q * lb.max()


def test_single_pixel_masks():
    f = C.textured_frame(64, 80, seed=4)
    lam = C.response(C.gray(f.numpy()), 3)
    H, W = lam.shape
    pad = np.pad(lam, 1, mode="edge")
    nbr = np.max(np.stack([pad[1 + a:H + 1 + a, 1 + b:W + 1 + b] for a in (-1, 0, 1) for b in (-1, 0, 1)]), 0)
    inner = np.zeros((H, W), bool)
    inner[2:-2, 2:-2] = True
    ys, xs = np.nonzero(inner & (lam > 0) & (lam < nbr))               # suppressed by a larger neighbour
    for y, x in zip(ys[:5], xs[:5]):
        assert len(_check(f, M.box(H, W, y, y + 1, x, x + 1), corners.params(10, 0.01, 0))[0]) == 0
    ys, xs = np.nonzero(inner & (lam > 0) & (lam == nbr))              # a local maximum: itself alone
    for y, x in zip(ys[:5], xs[:5]):
        got, _ = _check(f, M.box(H, W, y, y + 1, x, x + 1), corners.params(10, 0.5, 0))
        assert got.tolist() == [[x, y]]
        assert len(_check(f, M.box(H, W, y, y + 1, x, x + 1), corners.params(10, 1.0, 0))[0]) == 0   # lambda > lambda
    # a border pixel is never a candidate, even alone in its mask
    assert len(_check(f, M.box(H, W, 0, 1, 10, 11), corners.params(10, 0.01, 0))[0]) == 0


def test_mask_cuts_through_plateaus():
    """Checkerboard plateaus of equal responses cut by the mask: the tie rule decides what is kept."""
    for period, md in ((8, 0), (8, 10), (5, 3), (6, 1.5)):
        f = C.checkerboard(192, 256, period)
        H, W = 192, 256
        for region in (M.box(H, W, 13, 151, 29, 203), (np.add.outer(np.arange(H), np.arange(W)) % 7 < 4).astype(np.uint8),
                       (np.add.outer(np.arange(H), -np.arange(W)) > -60).astype(np.uint8)):
            want, _ = _check(f, region, corners.params(10 ** 5, 0.01, md, 3))
            assert len(want) > 20


def test_masks_with_exclusion_discs():
    f = C.textured_frame(192, 256, seed=7)
    region = M.disc(192, 256, 90, 120, 70)
    full, _ = _check(f, region, corners.params(500, 0.001, 5))
    pts = [[float(x) + 0.25, float(y) - 0.5] for x, y in full[::3]]
    for r in (0.0, 4.0, 12.5):
        got, _ = _check(f, region, corners.params(500, 0.001, 5, 3, r), pts)
        if r == 0:
            assert np.array_equal(got, full)
        else:
            assert len(set(map(tuple, got.tolist())) & set(map(tuple, full[::3].tolist()))) == 0


def test_batch_of_frames_with_different_masks():
    H, W = 120, 160
    frames = torch.stack([C.textured_frame(H, W, seed=s) for s in range(4)] + [C.checkerboard(H, W, 6)]).to(DEV)
    regions = np.stack([M.disc(H, W, 60, 80, 50), np.zeros((H, W), np.uint8), np.ones((H, W), np.uint8),
                        M.box(H, W, 3, 90, 17, 121), M.box(H, W, 30, 31, 40, 41)])
    pars = [corners.params(300, 0.01, 10, 3), corners.params(7, 0.3, 0, 5), corners.params(1000, 1e-3, 2.5, 7, 3),
            corners.params(50, 0.05, 37, 3, 9), corners.params(2000, 0.01, 0.5, 5)]
    E = 12
    g = torch.Generator().manual_seed(0)
    pts = torch.rand(5, E, 2, generator=g) * torch.tensor([W - 1.0, H - 1.0])
    cnt = [0, 12, 5, 3, 1]
    reg = torch.from_numpy(regions).to(DEV)
    found, counts, lam = _run(frames, pars, reg, (pts.to(DEV), cnt))
    for k in range(5):
        want, want_lam = M.corners_masked(frames[k].cpu().numpy(), regions[k], pars[k].max_corners,
                                          pars[k].quality_level, pars[k].min_distance, pars[k].block_size,
                                          pts[k, :cnt[k]].numpy(), pars[k].exclude_radius)
        n = int(counts[k])
        assert n == len(want) and torch.equal(lam[k], torch.from_numpy(want_lam))
        assert torch.equal(found[k, :n], torch.from_numpy(want).float()) and not found[k, n:].any()
    # one mask for every frame (mask stride 0) equals its copies
    one = reg[3:4].expand(5, H, W)
    assert one.stride(0) == 0
    a, b = _run(frames, pars, one), _run(frames, pars, one.contiguous())
    assert all(torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("src_hw", [(720, 1296), (37, 53), (384, 512), (192, 256), (1000, 1500), (5, 7), (448, 600),
                                    (896, 1200), (200, 300), (1, 1)])
def test_prepare_masks_equals_aten(src_hw):
    H, W = src_hw
    g = torch.Generator().manual_seed(H * 7 + W)
    vals = torch.randint(0, 3, (3, H, W), generator=g)
    at_model = None
    for out_hw in ((384, 512), (97, 131), (H * 2, W * 2)):
        want = None
        for dtype in (torch.uint8, torch.bool, torch.float32):
            src = (vals != 0) if dtype == torch.bool else vals.to(dtype)
            if dtype == torch.float32:   # values ATen keeps or drops: NaN is nonzero, -0 is zero, tiny values count
                src = torch.where(vals == 1, torch.tensor(float("nan")), torch.where(vals == 2, 1e-30, -0.0))
            src = src.to(DEV)
            ref = (F.interpolate(src[:, None].float(), out_hw, mode="nearest")[:, 0] != 0).to(torch.uint8)
            if want is None:
                want = ref
                at_model = ref if at_model is None else at_model
            assert torch.equal(ref, want)
            assert torch.equal(engine.prepare_masks(src, out_hw), ref)
            # strided: transposed planes, every other column, a channels-last slice
            t = src.transpose(1, 2).contiguous().transpose(1, 2)
            assert t.is_contiguous() == (min(H, W) == 1) and torch.equal(engine.prepare_masks(t, out_hw), ref)
            wide = torch.zeros(3, H, 2 * W, dtype=src.dtype, device=DEV)
            wide[:, :, ::2] = src
            assert torch.equal(engine.prepare_masks(wide[:, :, ::2], out_hw), ref)
            cl = torch.zeros(H, W, 4, dtype=src.dtype, device=DEV)
            cl[..., 1] = src[1]
            assert torch.equal(engine.prepare_masks(cl[None, ..., 1], out_hw), ref[1:2])
    if (H, W) in ((448, 600), (896, 1200), (200, 300)):   # ATen's fp32 index, not floor(d * H / 384)
        assert not np.array_equal(M.nearest_index(384, H), M.exact_index(384, H))
        assert np.array_equal(at_model[0].cpu().numpy(), M.resize_mask(vals[0].numpy(), (384, 512)))


def test_detect_corners_mask_forms():
    from cotracker_b200 import ingest
    from cotracker_b200.synthetic import texture_video
    H, W = 120, 216
    clips = torch.cat([texture_video(3, H, W, seed=s) for s in (4, 5)]).to(DEV)     # [2,3,3,H,W]
    m = torch.from_numpy(M.disc(H, W, 60, 100, 45))[None, None]
    ref = detect_corners(clips[:1], 200, frame=1, mask=m)
    assert ref.shape[1] > 5
    for form in (m.to(DEV), m.bool(), m.float().to(DEV), m.double() * 0.5, m.to(torch.int64).to(DEV)):
        assert torch.equal(detect_corners(clips[:1], 200, frame=1, mask=form), ref)
    # the queries are the restatement's on the prepared frame and the resized mask, in frame pixels
    f = ingest.prepare_video(clips[:1, 1:2], (384, 512), DEV)[0].cpu()
    want, _ = M.corners_masked(f.numpy(), M.resize_mask(m[0, 0].numpy(), (384, 512)), 200)
    xy = torch.from_numpy(want).float() * torch.tensor([(W - 1) / 511, (H - 1) / 383])
    assert torch.equal(ref[0, :, 1:].cpu(), xy.to(ref.dtype))
    # one mask for both clips, and a mask per clip, equal single calls
    both = detect_corners(clips, 200, frame=1, mask=m)
    assert torch.equal(both[0], ref) and torch.equal(both[1], detect_corners(clips[1:], 200, frame=1, mask=m))
    per = torch.cat([m, 1 - m])
    two = detect_corners(clips, 200, frame=1, mask=per, exclude=[torch.zeros(0, 2), torch.tensor([[50.0, 50.0]])],
                         exclude_radius=9)
    assert torch.equal(two[0], ref)
    assert torch.equal(two[1], detect_corners(clips[1:], 200, frame=1, mask=1 - m, exclude=[torch.tensor([[50.0, 50.0]])],
                                              exclude_radius=9))
    assert detect_corners(clips[:1], 200, frame=1, mask=torch.zeros(1, 1, H, W)).shape == (1, 0, 3)


def _predictor():
    from cotracker_b200.predictor import CoTrackerOnlinePredictor
    from cotracker_b200.synthetic import seeded_state_dict
    p = CoTrackerOnlinePredictor(checkpoint=None, window_len=S)
    p.model.load_state_dict(seeded_state_dict(53, offline=False, window_len=S, head_gain=10.0, vis_gain=100.0))
    return p.to(DEV)


def _kept(grid_size, region):
    """The grid points [1,m,2] at model resolution that region [384,512] keeps: read at (round(y), round(x))."""
    from cotracker_b200.predictor import get_points_on_a_grid
    pts = get_points_on_a_grid(grid_size, HW)
    keep = torch.from_numpy(region)[pts[0, :, 1].round().long(), pts[0, :, 0].round().long()] != 0
    return pts[:, keep]


def _equal(a, b):
    return len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b))


def test_open_with_segm_mask_equals_queries():
    from cotracker_b200.streams import OnlineStreams
    from cotracker_b200.synthetic import texture_video
    p = _predictor()
    video = texture_video(S + 2 * STEP, *HW, seed=2, shift=(2, 1)).to(DEV)
    region = M.disc(*HW, 200, 230, 120)
    mask = torch.from_numpy(region)[None, None]
    hub = OnlineStreams(p)
    for support in (False, True):
        pts = _kept(12, region)
        assert 0 < pts.shape[1] < 144
        q = torch.cat([torch.full_like(pts[:, :, :1], 3.0), pts], 2)
        a = hub.open(HW, grid_size=12, grid_query_frame=3, segm_mask=mask.to(DEV), add_support_grid=support)
        b = hub.open(HW, queries=q, add_support_grid=support)
        assert hub.track_ids(a) == hub.track_ids(b) == list(range(pts.shape[1]))
        for k in range(3):
            for sid in (a, b):
                hub.push(sid, video[:, STEP * k:STEP * k + S])
            out = hub.step(return_scores=True)
            assert out[a][0].shape[2] == pts.shape[1]
            assert torch.equal(out[a][0], out[b][0]) and torch.equal(out[a][1], out[b][1])
            assert _equal(out[a][2], out[b][2])
        hub.close(a)
        hub.close(b)
    with pytest.raises(ValueError, match="keeps none"):
        hub.open(HW, grid_size=12, segm_mask=torch.zeros(1, 1, *HW))
    # the online predictor: the same first-step argument, the same results
    outs = []
    for kw in (dict(grid_size=12, segm_mask=mask), dict(queries=torch.cat([torch.zeros_like(_kept(12, region)[:, :, :1]),
                                                                            _kept(12, region)], 2))):
        p(video[:, :S], is_first_step=True, add_support_grid=True, **kw)
        outs.append([p(video[:, STEP * k:STEP * k + S], add_support_grid=True) for k in range(3)])
    for x, y in zip(*outs):
        assert _equal(x, y)


def _by_hand_corners(hub, sid, region, max_tracks, md):
    """seed_corners(mask=) through public pieces: detect in the chunk's first new frame inside the mask, excluding
    discs around the stream's tracks at the last frame, then add_tracks."""
    from cotracker_b200 import ingest
    s = hub._streams[sid]
    st, chunk = s["state"], hub._pending[sid]
    frame = ingest.prepare_video(chunk[:, st.length - st.ind:st.length - st.ind + 1], HW, DEV)
    n_keep, scale = s["out"]
    ex = None
    if st.length:
        c = st.hist[0]
        row = (st.length - 1) % c.shape[0] if st.history is not None else st.length - 1
        ex = (c[row, :n_keep][None].contiguous(), [n_keep])
    reg = torch.from_numpy(region).to(DEV)[None]
    found, counts = engine.detect_corners(frame, corners.params(max_tracks, 0.01, md, 3, md), ex, mask=reg)
    n = int(counts[0])
    if n == 0:
        return []
    xy = (found[0, :n] * found.new_tensor(scale)).double()
    return hub.add_tracks(sid, torch.cat([xy.new_full((n, 1), float(st.length)), xy], 1)[None])


def test_seed_grid_and_seed_corners_equal_add_tracks_and_restore():
    from cotracker_b200.streams import OnlineStreams
    from cotracker_b200.synthetic import texture_video
    p = _predictor()
    video = texture_video(S + 6 * STEP, *HW, seed=5, shift=(1, 2)).to(DEV)
    hubs = [OnlineStreams(p), OnlineStreams(p)]
    sids = [h.open(HW, grid_size=4, history=h_) for h in hubs for h_ in (None, 12)]
    regions = [M.disc(*HW, 150 + 20 * k, 200 + 30 * k, 90) for k in range(4)]
    for k in range(4):
        for h, pair in zip(hubs, (sids[:2], sids[2:])):
            for sid in pair:
                h.push(sid, video[:, STEP * k:STEP * k + S])
        for a, b in zip(sids[:2], sids[2:]):
            mask = torch.from_numpy(regions[k])[None, None]
            ids = hubs[0].seed_grid(a, 9, segm_mask=mask.to(DEV) if k % 2 else mask)
            pts = _kept(9, regions[k])
            q = torch.cat([torch.full_like(pts[:, :, :1], float(hubs[1].length(b))), pts], 2)
            assert ids == hubs[1].add_tracks(b, q) and len(ids) == pts.shape[1] > 0
            ids = hubs[0].seed_corners(a, 10, min_distance=8, mask=mask)
            assert ids == _by_hand_corners(hubs[1], b, regions[k], 10, 8) and len(ids) > 0
        out = [h.step() for h in hubs]
        for a, b in zip(sids[:2], sids[2:]):
            assert hubs[0].track_ids(a) == hubs[1].track_ids(b)
            assert _equal(out[0][a], out[1][b])
    # nothing in the mask: the stream is unchanged
    empty = torch.zeros(1, 1, *HW)
    before = hubs[0].track_ids(sids[0])
    assert hubs[0].seed_grid(sids[0], 9, segm_mask=empty) == []
    hubs[0].push(sids[0], video[:, STEP * 4:STEP * 4 + S])
    assert hubs[0].seed_corners(sids[0], 10, mask=empty) == []
    assert hubs[0].track_ids(sids[0]) == before
    hubs[0].step()
    # a seeded stream parks and continues bit for bit
    sid = sids[1]
    snap = hubs[0].snapshot(sid)
    other = OnlineStreams(p)
    sid2 = other.restore(snap)
    for k in range(4, 6):
        hubs[0].push(sid, video[:, STEP * k:STEP * k + S])
        other.push(sid2, video[:, STEP * k:STEP * k + S])
        mask = torch.from_numpy(regions[k - 4])[None, None]
        assert hubs[0].seed_grid(sid, 5, segm_mask=mask) == other.seed_grid(sid2, 5, segm_mask=mask)
        assert hubs[0].seed_corners(sid, 5, mask=mask) == other.seed_corners(sid2, 5, mask=mask)
        assert _equal(hubs[0].step()[sid], other.step()[sid2])
