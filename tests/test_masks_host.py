"""CPU tests of region masks: the float64 restatement of masked corner selection (tests/mask_cases.py) against its own
three rules and against cv2.goodFeaturesToTrack(..., mask=...), ATen's nearest index rule for the mask resize, the
argument checks of the Python entry points before any device work, and the ABI surface of ct3_detect_corners_masked
and ct3_prepare_masks with their rejections before any launch."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import corner_cases as C
import mask_cases as M
from cotracker_b200 import corners, detect_corners, engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
S = 16
# mask resizes to 384 x 512 where ATen's fp32 index differs from floor(d * in / out) (found by search, checked below)
ODD_SIZES = ((448, 600), (896, 1200), (200, 300))


def apple_frames(idx=(0, 25, 49), hw=(384, 512)):
    v = np.load(os.path.join(ROOT, "tests", "golden", "apple_frames_120x216.npz"))["frames"]
    x = torch.from_numpy(v[list(idx)]).permute(0, 3, 1, 2).float()
    return 2 * (F.interpolate(x, hw, mode="bilinear", align_corners=True) / 255) - 1


def _regions(lam):
    H, W = lam.shape
    return [M.disc(H, W, H // 2, W // 2, min(H, W) // 3), M.box(H, W, 40, H - 100, 60, W // 2 + 7),
            M.without_global_max(lam), np.ones((H, W), np.uint8)]


def test_full_region_is_the_unmasked_selection():
    for f in list(apple_frames()) + [C.textured_frame(97, 131, seed=3), C.checkerboard(64, 96, 8)]:
        f = f.numpy()
        for q, md, b, m in ((0.01, 10, 3, 300), (0.001, 0, 5, 10 ** 6)):
            want, _ = C.corners(f, m, q, md, b)
            got, _ = M.corners_masked(f, np.ones(f.shape[1:], np.uint8), m, q, md, b)
            assert np.array_equal(got, want)


def test_masked_threshold_uses_the_region_maximum():
    """A region that leaves out the global maximum returns corners weaker than q times it."""
    f = apple_frames((0,))[0].numpy()
    q = 0.3
    _, lam = C.corners(f, 10, q, 0)
    region = M.without_global_max(lam, 60)
    got, _ = M.corners_masked(f, region, 10 ** 6, q, 0)
    vals = lam[got[:, 1], got[:, 0]]
    assert len(got) > 0 and (region[got[:, 1], got[:, 0]] == 1).all()
    assert vals.min() < q * lam.max() and vals.min() > q * lam[region != 0].max()


def test_neighbour_outside_the_region_suppresses():
    """A pixel inside the region whose 3x3 neighbourhood holds a larger response outside it is not returned, although
    it passes the threshold of its own (one-pixel) region."""
    f = C.textured_frame(64, 80, seed=4).numpy()
    _, lam = C.corners(f, 10, 0.01, 0)
    H, W = lam.shape
    nbr = np.max(np.stack([np.roll(np.roll(lam, a, 0), b, 1) for a in (-1, 0, 1) for b in (-1, 0, 1)]), 0)
    ys, xs = np.nonzero((lam > 0) & (lam < nbr))
    inner = (ys > 1) & (ys < H - 2) & (xs > 1) & (xs < W - 2)
    y, x = ys[inner][0], xs[inner][0]
    single = M.box(H, W, y, y + 1, x, x + 1)
    assert len(M.corners_masked(f, single, 10, 0.01, 0)[0]) == 0
    # the same pixel as a local maximum is returned alone
    peak = np.unravel_index(np.argmax(np.where(lam == nbr, lam, -1)[1:-1, 1:-1]), (H - 2, W - 2))
    py, px = peak[0] + 1, peak[1] + 1
    got, _ = M.corners_masked(f, M.box(H, W, py, py + 1, px, px + 1), 10, 0.01, 0)
    assert got.tolist() == [[px, py]]


def test_empty_region_and_candidates_inside():
    f = C.textured_frame(97, 131, seed=5).numpy()
    assert len(M.corners_masked(f, np.zeros((97, 131), np.uint8), 100)[0]) == 0
    region = M.disc(97, 131, 40, 70, 25)
    got, _ = M.corners_masked(f, region, 10 ** 6, 0.001, 0)
    assert len(got) > 10 and (region[got[:, 1], got[:, 0]] == 1).all()
    ex = got[::2].astype(np.float32) + 0.25
    excl, _ = M.corners_masked(f, region, 10 ** 6, 0.001, 0, 3, ex, 2.5)
    assert len(excl) and not set(map(tuple, excl.tolist())) & set(map(tuple, got[::2].tolist()))


def test_restatement_agrees_with_cv2_masks():
    """The masked restatement is cv2's mask semantics, on the same fp32 gray: more than 95 % of points shared, the bar
    of the unmasked test.  One region leaves out the frame's global maximum, so the masked threshold is exercised."""
    cv2 = pytest.importorskip("cv2")
    frames = list(apple_frames()) + [C.textured_frame(384, 512, seed=s) for s in (1, 2)]
    same = total = 0
    below_global = 0
    for f in frames:
        f = f.numpy()
        g = C.gray(f)
        lam = C.response(g, 3)
        for region in _regions(lam):
            for q, md, b, m in ((0.01, 10, 3, 300), (0.001, 5, 5, 1000), (0.3, 0, 7, 100)):
                got, lb = M.corners_masked(f, region, m, q, md, b)
                ref = cv2.goodFeaturesToTrack(g, m, q, md, mask=region, blockSize=b, useHarrisDetector=False)
                ref = np.zeros((0, 2), np.int64) if ref is None else ref.reshape(-1, 2).astype(np.int64)
                total += max(len(got), len(ref))
                same += len(set(map(tuple, got.tolist())) & set(map(tuple, ref.tolist())))
                if len(got):
                    below_global += int((lb[got[:, 1], got[:, 0]] <= q * lb.max()).sum())
    assert total > 1000 and same / total > 0.95, (same, total)
    assert below_global > 0


def test_nearest_index_is_atens_rule():
    for n_in, n_out in ((720, 384), (1296, 512), (37, 384), (53, 512), (384, 384), (192, 384), (5, 512), (1000, 7),
                        (448, 384), (896, 384), (200, 384), (600, 512)):
        got = F.interpolate(torch.arange(n_in, dtype=torch.float32)[None, None, None], (1, n_out), mode="nearest")
        assert np.array_equal(got[0, 0, 0].long().numpy(), M.nearest_index(n_out, n_in)), (n_in, n_out)
    # the sizes the GPU test resizes from differ from exact arithmetic somewhere
    for h, w in ODD_SIZES:
        assert (M.nearest_index(384, h) != M.exact_index(384, h)).any()
    m = (np.arange(37 * 53).reshape(37, 53) % 3 == 0).astype(np.uint8)
    want = F.interpolate(torch.from_numpy(m).float()[None, None], (384, 512), mode="nearest")[0, 0] != 0
    assert np.array_equal(M.resize_mask(m, (384, 512)), want.numpy().astype(np.uint8))


def test_python_entry_points_reject_bad_masks_without_gpu():
    v = torch.zeros(1, 4, 3, 48, 64, dtype=torch.uint8)
    for bad in (torch.zeros(1, 1, 47, 64), torch.zeros(2, 1, 48, 64), torch.zeros(1, 2, 48, 64), torch.zeros(1, 48, 64),
                torch.zeros(1, 1, 48, 64, dtype=torch.complex64), np.zeros((1, 1, 48, 64))):
        with pytest.raises(ValueError, match="mask"):
            detect_corners(v, 10, mask=bad)
    from cotracker_b200.predictor import CoTrackerOnlinePredictor
    from cotracker_b200.streams import OnlineStreams
    p = CoTrackerOnlinePredictor(checkpoint=None, window_len=S)
    ok = torch.ones(1, 1, 96, 128)
    for kw in (dict(queries=torch.zeros(1, 2, 3)), dict(grid_size=0), dict(segm_mask=torch.ones(1, 1, 96, 127))):
        args = dict(dict(queries=None, grid_size=5, segm_mask=ok), **kw)
        with pytest.raises(ValueError, match="segm_mask"):
            p._first_step_queries(1, (96, 128), args["queries"], args["grid_size"], 0, False, "cpu", args["segm_mask"])
    hub = OnlineStreams(p)
    state = hub.pool.open(torch.zeros(3, dtype=torch.int32), torch.zeros(3, 2))
    hub._streams[0] = dict(state=state, hw=(96, 128), out=(3, (1.0, 1.0)), ids=[0, 1, 2], next_id=3)
    with pytest.raises(KeyError):
        hub.seed_grid(4, 5)
    for g in (0, -1, 2.0, True):
        with pytest.raises(ValueError, match="grid_size"):
            hub.seed_grid(0, g)
    with pytest.raises(ValueError, match="segm_mask"):
        hub.seed_grid(0, 5, torch.ones(1, 1, 96, 64))
    with pytest.raises(ValueError, match="mask"):
        hub.seed_corners(0, 10, mask=torch.ones(1, 1, 48, 128))
    assert hub.track_ids(0) == [0, 1, 2]


def test_mask_entry_points_exported_and_declared():
    lib = engine.lib()
    with open(os.path.join(ROOT, "include", "ct3_b200.h")) as f:
        header = f.read()
    for name in ("ct3_detect_corners_masked", "ct3_prepare_masks"):
        assert hasattr(lib, name) and name in engine.EXPORTED_SYMBOLS
        assert re.search(rf"int {name}\(", header)
    assert lib.ct3_version() == 102
    assert ctypes.sizeof(engine.CornerParams) == 32
    assert engine.MASK_DTYPES == {torch.uint8: 0, torch.bool: 1, torch.float32: 2}


def test_detect_corners_masked_rejects_bad_arguments_in_the_library():
    """Each invalid argument returns CT3_EINVAL (CT3_ENOSPC for the workspace) with a message before any launch (fake
    pointers, legacy stream: reaching a launch would fail differently)."""
    lib = engine.lib()
    fr, out, cnt, ws, mk = (ctypes.c_void_p(1 << s) for s in (20, 24, 26, 28, 30))
    H, W, K = 48, 64, 2
    need = engine.corners_workspace_bytes(K, H, W)

    def call(params=None, **kw):
        a = dict(fr=fr, stride=3 * H * W, K=K, H=H, W=W, mask=mk, mstride=H * W, out=out, cnt=cnt, ws=ws, n=need)
        a.update(kw)
        table = (engine.CornerParams * K)(*(params or [corners.params(10)] * K))
        return lib.ct3_detect_corners_masked(a["fr"], a["stride"], a["K"], a["H"], a["W"], table, None, None, 0,
                                             a["mask"], a["mstride"], a["out"], a["cnt"], a["ws"], a["n"], None)

    cases = [
        (dict(mask=None), b"null argument"), (dict(fr=None), b"null argument"), (dict(cnt=None), b"null argument"),
        (dict(mstride=-1), b"mask_stride"), (dict(mstride=2 ** 63 - 1), b"mask stride extent"),
        (dict(K=0), b"K must be"), (dict(stride=-1), b"frame_stride"), (dict(H=2), b">= block_size"),
        (dict(params=[engine.CornerParams(10, 4, 0.01, 10.0, 0.0)] * K), b"block_size"),
        (dict(ws=ctypes.c_void_p((1 << 28) + 8)), b"aligned"),
    ]
    for kw, msg in cases:
        assert call(**kw) == -1, kw
        assert msg in lib.ct3_last_error(), (kw, lib.ct3_last_error())
    assert call(n=need - 1) == -3 and b"workspace too small" in lib.ct3_last_error()
    size = ctypes.c_size_t(0)
    assert lib.ct3_corners_workspace_bytes(K, H, W, ctypes.byref(size)) == 0 and size.value == need


def test_prepare_masks_rejects_bad_arguments_in_the_library():
    lib = engine.lib()
    src, out = ctypes.c_void_p(1 << 20), ctypes.c_void_p(1 << 24)

    def call(**kw):
        a = dict(src=src, dtype=0, K=2, H=48, W=64, sk=48 * 64, sh=64, sw=1, oh=384, ow=512, out=out)
        a.update(kw)
        return lib.ct3_prepare_masks(a["src"], a["dtype"], a["K"], a["H"], a["W"], a["sk"], a["sh"], a["sw"], a["oh"],
                                     a["ow"], a["out"], None)

    cases = [
        (dict(src=None), b"null argument"), (dict(out=None), b"null argument"), (dict(dtype=3), b"unknown mask dtype"),
        (dict(dtype=-1), b"unknown mask dtype"), (dict(K=0), b"K must be"), (dict(K=65536), b"K must be"),
        (dict(H=0), b"must be >= 1"), (dict(ow=0), b"must be >= 1"), (dict(sk=2 ** 62, K=3), b"stride extent"),
        (dict(sh=-2 ** 63), b"stride extent"), (dict(dtype=2, sw=2 ** 61), b"stride extent"),
        (dict(oh=65536, ow=65536), b"output plane too large"),
    ]
    for kw, msg in cases:
        assert call(**kw) == -1, kw
        assert msg in lib.ct3_last_error(), (kw, lib.ct3_last_error())
