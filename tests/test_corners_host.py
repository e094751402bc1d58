"""CPU tests of corner detection: the float64 restatement (tests/corner_cases.py) against real
cv2.goodFeaturesToTrack, its own rules (border, tie order, min_distance below 1, degenerate frames), the argument checks
of detect_corners and OnlineStreams.seed_corners before any device work, and the ABI surface of ct3_detect_corners."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import corner_cases as C
from cotracker_b200 import corners, detect_corners, engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
S = 16


def apple_frames(idx=(0, 25, 49), hw=(384, 512)):
    """Frames of the apple clip prepared on the CPU as the library prepares them: [n,3,384,512] fp32 in [-1, 1]."""
    v = np.load(os.path.join(ROOT, "tests", "golden", "apple_frames_120x216.npz"))["frames"]
    x = torch.from_numpy(v[list(idx)]).permute(0, 3, 1, 2).float()
    return 2 * (F.interpolate(x, hw, mode="bilinear", align_corners=True) / 255) - 1


def test_restatement_agrees_with_cv2():
    """The restatement is Shi-Tomasi: the points cv2 picks on the same fp32 gray.  cv2 computes in fp32, so near-ties
    and near-threshold pixels may differ; the observed agreement is recorded in DESIGN.md."""
    cv2 = pytest.importorskip("cv2")
    frames = list(apple_frames()) + [C.textured_frame(384, 512, seed=s) for s in (1, 2)]
    same = total = 0
    for f in frames:
        for q, md, b, m in ((0.01, 10, 3, 300), (0.001, 5, 5, 1000), (0.3, 0, 7, 100)):
            got, _ = C.corners(f.numpy(), m, q, md, b)
            ref = cv2.goodFeaturesToTrack(C.gray(f.numpy()), m, q, md, blockSize=b, useHarrisDetector=False)
            ref = np.zeros((0, 2), np.int64) if ref is None else ref.reshape(-1, 2).astype(np.int64)
            total += max(len(got), len(ref))
            same += len(set(map(tuple, got.tolist())) & set(map(tuple, ref.tolist())))
    assert total > 1000 and same / total > 0.95, (same, total)


def test_border_and_maximum_rules():
    f = C.textured_frame(97, 131, seed=3).numpy()
    got, lam = C.corners(f, 10 ** 6, 0.001, 0)
    H, W = lam.shape
    x, y = got[:, 0], got[:, 1]
    assert len(got) > 50
    assert x.min() >= 1 and y.min() >= 1 and x.max() <= W - 2 and y.max() <= H - 2
    for xi, yi in got:
        assert lam[yi, xi] == lam[yi - 1:yi + 2, xi - 1:xi + 2].max() and lam[yi, xi] > 0.001 * lam.max()
    vals = lam[y, x]
    assert np.all(np.diff(vals) <= 0)


def test_ties_go_to_the_larger_raster_index():
    f = C.checkerboard(64, 96, period=8).numpy()
    got, lam = C.corners(f, 10 ** 6, 0.01, 0)
    vals = lam[got[:, 1], got[:, 0]]
    idx = got[:, 1] * 96 + got[:, 0]
    assert len(np.unique(vals)) < len(vals) // 10          # thousands of equal responses
    for a in range(len(got) - 1):
        assert vals[a] > vals[a + 1] or idx[a] > idx[a + 1]


def test_min_distance_below_one_keeps_the_first_candidates():
    f = C.textured_frame(64, 80, seed=4).numpy()
    every, _ = C.corners(f, 10 ** 6, 0.001, 0)
    for md in (0.5, 1):
        got, _ = C.corners(f, 40, 0.001, md)
        assert np.array_equal(got, every[:40])
    spaced, _ = C.corners(f, 10 ** 6, 0.001, 10)
    d2 = ((spaced[:, None] - spaced[None]) ** 2).sum(-1) + np.eye(len(spaced), dtype=np.int64) * 100
    assert d2.min() >= 100


def test_degenerate_frames():
    flat = np.zeros((3, 32, 40), np.float32) + 0.25
    assert len(C.corners(flat, 10)[0]) == 0
    one = flat.copy()
    one[:, 15, 20] = 1.0
    got, _ = C.corners(one, 10, 0.01, 10)
    assert got.tolist() == [[20, 15]]


def test_exclusion_mask_is_a_set_of_discs():
    m = C.exclusion_mask(20, 30, np.array([[10.5, 5.0]], np.float32), 3)
    assert m[5, 10] == 0 and m[5, 8] == 0 and m[5, 13] == 0 and m[5, 14] == 1 and m[8, 11] == 1
    assert C.exclusion_mask(20, 30, np.array([[10.0, 5.0]]), 0).all()


def test_detect_corners_rejects_bad_arguments_without_gpu():
    v = torch.zeros(1, 4, 3, 48, 64, dtype=torch.uint8)
    bad = [
        dict(max_corners=0), dict(max_corners=2.0), dict(max_corners=True),
        dict(quality_level=0), dict(quality_level=1.5), dict(quality_level=float("nan")),
        dict(min_distance=-1), dict(min_distance=float("inf")),
        dict(block_size=4), dict(block_size=9), dict(exclude_radius=-0.5),
        dict(frame=4), dict(frame=-1), dict(frame=1.0),
        dict(interp_shape=(2, 512)), dict(interp_shape=(384,)),
        dict(exclude=torch.zeros(2, 3, 2)), dict(exclude=torch.zeros(1, 3, 3)), dict(exclude=[torch.zeros(3, 2)] * 2),
        dict(exclude=[torch.zeros(3)]),
        dict(video=torch.zeros(1, 4, 2, 48, 64)), dict(video=torch.zeros(4, 3, 48, 64)),
        dict(video=torch.zeros(1, 4, 3, 1, 64)), dict(video=np.zeros((1, 4, 3, 48, 64))),
    ]
    for kw in bad:
        args = dict(video=v, max_corners=kw.pop("max_corners", 10))
        args["video"] = kw.pop("video", v)
        with pytest.raises(ValueError):
            detect_corners(args["video"], args["max_corners"], **kw)


def _hub():
    from cotracker_b200.predictor import CoTrackerOnlinePredictor
    from cotracker_b200.streams import OnlineStreams
    return OnlineStreams(CoTrackerOnlinePredictor(checkpoint=None, window_len=S))


def test_seed_corners_rejects_bad_arguments_without_gpu():
    hub = _hub()
    state = hub.pool.open(torch.zeros(3, dtype=torch.int32), torch.zeros(3, 2))
    hub._streams[0] = dict(state=state, hw=(96, 128), out=(3, (1.0, 1.0)), ids=[0, 1, 2], next_id=3)
    with pytest.raises(KeyError):
        hub.seed_corners(5, 10)
    for kw in (dict(max_tracks=0), dict(quality_level=2.0), dict(block_size=2), dict(min_distance=-3),
               dict(exclude_radius=-1)):
        with pytest.raises(ValueError):
            hub.seed_corners(0, **dict(dict(max_tracks=10), **kw))
    with pytest.raises(ValueError, match="no pending chunk"):
        hub.seed_corners(0, 10)
    # a chunk that adds no frame: the stream has passed every frame of it
    state.ind, state.length = 8, 16
    hub._pending[0] = torch.zeros(1, 8, 3, 96, 128)
    with pytest.raises(ValueError, match="adds no frame"):
        hub.seed_corners(0, 10)
    assert hub.track_ids(0) == [0, 1, 2]


def test_params_carry_doubles():
    p = corners.params(300, 0.01, 10, 5, 2.5)
    assert (p.max_corners, p.block_size, p.quality_level, p.min_distance, p.exclude_radius) == (300, 5, 0.01, 10.0, 2.5)
    assert ctypes.sizeof(engine.CornerParams) == 32


def test_detect_corners_exported_and_declared():
    lib = engine.lib()
    with open(os.path.join(ROOT, "include", "ct3_b200.h")) as f:
        header = f.read()
    for name in ("ct3_detect_corners", "ct3_corners_workspace_bytes"):
        assert hasattr(lib, name) and name in engine.EXPORTED_SYMBOLS
        assert re.search(rf"int {name}\(", header)
    assert lib.ct3_version() == 102
    n = engine.corners_workspace_bytes(3, 384, 512)
    assert 28 * 3 * 384 * 512 <= n <= 28 * 3 * 384 * 512 + 8192


def test_detect_corners_rejects_bad_arguments_in_the_library():
    """Each invalid argument returns CT3_EINVAL (or CT3_ENOSPC for the workspace) with a message before any launch
    (fake pointers, legacy stream: reaching a launch would fail differently)."""
    lib = engine.lib()
    fr, out, cnt, ws = (ctypes.c_void_p(1 << s) for s in (20, 24, 26, 28))
    H, W, K = 48, 64, 2
    need = engine.corners_workspace_bytes(K, H, W)

    def call(params=None, counts=None, **kw):
        a = dict(fr=fr, stride=3 * H * W, K=K, H=H, W=W, ex=None, E=0, out=out, cnt=cnt, ws=ws, n=need)
        a.update(kw)
        ps = params or [corners.params(10)] * a["K"] if a["K"] > 0 else [corners.params(10)]
        table = (engine.CornerParams * max(1, len(ps)))(*ps)
        c = None if counts is None else (ctypes.c_int32 * len(counts))(*counts)
        return lib.ct3_detect_corners(a["fr"], a["stride"], a["K"], a["H"], a["W"], table, a["ex"], c, a["E"], a["out"],
                                      a["cnt"], a["ws"], a["n"], None)

    def raw(**kw):
        d = dict(max_corners=10, block_size=3, quality_level=0.01, min_distance=10.0, exclude_radius=0.0)
        d.update(kw)
        return engine.CornerParams(**d)

    cases = [
        (dict(fr=None), b"null argument"), (dict(out=None), b"null argument"), (dict(ws=None), b"null argument"),
        (dict(K=0), b"K must be"), (dict(K=65536), b"K must be"), (dict(H=0), b"must be >= 1"),
        (dict(H=65536, W=65536), b"frame plane too large"), (dict(ws=ctypes.c_void_p((1 << 28) + 8)), b"aligned"),
        (dict(stride=-1), b"frame_stride"), (dict(stride=2 ** 62), b"stride extent"), (dict(E=-1), b"E_max"),
        (dict(params=[raw(block_size=4)] * K), b"block_size must be 3, 5 or 7"),
        (dict(params=[raw(), raw(block_size=7)], H=6), b">= block_size"),
        (dict(params=[raw(quality_level=0.0)] * K), b"quality_level"),
        (dict(params=[raw(quality_level=1.01)] * K), b"quality_level"),
        (dict(params=[raw(quality_level=float("nan"))] * K), b"quality_level"),
        (dict(params=[raw(max_corners=0)] * K), b"max_corners"),
        (dict(params=[raw(min_distance=-1.0)] * K), b"min_distance"),
        (dict(params=[raw(min_distance=float("inf"))] * K), b"min_distance"),
        (dict(params=[raw(exclude_radius=float("nan"))] * K), b"exclude_radius"),
        (dict(counts=[1, 0], E=0), b"exclude_counts"), (dict(counts=[-1, 0], E=4), b"exclude_counts"),
        (dict(counts=[1, 0], E=4), b"without the exclude buffer"),
    ]
    for kw, msg in cases:
        assert call(**kw) == -1, kw
        assert msg in lib.ct3_last_error(), (kw, lib.ct3_last_error())
    assert call(n=need - 1) == -3 and b"workspace too small" in lib.ct3_last_error()
    size = ctypes.c_size_t(0)
    assert lib.ct3_corners_workspace_bytes(0, H, W, ctypes.byref(size)) == -1
    assert lib.ct3_corners_workspace_bytes(1, 2 ** 20, 2 ** 12, ctypes.byref(size)) == -1
    assert lib.ct3_corners_workspace_bytes(1, H, W, None) == -1
