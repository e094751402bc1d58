"""Evaluation harness (SURVEY 8(f4)): the numpy TAP-Vid metrics against the reference implementation's values pinned
in tests/golden/reference_host.npz and, on the GPU, EvaluationPredictor against the reference's EvaluationPredictor output pinned in a golden."""
import os

import numpy as np
import pytest
import torch

from cotracker_b200.evaluation import EvaluationPredictor, points_on_a_grid, tapvid_metrics

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _random_problem(seed, b=2, n=17, t=11):
    r = np.random.default_rng(seed)
    q = np.concatenate([r.integers(0, t, (b, n, 1)).astype(np.float64), r.uniform(0, 256, (b, n, 2))], axis=-1)
    gt = r.uniform(0, 256, (b, n, t, 2))
    pred = gt + r.normal(0, 3.0, gt.shape) * (r.uniform(size=(b, n, t, 1)) < 0.7)
    occ = r.uniform(size=(b, n, t)) < 0.3
    pocc = occ ^ (r.uniform(size=(b, n, t)) < 0.2)
    return q, occ, gt, pocc, pred


def test_perfect_prediction_scores_one():
    q, occ, gt, _, _ = _random_problem(0)
    m = tapvid_metrics(q, occ, gt, occ, gt, "strided")
    assert np.allclose(m["average_jaccard"], 1.0) and np.allclose(m["average_pts_within_thresh"], 1.0)
    assert np.isclose(m["occlusion_accuracy"].sum(), 1.0)      # the reference normalises by the batch total


def test_hand_computed_case():
    # one video, one track, 4 frames, query at frame 0 ("first": frames 1..3 scored)
    q = np.array([[[0.0, 5.0, 5.0]]])
    gt = np.array([[[[5, 5], [6, 5], [7, 5], [8, 5]]]], dtype=np.float64)
    pred = gt + np.array([0, 0.5, 3.0, 20.0])[None, None, :, None] * np.array([1.0, 0.0])
    occ = np.array([[[False, False, False, True]]])
    pocc = np.array([[[False, False, True, False]]])
    m = tapvid_metrics(q, occ, gt, pocc, pred, "first")
    assert np.isclose(m["occlusion_accuracy"][0], 1 / 3)
    assert np.isclose(m["pts_within_1"][0], 0.5) and np.isclose(m["pts_within_4"][0], 1.0)
    # thr 1: TP = frame 1; FP = frame 3 (pred visible, gt occluded) -> 1 / (2 + 1)
    assert np.isclose(m["jaccard_1"][0], 1 / 3)


@pytest.mark.parametrize("mode", ["first", "strided"])
def test_metrics_match_live_reference(mode):
    """Against the reference's compute_tapvid_metrics on the same problems (tests/golden/reference_host.npz)."""
    with np.load(os.path.join(GOLDEN, "reference_host.npz")) as z:
        for seed in range(4):
            prefix = f"tapvid_{mode}_{seed}_"
            want = {k[len(prefix):]: z[k] for k in z.files if k.startswith(prefix)}
            got = tapvid_metrics(*_random_problem(seed), mode)
            assert set(want) == set(got)
            for k in want:
                assert np.allclose(got[k], want[k], rtol=0, atol=1e-12), k


def test_grid_with_centre_matches_live_reference():
    with np.load(os.path.join(GOLDEN, "reference_host.npz")) as z:
        for i, (size, extent, centre) in enumerate(((8, (50, 50), (120.5, 77.25)), (5, (384, 512), None),
                                                    (1, (384, 512), None))):
            assert torch.equal(points_on_a_grid(size, extent, centre), torch.from_numpy(z[f"grid_{i}"]))


@pytest.mark.gpu
@pytest.mark.parametrize("single_point", [True, False])
def test_evaluation_predictor_matches_reference_golden(single_point):
    """tests/golden/eval_predictor.npz: the reference's EvaluationPredictor on a seeded clip (oracle/make_golden.py);
    tracks within 1e-3 px, and the TAP-Vid metrics of CUDA-vs-reference tracks are exactly 1."""
    from cases import load_golden
    from cotracker_b200.build import build_cotracker
    from oracle.make_golden import eval_case_inputs
    sd, video, queries = eval_case_inputs()
    want = load_golden("eval_predictor")
    model = build_cotracker(None, offline=True, window_len=60).eval()
    model.load_state_dict(sd)
    ev = EvaluationPredictor(model.to("cuda:0"), single_point=single_point, grid_size=5, local_grid_size=8)
    tracks, vis = ev(video.to("cuda:0"), queries.to("cuda:0"))
    key = "single" if single_point else "joint"
    wt, wv = want[f"tracks_{key}"], want[f"vis_{key}"]
    assert float((tracks.cpu() - wt).abs().max()) < 1e-3
    assert float((vis.cpu() - wv).abs().max()) < 1e-3
    q = queries[0].numpy()[None][..., [0, 2, 1]]                                     # (t, y, x)
    # random-init weights give visibility*confidence far below the usual 0.6 cut: threshold in the widest gap around
    # the median of the reference's values, so both classes are populated and no value sits on the threshold
    vals = np.sort(wv.numpy().ravel())
    mid = vals[len(vals) // 4: 3 * len(vals) // 4 + 1]
    i = int(np.argmax(np.diff(mid)))
    thr = 0.5 * (mid[i] + mid[i + 1])
    occ_w = (wv[0].numpy().T < thr)[None]
    occ_g = (vis[0].cpu().numpy().T < thr)[None]
    assert occ_w.any() and not occ_w.all()
    tw = wt[0].permute(1, 0, 2).numpy()[None].astype(np.float64)
    tg = tracks[0].cpu().permute(1, 0, 2).numpy()[None].astype(np.float64)
    m = tapvid_metrics(q, occ_w, tw, occ_g, tg, "first")
    assert m["average_pts_within_thresh"][0] == 1.0 and m["average_jaccard"][0] == 1.0
