"""Generate tests/golden/eval_predictor_single_t24.npz by running the UNMODIFIED reference's single-point
EvaluationPredictor (cotracker/models/evaluation_predictor.py:25-199, the TAP-Vid protocol) on seeded weights and a
seeded synthetic clip: 12 queries at varied frames over 24 frames.  Run in the build container only (the GPU box has
no reference checkout):

    python oracle/make_eval_single_golden.py

Only the outputs are stored; tests/test_gpu_groups.py rebuilds the inputs from eval_single_inputs().
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF = os.environ.get("COTRACKER_REFERENCE", "/root/reference")

from cotracker_b200.synthetic import random_queries, seeded_state_dict, texture_video  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "eval_predictor_single_t24.npz")


def eval_single_inputs():
    """Seeded inputs of the golden: offline weights, a 24-frame 128x160 clip, 12 queries at varied frames."""
    sd = seeded_state_dict(61, offline=True, window_len=60, head_gain=10.0, vis_gain=100.0)
    video = texture_video(24, 128, 160, seed=62)
    queries = random_queries(12, 24, 128, 160, seed=63)
    return sd, video, queries


def main():
    sys.path.insert(0, REF)
    from cotracker.models.build_cotracker import build_cotracker
    from cotracker.models.evaluation_predictor import EvaluationPredictor
    sd, video, queries = eval_single_inputs()
    m = build_cotracker(None, offline=True, window_len=60).eval()
    m.load_state_dict(sd)
    with torch.no_grad():
        ev = EvaluationPredictor(m, single_point=True, grid_size=5, local_grid_size=8)
        tr, vi = ev(video, queries)
    out = dict(tracks=tr.numpy(), vis=vi.numpy())
    np.savez_compressed(GOLDEN, **out)
    print("eval_predictor_single_t24", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
