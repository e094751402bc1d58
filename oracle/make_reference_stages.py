"""Pin what the stage-level and host-logic tests compare against from the UNMODIFIED reference (imported from
$COTRACKER_REFERENCE) as golden data, so those tests run on any machine:

    python oracle/make_reference_stages.py

writes tests/golden/reference_stages.npz (tests/test_oracle_vs_reference.py) and tests/golden/reference_host.npz
(tests/test_host_logic.py, tests/test_evaluation.py).  Inputs are re-created from the seeds the tests use; large
outputs (except the correlation volume, which the corr_mlp check
feeds back in) are stored as a fixed seeded sample of their elements (`<name>__idx` = flat indices, `<name>` = values) to
keep every file well under 1 MB.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
REF = os.environ.get("COTRACKER_REFERENCE", "/root/reference")
SAMPLE = 8192

from cotracker_b200.synthetic import random_queries, seeded_state_dict, texture_video  # noqa: E402


def sampled(out, name, t, full=False):
    a = t.detach().double().numpy().reshape(-1) if isinstance(t, torch.Tensor) else np.asarray(t, np.float64).reshape(-1)
    if a.size > SAMPLE and not full:
        idx = np.sort(np.random.default_rng(len(out)).choice(a.size, SAMPLE, replace=False)).astype(np.int32)
        out[name + "__idx"] = idx
        a = a[idx]
    out[name] = a.astype(np.float32)


def stages():
    from cases import stage_inputs
    from cotracker.models.build_cotracker import build_cotracker
    from cotracker.models.core.cotracker.cotracker3_online import posenc
    sd = seeded_state_dict(2024, offline=True, window_len=60, head_gain=10.0, vis_gain=100.0)
    m = build_cotracker(None, offline=True, window_len=60).eval()
    m.load_state_dict(sd)
    x = stage_inputs()
    out = {}
    with torch.no_grad():
        sampled(out, "updateformer", m.updateformer(x["uf_x"]))
        feat = m.get_correlation_feat(x["corr_fm"], x["corr_coords"])
        N = x["corr_sup"].shape[2]
        s = x["corr_sup"].view(1, 1, 7, 7, N, 128).squeeze(1).permute(0, 3, 1, 2, 4)
        vol = torch.einsum("btnhwc,bnijc->btnhwij", feat, s).reshape(-1, N, 2401)
        sampled(out, "corr_volume", vol, full=True)        # also the exact input of the corr_mlp comparison
        sampled(out, "corr_mlp_big", m.corr_mlp(vol * 10))
        _, sup = m.get_track_feat(x["sup_fm"], x["sup_qf"], x["sup_qc"], support_radius=3)
        sampled(out, "support", sup[0])
        out["posenc"] = posenc(x["posenc_x"], 0, 10).numpy()
        for t in (60, 16, 7):
            out[f"time_embed_{t}"] = m.interpolate_time_embed(torch.zeros(1, t, 1110), t).numpy()
        sampled(out, "fnet", m.fnet(x["enc_v"]))
        wc, wv, _, _ = m(x["fwd_video"], x["fwd_q"], iters=3)
        out["fwd_coords"], out["fwd_vis"] = wc.numpy(), wv.numpy()
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "reference_stages.npz"), **out)


def host():
    from test_evaluation import _random_problem
    from cotracker.evaluation.core.eval_utils import compute_tapvid_metrics
    from cotracker.models.core.embeddings import get_1d_sincos_pos_embed_from_grid
    from cotracker.models.core.model_utils import get_points_on_a_grid
    out = {}
    for mode in ("first", "strided"):
        for seed in range(4):
            for k, v in compute_tapvid_metrics(*_random_problem(seed), mode).items():
                out[f"tapvid_{mode}_{seed}_{k}"] = np.asarray(v)
    for i, (size, extent, centre) in enumerate(((8, (50, 50), (120.5, 77.25)), (5, (384, 512), None),
                                                (1, (384, 512), None), (30, (384, 512), None))):
        out[f"grid_{i}"] = get_points_on_a_grid(size, extent, centre).numpy()
    for L in (16, 60):
        out[f"sincos_{L}"] = get_1d_sincos_pos_embed_from_grid(1110, torch.linspace(0, L - 1, L).reshape(1, L, 1)[0]).numpy()
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "reference_host.npz"), **out)


if __name__ == "__main__":
    sys.path.insert(0, REF)
    torch.set_num_threads(max(1, min(16, len(os.sched_getaffinity(0)))))
    stages()
    host()
