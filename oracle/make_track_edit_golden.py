"""Generate tests/golden/online_track_edits.npz: the UNMODIFIED reference online predictor (imported from
/root/reference) on seeded weights and synthetic clips, with tracks added and retired between its calls.  Run in the
build container only (the GPU box has no /root/reference):

    python oracle/make_track_edit_golden.py

An edit between two calls edits the N axis of every per-track tensor of the predictor and its model, the way
`OnlineStreams.add_tracks` / `retire_tracks` define it: `predictor.queries` and `predictor.N`,
`model.online_track_feat[l]` / `online_track_support[l]` (4 levels) and `model.online_coords_predicted` /
`online_vis_predicted` / `online_conf_predicted`.  Retiring deletes columns.  Adding inserts columns after the user
tracks and before the support grid: zero features, and at every frame so far the query point (model resolution) with
vis and conf logits 0.  The case is defined here (CASE, STREAMS, EDITS) and read by the tests; it is not one of
make_golden.CASES.  The file stores, per stream s and step k, `tracks{k}_{s}` / `visibility{k}_{s}` and the reference's
vis * conf probabilities `prob_visconf{k}_{s}` (support-grid columns still attached), for compare's threshold margin.
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

NAME = "online_track_edits"
CASE = dict(window_len=16, steps=6, iters=6, wseed=61, head_gain=5.0, vis_gain=30.0, interp_shape=(384, 512))
# name -> frame size, video seed and the open() arguments (queries: (N, query frames below T, seed) of random_queries)
STREAMS = {
    "a": dict(H=160, W=224, vseed=62, grid_size=4),
    "b": dict(H=144, W=192, vseed=63, queries=(5, 16, 64), add_support_grid=True),
}
# name -> {k: (ids to retire, queries [(t, x, y)] to add in frame pixels)}, applied before step k (stream length 8k + 8
# from k = 1 on).  a: an add before the first step; adds at length 24 whose query frames enter one window later (24,
# 30), two windows later (35) and four (50); a retire of entered tracks and of the not yet entered one (t = 50); an add
# and a retire in one gap.  b (support grid): the same around its 36 grid points.
EDITS = {
    "a": {0: ([], [(0, 30.0, 40.0), (5, 200.0, 120.0)]),
          2: ([], [(24, 50.0, 60.0), (30, 100.0, 100.0), (35, 150.0, 80.0), (50, 60.0, 130.0)]),
          4: ([1, 17, 18, 21], []),
          5: ([0, 19], [(48, 80.0, 20.0), (53, 10.0, 150.0)])},
    "b": {0: ([], [(3, 40.0, 50.0)]),
          1: ([], [(16, 90.0, 70.0), (27, 120.0, 30.0)]),
          3: ([1, 7], []),
          4: ([0], [(44, 20.0, 100.0)])},
}


def frames_needed():
    return CASE["window_len"] // 2 * (CASE["steps"] + 1)


def case_inputs():
    """-> (state dict, {stream: (video [1,T,3,H,W], open() keyword arguments)})."""
    sd = seeded_state_dict(CASE["wseed"], offline=False, window_len=CASE["window_len"], head_gain=CASE["head_gain"],
                           vis_gain=CASE["vis_gain"])
    out = {}
    for s, c in STREAMS.items():
        video = texture_video(frames_needed(), c["H"], c["W"], seed=c["vseed"])
        kw = dict(add_support_grid=c.get("add_support_grid", False))
        if "queries" in c:
            n, t, seed = c["queries"]
            kw["queries"] = random_queries(n, t, c["H"], c["W"], seed=seed)
        else:
            kw["grid_size"] = c["grid_size"]
        out[s] = (video, kw)
    return sd, out


def edit_queries(adds):
    """[(t, x, y)] -> queries [1,m,3] in frame pixels (None for no add)."""
    return torch.tensor(adds, dtype=torch.float32)[None] if adds else None


def plan_edit(ids, n, retire, m, next_id):
    """The column edit of a stream whose user tracks (ids `ids`) are its first len(ids) of n columns: -> (kept columns
    in order, the number of kept user columns the m new ones follow, the ids after the edit, the next free id)."""
    gone = {ids.index(i) for i in retire}
    keep = [c for c in range(n) if c not in gone]
    at = len(ids) - len(gone)
    return keep, at, [i for i in ids if i not in retire] + list(range(next_id, next_id + m)), next_id + m


def columns(x, dim, keep, at, new):
    """x with columns `keep` along `dim`, and `new` inserted after the first `at` of them."""
    k = x.index_select(dim, torch.tensor(keep, dtype=torch.long))
    return torch.cat([k.narrow(dim, 0, at), new.to(x.dtype), k.narrow(dim, at, len(keep) - at)], dim)


def scale_queries(q, H, W, interp_shape):
    """Frame pixels -> model resolution, as the reference predictor's first step scales its queries."""
    q = q.clone()
    q[:, :, 1:] *= q.new_tensor([(interp_shape[1] - 1) / (W - 1), (interp_shape[0] - 1) / (H - 1)])
    return q


def edit_reference(p, ids, next_id, retire, adds, H, W):
    """The edit of the reference CoTrackerOnlinePredictor `p` between two calls.  -> (ids, next_id) after it."""
    q = edit_queries(adds)
    q = torch.zeros(1, 0, 3) if q is None else scale_queries(q, H, W, p.interp_shape)
    m = q.shape[1]
    keep, at, ids, next_id = plan_edit(ids, p.queries.shape[1], retire, m, next_id)
    p.queries = columns(p.queries, 1, keep, at, q)
    p.N = at + m
    model = p.model
    if model.online_coords_predicted is not None:
        for lvl in range(len(model.online_track_feat)):
            f, s = model.online_track_feat[lvl], model.online_track_support[lvl]
            model.online_track_feat[lvl] = columns(f, 2, keep, at, f.new_zeros(1, f.shape[1], m, f.shape[3]))
            model.online_track_support[lvl] = columns(s, 2, keep, at, s.new_zeros(1, s.shape[1], m, s.shape[3]))
        T = model.online_coords_predicted.shape[1]
        point = q[:, None, :, 1:3] / model.stride * model.stride
        model.online_coords_predicted = columns(model.online_coords_predicted, 2, keep, at, point.expand(1, T, m, 2))
        model.online_vis_predicted = columns(model.online_vis_predicted, 2, keep, at, torch.zeros(1, T, m))
        model.online_conf_predicted = columns(model.online_conf_predicted, 2, keep, at, torch.zeros(1, T, m))
    return ids, next_id


def run_reference():
    sys.path.insert(0, REF)
    from cotracker.predictor import CoTrackerOnlinePredictor

    from oracle.make_golden import record_model_outputs

    sd, streams = case_inputs()
    step = CASE["window_len"] // 2
    out = {}
    with torch.no_grad():
        for s, (video, kw) in streams.items():
            p = CoTrackerOnlinePredictor(checkpoint=None, window_len=CASE["window_len"])
            p.model.load_state_dict(sd)
            probs = record_model_outputs(p.model)
            H, W = video.shape[3:]
            p(video_chunk=video[:, :1], is_first_step=True, **kw)
            ids, next_id = list(range(p.N)), p.N
            for k in range(CASE["steps"]):
                if k in EDITS[s]:
                    ids, next_id = edit_reference(p, ids, next_id, *EDITS[s][k], H, W)
                tr, vi = p(video_chunk=video[:, step * k:step * k + 2 * step], add_support_grid=kw["add_support_grid"])
                out[f"tracks{k}_{s}"], out[f"visibility{k}_{s}"] = tr.clone(), vi.clone()
                out[f"prob_visconf{k}_{s}"] = probs[k][0] * probs[k][1]
                assert tr.shape[2] == len(ids)
    return {k: v.numpy() for k, v in out.items()}


def main():
    out = run_reference()
    path = os.path.join(ROOT, "tests", "golden", NAME + ".npz")
    np.savez_compressed(path, **out)
    print(NAME, {k: v.shape for k, v in out.items() if k.endswith("_a") or k.endswith("_b")}, os.path.getsize(path),
          "bytes")


if __name__ == "__main__":
    main()
