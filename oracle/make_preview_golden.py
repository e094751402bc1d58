"""Generate tests/golden/online_preview.npz: the UNMODIFIED reference online predictor (imported from /root/reference)
on seeded weights and a synthetic clip, with previews between its window steps.  Run in the build container only (the
GPU box has no /root/reference):

    python oracle/make_preview_golden.py

A preview of frame f is the reference's own answer for a video that ends at f: a `copy.deepcopy` of the predictor,
called on the chunk from the current window start w = max(0, length - (window_len - step)) to frame f, as
online_demo.py calls it on its last chunk.  The copy is dropped afterwards, so the original runs on as if the preview
had never been made.  The case is defined here (CASE, PLAN) and read by the tests.  The file stores, per entry of
PLAN, `tracks_<name>` / `visibility_<name>` and the reference's probabilities `prob_vis_<name>`,
`prob_conf_<name>` and their product `prob_visconf_<name>` (every column), for compare's threshold margin.
"""
from __future__ import annotations

import copy
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF = os.environ.get("COTRACKER_REFERENCE", "/root/reference")

from cotracker_b200.synthetic import seeded_state_dict, texture_video  # noqa: E402

NAME = "online_preview"
CASE = dict(window_len=16, T=40, H=160, W=224, wseed=71, vseed=72, qseed=73, head_gain=5.0, vis_gain=30.0, grid=4,
            late=8)
# in order: ("c", k) commits window k (the chunk of frames [8k, 8k + 16): the stream then holds 16, 24, 32 frames);
# ("p", f) previews frame f.  Before the first step (T = 1 and T = 10), the first new frame after a commit (f = 16,
# T = 9), a middle frame (T = 12), the last frame before a commit (T = 15), one in each later window, and a full-window
# preview (f = 39, T = 16).
PLAN = [("p", 0), ("p", 9), ("c", 0), ("p", 16), ("p", 19), ("p", 22), ("c", 1), ("p", 28), ("c", 2), ("p", 33),
        ("p", 39)]


def entry_name(kind: str, x: int) -> str:
    return f"commit{x}" if kind == "c" else f"preview{x}"


def window_start(length: int) -> int:
    step = CASE["window_len"] // 2
    return max(0, length - (CASE["window_len"] - step))


def case_inputs():
    """-> (state dict, video [1,T,3,H,W], queries [1,N,3] in frame pixels): a grid x grid lattice at frame 0 and
    `late` queries whose frames fall in later windows (8..35), so tracks enter the window in every step."""
    sd = seeded_state_dict(CASE["wseed"], offline=False, window_len=CASE["window_len"], head_gain=CASE["head_gain"],
                           vis_gain=CASE["vis_gain"])
    H, W, g = CASE["H"], CASE["W"], CASE["grid"]
    video = texture_video(CASE["T"], H, W, seed=CASE["vseed"])
    ys, xs = torch.meshgrid(torch.linspace(8, H - 9, g), torch.linspace(8, W - 9, g), indexing="ij")
    grid = torch.stack([torch.zeros(g * g), xs.flatten(), ys.flatten()], 1)
    gen = torch.Generator().manual_seed(CASE["qseed"])
    n = CASE["late"]
    late = torch.stack([torch.randint(8, 36, (n,), generator=gen).float(), torch.rand(n, generator=gen) * (W - 1),
                        torch.rand(n, generator=gen) * (H - 1)], 1)
    return sd, video, torch.cat([grid, late])[None]


def _call(pred, chunk):
    """pred(chunk) with the reference model's (vis, conf) probabilities of the call -> (tracks, visibility, vis, conf).
    The wrapper is an instance attribute, removed again so that `copy.deepcopy(pred)` copies a plain model."""
    from oracle.make_golden import record_model_outputs

    rec = record_model_outputs(pred.model)
    try:
        tr, vi = pred(video_chunk=chunk)
    finally:
        del pred.model.forward
    return tr, vi, rec[0][0], rec[0][1]


def run_reference():
    sys.path.insert(0, REF)
    from cotracker.predictor import CoTrackerOnlinePredictor

    sd, video, queries = case_inputs()
    step = CASE["window_len"] // 2
    out = {}
    with torch.no_grad():
        p = CoTrackerOnlinePredictor(checkpoint=None, window_len=CASE["window_len"])
        p.model.load_state_dict(sd)
        p(video_chunk=video[:, :1], is_first_step=True, queries=queries)
        length = 0
        for kind, x in PLAN:
            if kind == "c":
                assert length == (0 if x == 0 else step * x + step)
                res = _call(p, video[:, step * x:step * x + 2 * step])
                length = step * x + 2 * step
            else:
                assert x >= length
                res = _call(copy.deepcopy(p), video[:, window_start(length):x + 1])
                assert res[0].shape[1] == x + 1
            name = entry_name(kind, x)
            tr, vi, pv, pc = res
            out[f"tracks_{name}"], out[f"visibility_{name}"] = tr.clone(), vi.clone()
            out[f"prob_vis_{name}"], out[f"prob_conf_{name}"] = pv, pc
            out[f"prob_visconf_{name}"] = pv * pc
    return {k: v.numpy() for k, v in out.items()}


def main():
    out = run_reference()
    path = os.path.join(ROOT, "tests", "golden", NAME + ".npz")
    np.savez_compressed(path, **out)
    print(NAME, {k: v.shape for k, v in out.items() if k.startswith("tracks")}, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
