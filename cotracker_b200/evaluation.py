"""Evaluation harness -- SURVEY.md 8(f) rank 4.

    tapvid_metrics        -- reference cotracker/evaluation/core/eval_utils.py:12-138 (compute_tapvid_metrics)
    EvaluationPredictor   -- reference cotracker/models/evaluation_predictor.py:25-199

`tapvid_metrics` is plain numpy (no GPU): TAP-Vid occlusion accuracy, points-within-threshold (delta_avg) and
Jaccard (AJ) at 1/2/4/8/16 px.  `EvaluationPredictor` wraps a cotracker_b200 offline model the way the
reference's benchmark code drives it: one query point at a time with an 8x8 local grid and a 5x5 global grid as
helper tracks (single_point=True, the TAP-Vid protocol), or all queries jointly.  The model behind it is the same
CUDA path as everywhere else (libct3_b200.so); SIFT helper points (sift_size > 0) are not provided.
In single-point mode every query's 90-track set is one group of a grouped update loop (as `forward_groups`): the clip
is resized (cotracker_b200.ingest) and encoded once, and all groups share one update loop, in as few passes as fit in
device memory (`plan_passes`).  Each group's result
is bit-identical to a model call on that group alone, so the split into passes does not change the output.
With no datasets or checkpoints in this environment the harness is exercised by scoring the CUDA tracks against
the reference's tracks on synthetic clips (tests/test_evaluation.py): identical outputs score 1.0 everywhere.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

THRESHOLDS = (1, 2, 4, 8, 16)


def tapvid_metrics(query_points: np.ndarray, gt_occluded: np.ndarray, gt_tracks: np.ndarray,
                   pred_occluded: np.ndarray, pred_tracks: np.ndarray, query_mode: str) -> Dict[str, np.ndarray]:
    """TAP-Vid metrics per video.  Shapes: query_points [b,n,3] as (t, y, x); *_occluded [b,n,t] bool;
    *_tracks [b,n,t,2] as (x, y) in raster coordinates (the paper's numbers assume 256x256).
    query_mode "first": only frames strictly after the query frame are scored; "strided": every other frame."""
    b, n, t = gt_occluded.shape
    frames = np.arange(t)
    qf = np.round(query_points[..., 0]).astype(np.int32)                       # [b,n]
    if query_mode == "first":
        scored = frames[None, None, :] > qf[..., None]
    elif query_mode == "strided":
        scored = frames[None, None, :] != qf[..., None]
    else:
        raise ValueError("Unknown query mode " + query_mode)

    def per_video(mask):
        return np.sum(mask & scored, axis=(1, 2))

    out: Dict[str, np.ndarray] = {}
    # NB: the denominator is the number of scored points of the WHOLE batch (reference eval_utils.py:75-78)
    out["occlusion_accuracy"] = per_video(pred_occluded == gt_occluded) / np.sum(scored)
    gt_vis, pred_vis = ~gt_occluded.astype(bool), ~pred_occluded.astype(bool)
    d2 = np.sum(np.square(pred_tracks - gt_tracks), axis=-1)
    n_gt_vis = per_video(gt_vis)
    within_all, jac_all = [], []
    for thr in THRESHOLDS:
        close = d2 < thr * thr
        hit = close & gt_vis
        out[f"pts_within_{thr}"] = per_video(hit) / n_gt_vis
        # false positive: predicted visible where the ground truth is occluded or further than the threshold
        false_pos = per_video(pred_vis & (~gt_vis | ~close))
        out[f"jaccard_{thr}"] = per_video(hit & pred_vis) / (n_gt_vis + false_pos)
        within_all.append(out[f"pts_within_{thr}"])
        jac_all.append(out[f"jaccard_{thr}"])
    out["average_jaccard"] = np.mean(np.stack(jac_all, axis=1), axis=1)
    out["average_pts_within_thresh"] = np.mean(np.stack(within_all, axis=1), axis=1)
    return out


def points_on_a_grid(size: int, extent, center=None, device="cpu") -> torch.Tensor:
    """size x size grid of (x, y) points over an (H, W) extent around `center` (cy, cx), margin W/64, row-major
    (contract of reference model_utils.py:83-139)."""
    H, W = float(extent[0]), float(extent[1])
    if size == 1:
        return torch.tensor([W / 2, H / 2], device=device)[None, None]
    cy, cx = (H / 2, W / 2) if center is None else (float(center[0]), float(center[1]))
    m = W / 64
    ys = torch.linspace(m - H / 2 + cy, H / 2 + cy - m, size, device=device)
    xs = torch.linspace(m - W / 2 + cx, W / 2 + cx - m, size, device=device)
    gy, gx = torch.meshgrid(ys, xs, indexing="ij")
    return torch.stack([gx, gy], dim=-1).reshape(1, -1, 2)


def pass_bytes(T: int, N: int, G: int, H4: int, W4: int, frames: Optional[int] = None, ragged: bool = False) -> int:
    """Device memory of one grouped update-loop pass over N tracks in G groups and T frames: the library workspace
    plus the per-track support features [4,49,N,128] and the per-frame state and outputs (about 16 floats).
    frames: the pyramid frames of a pass with a frame map (engine.workspace_bytes).  ragged: the groups have lengths of
    their own (ct3_loop_shape.group_T), which adds a time embedding per group."""
    from . import engine
    ws = engine.workspace_bytes(T, N, H4, W4, groups=G, frames=frames, group_T=[T] * G if ragged else None)
    return ws + N * (4 * 49 * 128 * 4 + T * 16 * 4) + (G * T * 1110 * 4 if ragged else 0)


def pass_budget_bytes(model, device, T: int, ih: int, iw: int) -> int:
    """Device memory one grouped pass of `model` on a T-frame clip at ih x iw may use: what is free plus the model's
    cached update-loop workspace (it is regrown per pass), less the encoder's workspace and two copies of the pyramid."""
    from . import engine
    free, _ = torch.cuda.mem_get_info(device)
    free += torch.cuda.memory_reserved(device) - torch.cuda.memory_allocated(device)
    ws = model._ws.buf
    if ws is not None and ws.device == torch.device(device):
        free += ws.numel()
    s = model.stride
    pyr = engine.pyramid_layout(T, ih // s, iw // s)[3] * 4
    reserve = engine.encoder_workspace_bytes(T, ih, iw) + 2 * pyr + (1 << 30)
    return int(0.9 * max(0, free - reserve))


def slab_tracks_for(T: int, N: int, G: int, H4: int, W4: int, frames: Optional[int], budget_bytes: int,
                    group_T: Optional[Sequence[int]] = None) -> Optional[int]:
    """Track slabs of one update-loop pass (ct3_loop_shape.slab_tracks, DESIGN.md §4.4.5): None when the full workspace
    fits `budget_bytes`, so every pass that fits runs exactly as without slabs; else the largest slab_tracks whose
    workspace fits (the workspace never shrinks as slab_tracks grows), or 1 when none does.
    frames: the pyramid frames of a pass with a frame map; group_T: its group lengths (engine.workspace_bytes)."""
    from . import engine
    if engine.workspace_bytes(T, N, H4, W4, groups=G, frames=frames, group_T=group_T) <= budget_bytes:
        return None
    lo, hi = 1, max(1, N - 1)
    while lo < hi:
        mid = (lo + hi + 1) // 2
        if engine.workspace_bytes(T, N, H4, W4, groups=G, frames=frames, slab_tracks=mid,
                                  group_T=group_T) <= budget_bytes:
            lo = mid
        else:
            hi = mid - 1
    return lo


def plan_dense_passes(n_offsets: int, n_tracks: int, backward: bool, T: int, H4: int, W4: int, budget_bytes: int,
                      frames: Optional[int] = None) -> Tuple[List[int], List[Tuple[int, int]]]:
    """Groups and passes of the predictor's dense mode: one group of n_tracks per grid offset, followed by that
    offset's reversed group with backward tracking, split by `plan_passes` (T: frames of one update loop; frames: the
    pyramid frames a pass with reversed groups reads, None when it has none).  -> (group sizes, passes)."""
    sizes = [n_tracks] * (n_offsets * (2 if backward else 1))
    return sizes, plan_passes(sizes, T, H4, W4, budget_bytes,
                              lambda T_, N, G, H4_, W4_: pass_bytes(T_, N, G, H4_, W4_, frames))


def plan_passes(group_sizes: Sequence[int], T: int, H4: int, W4: int, budget_bytes: int,
                bytes_fn: Optional[Callable[[int, int, int, int, int], int]] = None) -> List[Tuple[int, int]]:
    """Split the groups, in order, into as few passes [g0, g1) as keep bytes_fn(T, N, G, H4, W4) (default
    `pass_bytes`) within `budget_bytes`.  A pure host function; a group that alone exceeds the budget gets a pass of
    its own."""
    fn = bytes_fn or pass_bytes
    passes, g0, n = [], 0, 0
    for g, size in enumerate(group_sizes):
        if g > g0 and fn(T, n + size, g + 1 - g0, H4, W4) > budget_bytes:
            passes.append((g0, g))
            g0, n = g, 0
        n += size
    if len(group_sizes) > 0:
        passes.append((g0, len(group_sizes)))
    return passes


def plan_clip_passes(n_clips: int, group_sizes: Sequence[int], T: int, H4: int, W4: int, budget_bytes: int,
                     frames_fn: Optional[Callable[[int], Optional[int]]] = None) -> List[Tuple[int, int]]:
    """Split the clips of a batch, in order, into passes [b0, b1): as few as keep a pass within `budget_bytes`.
    group_sizes: the groups every clip brings, or a list of n_clips such lists when the clips (streams) differ.  A pass
    over clips [b0, b1) costs pass_bytes(T, their tracks, their groups, H4, W4, frames_fn(b1 - b0)) at T frames per
    update loop; frames_fn(n): the pyramid frames such a pass reads through its frame map (None: it has none).  When
    every clip brings the same groups the passes are of even size.  A pure host function; a clip that alone exceeds the
    budget gets a pass of its own.  The library takes any number of groups up to the number of tracks, which a batch
    of clips with at least one track per group cannot exceed."""
    ragged = len(group_sizes) > 0 and isinstance(group_sizes[0], (list, tuple))
    per_clip = [list(g) for g in group_sizes] if ragged else [list(group_sizes)] * n_clips
    if len(per_clip) != n_clips:
        raise ValueError(f"{len(per_clip)} group lists for {n_clips} clips")
    passes, b0, N, G = [], 0, 0, 0
    for b, sizes in enumerate(per_clip):
        if b > b0 and pass_bytes(T, N + sum(sizes), G + len(sizes), H4, W4,
                                 frames_fn(b + 1 - b0) if frames_fn else None) > budget_bytes:
            passes.append((b0, b))
            b0, N, G = b, 0, 0
        N, G = N + sum(sizes), G + len(sizes)
    if n_clips > 0:
        passes.append((b0, n_clips))
    if not ragged and passes:   # same cost per clip: spread the clips evenly over as many passes
        per = -(-n_clips // len(passes))
        passes = [(b0, min(n_clips, b0 + per)) for b0 in range(0, n_clips, per)]
    return passes


def plan_ragged_passes(lengths: Sequence[int], tracks: Sequence[int], groups: Sequence[int], H4: int, W4: int,
                       budget_bytes: int, pad_fraction: float, frames: int, pad_rows: int = 0) -> List[List[int]]:
    """Passes of clips of different lengths (`CoTrackerPredictor` on a list): clip b has lengths[b] frames, tracks[b]
    tracks in all and groups[b] query groups.  The clips are taken shortest first; a pass pads every clip to its
    longest one.  Padding is counted in token rows: each clip's point tracks and the 64 virtual tracks of each of its
    groups, times the frames it is padded by.  A new pass starts when the next clip would take the pass past
    `budget_bytes` (`pass_bytes` with group lengths, `frames` pyramid frames), or its padded token rows past
    pad_fraction times its real ones plus pad_rows.  A pure host function: -> the clips of each pass (indices into
    `lengths`), shortest first; a clip that alone exceeds the budget gets a pass of its own.  Groups are independent,
    so the split changes no result."""
    if not (len(lengths) == len(tracks) == len(groups)):
        raise ValueError(f"{len(lengths)} lengths, {len(tracks)} track counts and {len(groups)} group counts")
    rows = [tracks[b] + 64 * groups[b] for b in range(len(lengths))]   # token rows per frame
    order = sorted(range(len(lengths)), key=lambda b: (lengths[b], b))
    passes: List[List[int]] = []
    cur: List[int] = []
    for b in order:
        if cur:
            T, N, G = lengths[b], sum(tracks[c] for c in cur) + tracks[b], sum(groups[c] for c in cur) + groups[b]
            real = sum(rows[c] * lengths[c] for c in cur + [b])
            padded = sum(rows[c] for c in cur + [b]) * T - real
            if pass_bytes(T, N, G, H4, W4, frames, ragged=True) > budget_bytes or padded > pad_fraction * real + pad_rows:
                passes.append(cur)
                cur = []
        cur.append(b)
    if cur:
        passes.append(cur)
    return passes


class EvaluationPredictor(torch.nn.Module):
    """Benchmark-protocol wrapper around an offline CoTracker3 model (B = 1).

    forward(video [1,T,3,H,W] in 0..255, queries [1,N,3] = (t, x, y) in input pixels)
        -> (tracks [1,T,N,2] in input pixels, visibility*confidence [1,T,N] probabilities)
    """

    def __init__(self, cotracker_model, interp_shape: Tuple[int, int] = (384, 512), grid_size: int = 5,
                 local_grid_size: int = 8, single_point: bool = True, sift_size: int = 0,
                 num_uniformly_sampled_pts: int = 0, n_iters: int = 6, local_extent: int = 50,
                 pass_budget_bytes: Optional[int] = None) -> None:
        """pass_budget_bytes: device memory one single-point pass may use (None: derived from free device memory)."""
        super().__init__()
        if sift_size > 0:
            raise NotImplementedError("SIFT helper points are not provided by this build")
        self.grid_size = grid_size
        self.local_grid_size = local_grid_size
        self.single_point = single_point
        self.sift_size = 0
        self.interp_shape = interp_shape
        self.n_iters = n_iters
        self.num_uniformly_sampled_pts = num_uniformly_sampled_pts
        self.local_extent = local_extent
        self.pass_budget_bytes = pass_budget_bytes
        self.model = cotracker_model
        self.model.eval()

    def _helpers(self, video, query: Optional[torch.Tensor]) -> torch.Tensor:
        """Helper tracks appended after the evaluated ones: [local grid around the query], global grid, random."""
        dev, extra = video.device, []
        if query is not None and self.local_grid_size > 0:
            loc = points_on_a_grid(self.local_grid_size, (self.local_extent, self.local_extent),
                                   (query[0, 0, 2].item(), query[0, 0, 1].item()), device=dev)
            extra.append(torch.cat([torch.zeros_like(loc[:, :, :1]), loc], dim=2))
        if self.grid_size > 0:
            g = points_on_a_grid(self.grid_size, video.shape[3:], device=dev)
            extra.append(torch.cat([torch.zeros_like(g[:, :, :1]), g], dim=2))
        if self.num_uniformly_sampled_pts > 0:
            k, T, (H, W) = self.num_uniformly_sampled_pts, video.shape[1], video.shape[3:]
            tt = torch.randint(0, T, (k, 1), device=dev).float()
            xy = torch.rand(k, 2, device=dev) * torch.tensor([W, H], device=dev, dtype=torch.float32)
            extra.append(torch.cat([tt, xy], dim=1)[None])
        return torch.cat(extra, dim=1) if extra else video.new_zeros(1, 0, 3)

    @torch.no_grad()
    def forward(self, video, queries):
        from . import ingest
        ingest.reject_encoded_clip(video, "EvaluationPredictor")
        B, T, C, H, W = video.shape
        assert queries.shape[0] == 1 and queries.shape[2] == 3 and B == 1
        N = queries.shape[1]
        ih, iw = self.interp_shape
        dev = ingest.model_device(self.model)
        frames = ingest.prepare_video(video, (ih, iw), dev)
        video = frames[None]                               # [1,T,3,ih,iw]: the shape and device the helpers use
        queries = queries.to(dev).clone()
        queries[:, :, 1] *= (iw - 1) / (W - 1)
        queries[:, :, 2] *= (ih - 1) / (H - 1)
        if self.single_point:
            tracks = video.new_zeros(B, T, N, 2)
            vis = video.new_zeros(B, T, N)
            conf = video.new_zeros(B, T, N)
            # one group per query: the query followed by its helpers (random draws in the reference's per-query order)
            groups = [torch.cat([queries[:, i:i + 1], self._helpers(video, queries[:, i:i + 1])], dim=1)
                      for i in range(N)]
            sizes = [g.shape[1] for g in groups]
            first = np.concatenate([[0], np.cumsum(sizes)]).tolist()
            q_all = torch.cat(groups, dim=1)
            stride = self.model.stride
            T_loop = T if not hasattr(self.model, "init_video_online_processing") else self.model.window_len
            budget = self.pass_budget_bytes
            if budget is None:
                budget = pass_budget_bytes(self.model, video.device, T, ih, iw)
            pyr = self.model._encode_clip(frames)          # every pass runs on the same pyramid
            del frames, video
            for g0, g1 in plan_passes(sizes, T_loop, ih // stride, iw // stride, budget):
                a, b = first[g0], first[g1]
                tr, vi, cf, _ = self.model._track_pyramid(pyr, T, ih, iw, q_all[:, a:b], self.n_iters, sizes[g0:g1])
                cols = [first[g] - a for g in range(g0, g1)]
                tracks[:, :, g0:g1] = tr[:, :, cols, :2]
                vis[:, :, g0:g1] = vi[:, :, cols]
                conf[:, :, g0:g1] = cf[:, :, cols]
        else:
            q_all = torch.cat([queries, self._helpers(video, None)], dim=1)
            tr, vi, cf, _ = self.model._track_frames(frames, q_all, iters=self.n_iters)
            tracks, vis, conf = tr[:, :, :N].clone(), vi[:, :, :N], cf[:, :, :N]
        tracks[..., 0] *= (W - 1) / float(iw - 1)
        tracks[..., 1] *= (H - 1) / float(ih - 1)
        return tracks, vis * conf
