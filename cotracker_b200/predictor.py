"""Public inference API -- drop-in for the reference's cotracker/predictor.py.

    CoTrackerPredictor        (reference predictor.py:14-209)
    CoTrackerOnlinePredictor  (reference predictor.py:212-309)

Same constructor arguments, call signatures, return types ((tracks[B,T,N,2] float32 in input pixels,
visibility[B,T,N] bool)), attributes (`model`, `interp_shape`, `support_grid_size`, `step`) and online state
machine.  The model behind it is `cotracker_b200.model` whose update loop runs in libct3_b200.so.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import ingest
from .build import build_cotracker


def get_points_on_a_grid(size: int, extent, device="cpu") -> torch.Tensor:
    """size x size query grid (x, y) over an (H, W) extent with a W/64 margin, row-major, shape [1, size^2, 2]
    (contract of reference model_utils.py:83-139 with the default centre)."""
    H, W = float(extent[0]), float(extent[1])
    if size == 1:
        return torch.tensor([W / 2, H / 2], device=device)[None, None]
    margin = W / 64
    ys = torch.linspace(margin, H - margin, size, device=device)
    xs = torch.linspace(margin, W - margin, size, device=device)
    gy, gx = torch.meshgrid(ys, xs, indexing="ij")
    return torch.stack([gx, gy], dim=-1).reshape(1, -1, 2)


class CoTrackerPredictor(torch.nn.Module):
    def __init__(self, checkpoint="./checkpoints/scaled_offline.pth", offline=True, v2=False, window_len=60):
        super().__init__()
        self.v2 = v2
        self.support_grid_size = 6
        model = build_cotracker(checkpoint, v2=v2, offline=offline, window_len=window_len)
        self.interp_shape = model.model_resolution
        self.model = model
        self.model.eval()

    @torch.no_grad()
    def forward(self, video, queries: torch.Tensor = None, segm_mask: torch.Tensor = None, grid_size: int = 0,
                grid_query_frame: int = 0, backward_tracking: bool = False):
        if queries is None and grid_size == 0:
            return self._compute_dense_tracks(video, grid_query_frame=grid_query_frame,
                                              backward_tracking=backward_tracking)
        return self._compute_sparse_tracks(video, queries, segm_mask, grid_size,
                                           add_support_grid=(grid_size == 0 or segm_mask is not None),
                                           grid_query_frame=grid_query_frame, backward_tracking=backward_tracking)

    def _compute_dense_tracks(self, video, grid_query_frame, grid_size=80, backward_tracking=False):
        *_, H, W = video.shape
        grid_step = W // grid_size
        gw, gh = W // grid_step, H // grid_step
        clip = _EncodedClip(self.model, video, self.interp_shape)   # one resize + encoder pass for every offset
        dev = clip.device
        tracks = visibilities = None
        pts = torch.zeros((video.shape[0], gw * gh, 3), device=dev)
        pts[:, :, 0] = grid_query_frame
        base_x = (torch.arange(gw, device=dev).repeat(gh) * grid_step).float()
        base_y = (torch.arange(gh, device=dev).repeat_interleave(gw) * grid_step).float()
        for offset in range(grid_step * grid_step):
            print(f"step {offset} / {grid_step * grid_step}")
            pts[:, :, 1] = base_x + offset % grid_step
            pts[:, :, 2] = base_y + offset // grid_step
            t_step, v_step = self._sparse_tracks(clip, video.shape, queries=pts, backward_tracking=backward_tracking)
            tracks = t_step if tracks is None else torch.cat([tracks, t_step], dim=2)
            visibilities = v_step if visibilities is None else torch.cat([visibilities, v_step], dim=2)
        return tracks, visibilities

    def _compute_sparse_tracks(self, video, queries, segm_mask=None, grid_size=0, add_support_grid=False,
                               grid_query_frame=0, backward_tracking=False):
        clip = _EncodedClip(self.model, video, self.interp_shape)
        return self._sparse_tracks(clip, video.shape, queries, segm_mask, grid_size, add_support_grid,
                                   grid_query_frame, backward_tracking)

    def _sparse_tracks(self, clip, video_shape, queries, segm_mask=None, grid_size=0, add_support_grid=False,
                       grid_query_frame=0, backward_tracking=False):
        B, T, C, H, W = video_shape
        ih, iw = self.interp_shape
        dev = clip.device
        if queries is not None:
            B, N, D = queries.shape
            assert D == 3
            queries = queries.to(dev).clone()
            queries[:, :, 1:] *= queries.new_tensor([(iw - 1) / (W - 1), (ih - 1) / (H - 1)])
        elif grid_size > 0:
            grid_pts = get_points_on_a_grid(grid_size, self.interp_shape, device=dev)
            if segm_mask is not None:
                segm_mask = F.interpolate(segm_mask.to(dev), tuple(self.interp_shape), mode="nearest")
                keep = segm_mask[0, 0][(grid_pts[0, :, 1]).round().long().cpu(),
                                       (grid_pts[0, :, 0]).round().long().cpu()].bool()
                grid_pts = grid_pts[:, keep]
            queries = torch.cat([torch.ones_like(grid_pts[:, :, :1]) * grid_query_frame, grid_pts], dim=2).repeat(B, 1, 1)
        n_support = self.support_grid_size ** 2
        if add_support_grid:
            sup = get_points_on_a_grid(self.support_grid_size, self.interp_shape, device=dev)
            sup = torch.cat([torch.zeros_like(sup[:, :, :1]), sup], dim=2).repeat(B, 1, 1)
            queries = torch.cat([queries, sup], dim=1)

        tracks, visibilities, *_ = clip.track(queries)

        if backward_tracking:
            tracks, visibilities = self._compute_backward_tracks(clip, queries, tracks, visibilities)
            if add_support_grid:
                queries[:, -n_support:, 0] = T - 1
        if add_support_grid:
            tracks = tracks[:, :, :-n_support]
            visibilities = visibilities[:, :, :-n_support]
        visibilities = visibilities > 0.9

        # query points are, by definition, where they were asked for and visible (reference :173-185)
        n = tracks.size(2)
        idx = torch.arange(n, device=tracks.device)
        for b in range(len(queries)):
            qt = queries[b, :n, 0].to(torch.int64)
            tracks[b, qt, idx] = queries[b, :n, 1:]
            visibilities[b, qt, idx] = True

        tracks *= tracks.new_tensor([(W - 1) / (iw - 1), (H - 1) / (ih - 1)])
        return tracks, visibilities

    def _compute_backward_tracks(self, clip, queries, tracks, visibilities):
        """The model on the clip played backwards (reference :187-209), on the forward pass's pyramid reversed in place."""
        T = clip.T
        inv_queries = queries.clone()
        inv_queries[:, :, 0] = T - inv_queries[:, :, 0] - 1
        inv_tracks, inv_vis, *_ = clip.track(inv_queries, reverse=True)
        inv_tracks, inv_vis = inv_tracks.flip(1), inv_vis.flip(1)
        before_query = torch.arange(T, device=queries.device)[None, :, None] < queries[:, None, :, 0]
        tracks = torch.where(before_query[..., None], inv_tracks, tracks)
        visibilities = torch.where(before_query, inv_vis, visibilities)
        return tracks, visibilities


class _EncodedClip:
    """One predictor call's clip, resized + normalised (cotracker_b200.ingest) and encoded once; every model pass of
    the call (dense offsets, backward tracking) runs on this one pyramid.  A pass on the clip played backwards reverses
    the frames of the pyramid in place (the encoder is strictly per frame, so that is the reversed clip's pyramid), and
    a later forward pass reverses them back: device memory never holds a second pyramid."""

    ITERS = 6

    def __init__(self, model, video, interp_shape):
        frames = ingest.prepare_video(video, interp_shape, ingest.model_device(model))
        self.model, self.device = model, frames.device
        self.T, _, self.H, self.W = frames.shape
        self.pyr = model._encode_clip(frames)
        self._reversed = False

    def track(self, queries, reverse=False):
        """The model's 4-tuple for queries [1,N,3] (model resolution) on the clip, or on the clip played backwards."""
        if queries.shape[0] != 1:
            raise ValueError("CoTracker3 inference requires B == 1 (the reference fails for B > 1 as well)")
        if reverse != self._reversed:
            self.model._reverse_clip_pyramid_(self.pyr, self.T, self.H, self.W)
            self._reversed = reverse
        return self.model._track_pyramid(self.pyr, self.T, self.H, self.W, queries, self.ITERS, [queries.shape[1]])


class CoTrackerOnlinePredictor(torch.nn.Module):
    def __init__(self, checkpoint="./checkpoints/scaled_online.pth", offline=False, v2=False, window_len=16):
        super().__init__()
        self.v2 = v2
        self.support_grid_size = 6
        model = build_cotracker(checkpoint, v2=v2, offline=False, window_len=window_len)
        self.interp_shape = model.model_resolution
        self.step = model.window_len // 2
        self.model = model
        self.model.eval()

    @torch.no_grad()
    def forward(self, video_chunk, is_first_step: bool = False, queries: torch.Tensor = None, grid_size: int = 5,
                grid_query_frame: int = 0, add_support_grid=False):
        B, T, C, H, W = video_chunk.shape
        ih, iw = self.interp_shape
        dev = ingest.model_device(self.model)
        if is_first_step:
            # (re)start a video: reset the model state and remember the queries (reference :242-274)
            self.model.init_video_online_processing()
            if queries is not None:
                B, N, D = queries.shape
                self.N = N
                assert D == 3
                queries = queries.to(dev).clone()
                queries[:, :, 1:] *= queries.new_tensor([(iw - 1) / (W - 1), (ih - 1) / (H - 1)])
                if add_support_grid:
                    sup = get_points_on_a_grid(self.support_grid_size, self.interp_shape, device=dev)
                    sup = torch.cat([torch.zeros_like(sup[:, :, :1]), sup], dim=2)
                    queries = torch.cat([queries, sup], dim=1)
            elif grid_size > 0:
                grid_pts = get_points_on_a_grid(grid_size, self.interp_shape, device=dev)
                self.N = grid_size ** 2
                queries = torch.cat([torch.ones_like(grid_pts[:, :, :1]) * grid_query_frame, grid_pts], dim=2)
            self.queries = queries
            return (None, None)

        frames = ingest.prepare_video(video_chunk, self.interp_shape, dev)
        tracks, visibilities, confidence, __ = self.model._track_frames(frames, self.queries, iters=6, is_online=True)
        if add_support_grid:
            tracks = tracks[:, :, :self.N]
            visibilities = visibilities[:, :, :self.N]
            confidence = confidence[:, :, :self.N]
        visibilities = visibilities * confidence
        scale = tracks.new_tensor([(W - 1) / (iw - 1), (H - 1) / (ih - 1)])
        return tracks * scale, visibilities > 0.6
