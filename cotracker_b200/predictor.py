"""Public inference API -- drop-in for the reference's cotracker/predictor.py.

    CoTrackerPredictor        (reference predictor.py:14-209)
    CoTrackerOnlinePredictor  (reference predictor.py:212-309)

Same constructor arguments, call signatures, return types ((tracks[B,T,N,2] float32 in input pixels,
visibility[B,T,N] bool)), attributes (`model`, `interp_shape`, `support_grid_size`, `step`) and online state
machine.  The model behind it is `cotracker_b200.model` whose update loop runs in libct3_b200.so.

B clips of one length and size are tracked together (the reference fails for B > 1): one resize, one encoder pass and,
memory permitting, one update-loop pass for the whole batch; slot b of the result is bit-identical to the call on
`video[b:b+1]` (and `queries[b:b+1]`).  `segm_mask` keeps a different number of points per clip and is for B = 1 only.
A list of [1,T_b,3,H_b,W_b] clips of any lengths and sizes (offline model, sparse queries) is tracked the same way, with
per-clip `queries` / `segm_mask` lists; it returns lists, and entry b is bit-identical to the call on clip b alone.
A clip, or an entry of such a list, may be a `YUVClip` (NV12, I420 or YUYV frames): results are `torch.equal` to the
call on its RGB conversion by cv2.cvtColor.  It may also be a `Crop`, a window of each frame of a clip or a YUVClip:
results are `torch.equal` to the call on the materialised window, in window pixels.

`return_scores=True` (both predictors) adds a third output, `TrackScores(visibility, confidence)`: the model's
probabilities sigmoid(vis) and sigmoid(conf), fp32 on the device, of the visibility output's shape (a list of them for a
list call).  They pass the same backward merge, support-grid drop and frame selection as the visibility.  The offline
predictor's visibility is `scores.visibility > 0.9` except at the query points, which it pins to True while the scores
keep the model's values there; the online predictor's is `scores.visibility * scores.confidence > 0.6`, bit for bit.
Tracks and visibility are the same with and without the flag.

`CoTrackerPredictor.encode(video)` resizes and encodes a clip once and returns an `EncodedClip`, which the offline
predictor takes wherever it takes a video, in every mode and any number of times: `predictor(predictor.encode(video),
**kw)` is `torch.equal` to `predictor(video, **kw)`, because a direct call is that same encode followed by the same
tracking path.  `clip.to("cpu")` parks an idle clip in pinned host memory and `clip.to(device)` brings it back
bit-identical.
"""
from __future__ import annotations

import copy
from typing import NamedTuple, Optional

import torch
import torch.nn.functional as F

from . import corners, engine, ingest
from .build import build_cotracker
from .evaluation import pass_budget_bytes, plan_clip_passes, plan_dense_passes, plan_ragged_passes

# Backward tracking runs the forward and the reversed queries as two groups of one update-loop pass while one direction
# has at most this many tracks x loop frames, and as two passes above it.  Measured on an H100 (DESIGN.md 4.4.2): one
# pass is faster at 136 x 50 (-10 %) and 6436 x 16 (-2 %); at 6436 x 50 the loop is throughput-bound, one pass is not
# faster (+0.3 %) and needs twice the update-loop workspace (45.8 instead of 24.6 GiB).
BACKWARD_GROUP_TRACK_FRAMES = 1 << 17

# A list call pads the clips of one update-loop pass to its longest clip, and starts a new pass before its padded token
# rows (points and virtual tracks) exceed RAGGED_PAD_FRACTION times the real ones plus RAGGED_PAD_ROWS
# (`plan_ragged_passes`).  Set by a sweep on an H100 (DESIGN.md 5.1, scripts/ragged_bench.py), 512x512 clips of 16-64
# frames, clips/s against one call per clip:
#   fraction       0      0.1    0.25   0.5    1     | rows 2^14  2^16
#   8 clips, grid 10   -2 %   +4 %   +7 %   +7 %   -2 %  |   +6 %    -2 %
#   32 clips, grid 10  -4 %   +8 %   +8 %   +7 %   -1 %  |   +8 %    +4 %
#   8 clips, grid 30   -1 %   -1 %   -5 %   -9 %  -26 %  |   -4 %    -9 %
# Padding pays where the loop is launch-bound (grid 10) and costs where it is throughput-bound (grid 30); 0.1 keeps
# most of the gain at grid 10 for the smallest loss at grid 30.  A fixed row allowance (which favours small passes)
# did no better than a fraction, so it is 0.
RAGGED_PAD_FRACTION = 0.1
RAGGED_PAD_ROWS = 0


class TrackScores(NamedTuple):
    """Per-track, per-frame probabilities of the model, fp32 [B,T,N] on the device: `visibility` = sigmoid(vis),
    `confidence` = sigmoid(conf) (reference cotracker3_offline.py:215-216, cotracker3_online.py:524-525)."""
    visibility: torch.Tensor
    confidence: torch.Tensor


def _check_return_scores(return_scores):
    if not isinstance(return_scores, bool):
        raise ValueError(f"return_scores must be True or False, got {type(return_scores).__name__}")


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
        self._list_budget_bytes = None   # device memory of one pass of a list call (None: from free device memory)

    @torch.no_grad()
    def forward(self, video, queries: torch.Tensor = None, segm_mask: torch.Tensor = None, grid_size: int = 0,
                grid_query_frame: int = 0, backward_tracking: bool = False, return_scores: bool = False):
        """-> (tracks, visibility), or with return_scores=True (tracks, visibility, TrackScores) (module docstring).
        video may be an `EncodedClip` of `encode`; the call then neither uploads nor encodes, and leaves the clip as it
        was."""
        _check_return_scores(return_scores)
        if isinstance(video, (list, tuple)):
            return self._track_list(list(video), queries, segm_mask, grid_size, grid_query_frame, backward_tracking,
                                    return_scores)
        encoded = isinstance(video, EncodedClip)
        if encoded:
            video = self._check_clip(video)
        if segm_mask is not None and (video.B if encoded else video.shape[0]) != 1:
            raise ValueError("segm_mask keeps a different number of grid points per clip: it needs B == 1")
        # a direct call is `encode` without the weights' fingerprint, which only a clip that outlives the call needs
        clip = video if encoded else EncodedClip(self.model, video, self.interp_shape)
        if queries is None and grid_size == 0:
            return self._compute_dense_tracks(clip, grid_query_frame=grid_query_frame,
                                              backward_tracking=backward_tracking, return_scores=return_scores)
        return self._compute_sparse_tracks(clip, queries, segm_mask, grid_size,
                                           add_support_grid=(grid_size == 0 or segm_mask is not None),
                                           grid_query_frame=grid_query_frame, backward_tracking=backward_tracking,
                                           return_scores=return_scores)

    @torch.no_grad()
    def encode(self, video) -> "EncodedClip":
        """video ([B,T,3,H,W] uint8 or float, host or device, any strides, a `YUVClip` or a `Crop`: anything one call
        takes)
        -> its `EncodedClip`: resized, normalised and encoded once, on the model's device, for any number of calls."""
        if isinstance(video, (list, tuple, EncodedClip)):
            raise TypeError(f"encode takes one clip [B,T,3,H,W] or a YUVClip, got {type(video).__name__} (list calls "
                            "take pixels; an EncodedClip is encoded already)")
        return EncodedClip(self.model, video, self.interp_shape, weights=self.model.weights_fingerprint())

    def _check_clip(self, clip: "EncodedClip") -> "EncodedClip":
        """The ValueErrors of an EncodedClip this predictor cannot track, raised before any work.  -> the clip, bound
        to this predictor's model (a shallow copy sharing the pyramid when another predictor's model encoded it)."""
        if clip.parked:
            raise ValueError("the EncodedClip is parked on the host: bring it back with clip.to(device) first")
        if tuple(clip.interp_shape) != tuple(self.interp_shape):
            raise ValueError(f"the EncodedClip was encoded at interp_shape {tuple(clip.interp_shape)}, this predictor "
                             f"tracks at {tuple(self.interp_shape)}")
        if clip.stride != self.model.stride:
            raise ValueError(f"the EncodedClip was encoded at stride {clip.stride}, this predictor's model has stride "
                             f"{self.model.stride}")
        if clip.loop != _loop(self.model):
            raise ValueError(f"the EncodedClip was encoded for the {clip.loop} model, this predictor runs the "
                             f"{_loop(self.model)} model")
        dev = ingest.model_device(self.model)
        if clip.device != dev:
            raise ValueError(f"the EncodedClip is on {clip.device}, the predictor's model on {dev}: move one of them")
        if clip.weights != self.model.weights_fingerprint():
            raise ValueError("the EncodedClip was encoded with other weights than the predictor's model has now "
                             "(weights_fingerprint differs): encode the video again")
        if clip.model is not self.model:
            clip = copy.copy(clip)
            clip.model = self.model
        return clip

    def _track_list(self, clips, queries, segm_mask, grid_size, grid_query_frame, backward_tracking,
                    return_scores=False):
        """Clips [1,T_b,3,H_b,W_b] of any lengths and sizes: one resize per clip into one frame buffer, one encoder
        pass, and as few update-loop passes as the memory budget and RAGGED_PAD_FRACTION allow, each clip's groups
        padded to the longest clip of their pass (ct3_loop_shape.group_T).  -> (tracks, visibility), lists in input
        order, entry b bit-identical to the call on clip b with its own queries / segm_mask; return_scores=True adds
        a list of TrackScores."""
        B = len(clips)
        _check_list_call(self.model, clips, queries, segm_mask, grid_size, grid_query_frame)
        qs = [None] * B if queries is None else list(queries)
        masks = [None] * B if segm_mask is None else list(segm_mask)
        lengths = [int(c.shape[1]) for c in clips]
        ih, iw = self.interp_shape
        dev = ingest.model_device(self.model)
        first = [sum(lengths[:b]) for b in range(B)]
        frames = torch.empty(sum(lengths), 3, ih, iw, device=dev)
        for b, clip in enumerate(clips):
            ingest.prepare_video(clip, (ih, iw), dev, out=frames[first[b]:first[b] + lengths[b]])
        pyr = self.model._encode_clip(frames)
        del frames
        at = _Device(dev)
        add = [grid_size == 0 or m is not None for m in masks]
        mq = [self._model_queries(at, c.shape, q, m, grid_size, a, grid_query_frame)
              for c, q, m, a in zip(clips, qs, masks, add)]
        groups = [[(q, first[b], lengths[b], False)] + ([(_reversed_queries(q, lengths[b]), first[b], lengths[b], True)]
                                                         if backward_tracking else [])
                  for b, q in enumerate(mq)]
        s = self.model.stride
        budget = self._list_budget_bytes
        if budget is None:
            budget = pass_budget_bytes(self.model, dev, sum(lengths), ih, iw)
        passes = plan_ragged_passes(lengths, [sum(g[0].shape[1] for g in gs) for gs in groups],
                                    [len(gs) for gs in groups], ih // s, iw // s, budget, RAGGED_PAD_FRACTION,
                                    sum(lengths), RAGGED_PAD_ROWS)
        outs = [None] * B
        for p in passes:
            res = self.model._track_ragged(pyr, ih, iw, [g for b in p for g in groups[b]], EncodedClip.ITERS,
                                           scores=return_scores)
            for b in p:
                outs[b], res = res[:len(groups[b])], res[len(groups[b]):]
        res = [self._finish(mq[b], outs[b][0], outs[b][1] if backward_tracking else None, clips[b].shape, add[b],
                            return_scores) for b in range(B)]
        return tuple(list(r) for r in zip(*res))

    def _compute_dense_tracks(self, clip, grid_query_frame, grid_size=80, backward_tracking=False,
                              return_scores=False):
        """grid_step^2 shifted grids, one query group per offset (and one reversed group per offset with backward
        tracking), tracked in as few grouped passes over the one EncodedClip as fit in device memory."""
        H, W = clip.input_hw
        grid_step = W // grid_size
        gw, gh = W // grid_step, H // grid_step
        dev = clip.device
        n_off = grid_step * grid_step
        base_x = (torch.arange(gw, device=dev).repeat(gh) * grid_step).float()
        base_y = (torch.arange(gh, device=dev).repeat_interleave(gw) * grid_step).float()
        queries = []
        for offset in range(n_off):
            pts = torch.zeros((clip.B, gw * gh, 3), device=dev)
            pts[:, :, 0] = grid_query_frame
            pts[:, :, 1] = base_x + offset % grid_step
            pts[:, :, 2] = base_y + offset // grid_step
            queries.append(self._model_queries(clip, clip.video_shape, pts))
        per = 2 if backward_tracking else 1
        groups = [g for q in queries for g in ([q, _reversed_queries(q, clip.T)] if backward_tracking else [q])]
        _, passes = plan_dense_passes(n_off, gw * gh, backward_tracking, *clip.pass_shape(backward_tracking))
        outs = []
        for g0, g1 in passes:
            for g in range(g0, g1):
                if g % per == 0:
                    print(f"step {g // per} / {n_off}")
            outs += clip.track_groups(groups[g0:g1], [g % per == 1 for g in range(g0, g1)], return_scores)
        tracks = visibilities = probs = None
        for i in range(n_off):
            step = self._finish(queries[i], outs[per * i], outs[per * i + 1] if backward_tracking else None,
                                clip.video_shape, scores=return_scores)
            t_step, v_step = step[:2]
            tracks = t_step if tracks is None else torch.cat([tracks, t_step], dim=2)
            visibilities = v_step if visibilities is None else torch.cat([visibilities, v_step], dim=2)
            if return_scores:
                probs = step[2] if probs is None else TrackScores(*(torch.cat([a, b], dim=2)
                                                                    for a, b in zip(probs, step[2])))
        return (tracks, visibilities, probs) if return_scores else (tracks, visibilities)

    def _compute_sparse_tracks(self, clip, queries, segm_mask=None, grid_size=0, add_support_grid=False,
                               grid_query_frame=0, backward_tracking=False, return_scores=False):
        return self._sparse_tracks(clip, clip.video_shape, queries, segm_mask, grid_size, add_support_grid,
                                   grid_query_frame, backward_tracking, return_scores)

    def _sparse_tracks(self, clip, video_shape, queries, segm_mask=None, grid_size=0, add_support_grid=False,
                       grid_query_frame=0, backward_tracking=False, return_scores=False):
        queries = self._model_queries(clip, video_shape, queries, segm_mask, grid_size, add_support_grid,
                                      grid_query_frame)
        if backward_tracking:   # the clip played backwards (reference :187-209) is a reversed group
            inv = _reversed_queries(queries, clip.T)
            if queries.shape[1] * clip.loop_frames() <= BACKWARD_GROUP_TRACK_FRAMES:
                fwd, bwd = clip.track_groups([queries, inv], [False, True], return_scores)
            else:
                (fwd,), (bwd,) = (clip.track_groups([queries], [False], return_scores),
                                  clip.track_groups([inv], [True], return_scores))
        else:
            (fwd,), bwd = clip.track_groups([queries], [False], return_scores), None
        return self._finish(queries, fwd, bwd, video_shape, add_support_grid, return_scores)

    def _model_queries(self, clip, video_shape, queries, segm_mask=None, grid_size=0, add_support_grid=False,
                       grid_query_frame=0):
        """The queries [B,N,3] at model resolution (reference :100-160), support grid appended."""
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
        if add_support_grid:
            sup = get_points_on_a_grid(self.support_grid_size, self.interp_shape, device=dev)
            sup = torch.cat([torch.zeros_like(sup[:, :, :1]), sup], dim=2).repeat(B, 1, 1)
            queries = torch.cat([queries, sup], dim=1)
        return queries

    def _finish(self, queries, fwd, bwd, video_shape, add_support_grid=False, scores=False):
        """(tracks, visibility) of the forward pass, merged with the backward pass's before each query frame
        (reference :187-209), support grid dropped, query points pinned, scaled to the input (reference :161-190).
        scores=True: fwd / bwd also hold the confidence third, and the result gains the TrackScores of the same merge
        and columns, not pinned at the query points (one kernel still)."""
        B, T, C, H, W = video_shape
        ih, iw = self.interp_shape
        n_keep = queries.shape[1] - (self.support_grid_size ** 2 if add_support_grid else 0)
        # query points are, by definition, where they were asked for and visible (reference :173-185); one kernel
        fwd, bwd = [None if p is None else tuple(x.contiguous() for x in p[:3 if scores else 2]) for p in (fwd, bwd)]
        out = engine.finish_tracks(fwd, bwd, queries.float().contiguous(), n_keep, 0.9,
                                   ((W - 1) / (iw - 1), (H - 1) / (ih - 1)), scores=scores)
        return (out[0], out[1], TrackScores(out[2], out[3])) if scores else out


class _Device:
    """The device of a list call's clips, where `_model_queries` takes an `EncodedClip`."""

    def __init__(self, device):
        self.device = device


def _check_list_call(model, clips, queries, segm_mask, grid_size, grid_query_frame):
    """The ValueErrors of a list call, raised before any work."""
    if hasattr(model, "init_video_online_processing"):
        raise ValueError("a list of clips needs the offline model (offline=True)")
    B = len(clips)
    if B == 0:
        raise ValueError("the list of clips is empty")
    for name, lst in (("queries", queries), ("segm_mask", segm_mask)):
        if lst is not None and (not isinstance(lst, (list, tuple)) or len(lst) != B):
            raise ValueError(f"{name} must be a list of {B} entries, one per clip")
    for b, c in enumerate(clips):
        ingest.reject_encoded_clip(c, f"entry {b} of a list call")
        clip = torch.is_tensor(c) or isinstance(c, (ingest.YUVClip, ingest.Crop))
        if not clip or c.dim() != 5 or c.shape[0] != 1 or c.shape[1] < 1 or c.shape[2] != 3:
            raise ValueError(f"clip {b} must be a [1,T,3,H,W] tensor, got "
                             f"{tuple(c.shape) if clip else type(c).__name__}")
    for b, c in enumerate(clips):
        T = c.shape[1]
        q = None if queries is None else queries[b]
        if q is None:
            if grid_size <= 0:
                raise ValueError("a list of clips needs queries for every clip or grid_size > 0 "
                                 "(dense mode takes one clip)")
            if not 0 <= grid_query_frame < T:
                raise ValueError(f"clip {b}: grid_query_frame {grid_query_frame} lies outside its {T} frames")
            continue
        if not torch.is_tensor(q) or q.dim() != 3 or q.shape[0] != 1 or q.shape[2] != 3:
            raise ValueError(f"queries[{b}] must be a [1,N,3] tensor")
        t = q[0, :, 0].long()
        if t.numel() and (int(t.min()) < 0 or int(t.max()) >= T):
            raise ValueError(f"clip {b}: a query frame lies outside its {T} frames")


def _reversed_queries(queries, T: int):
    """The queries on the clip played backwards: query frame t becomes T-1-t (reference :192-195)."""
    inv = queries.clone()
    inv[:, :, 0] = T - inv[:, :, 0] - 1
    return inv


def _loop(model) -> str:
    """How a model runs the update loop over a clip, which decides the padding frames its pyramid holds."""
    if hasattr(model, "init_video_online_processing"):
        return f"sliding-window (window_len {model.window_len})"
    return "one-window"


class EncodedClip:
    """Clips (a batch of B) resized + normalised (cotracker_b200.ingest) and encoded once into one pyramid, made by
    `CoTrackerPredictor.encode` (and by every direct predictor call, for that call).  Every model pass of a call
    (dense offsets, backward tracking, the sub-batches of a batch that does not fit in device memory at once) runs on
    this one pyramid, and no pass writes to it, so one clip serves any number of calls.  A pass on the clip played
    backwards is a reversed query group (model `reversed_groups`): it reads the forward pyramid through a frame map, so
    device memory never holds a second pyramid and the pyramid is never reversed.

    It records what a call needs to scale queries and results and to check that a predictor may track it: `B`, `T`,
    the input frame size `input_hw` (`video_shape` = (B, T, 3, H, W)), the model resolution `interp_shape` (= `H`,
    `W`), the model's `stride` and update `loop`, its `device` and `weights`, the `weights_fingerprint()` of the model
    that encoded it.  `nbytes` is the device memory it holds.

    `to("cpu")` parks it in pinned host memory and frees its device memory; `to(device)` brings it back.  Levels 1-3 of
    the pyramid are 2x2 average pools of level 0, so only level 0 is parked (`host`, [B, T', H/s, W/s, 128] fp32, 6.3 of
    the 8.4 MB of a 384x512 frame), and the sliding-window model's padding frames are left out when they are copies of
    each clip's last frame.  On return the padding is copied again and `ct3_pyramid_pools` recomputes levels 1-3 with
    the kernel the encoder ran, so the pyramid is bit-identical to the one parked.  Each direction is one DMA per clip
    straight between the device pyramid and the pinned park: no staging buffer, and no pinned memory beyond the parked
    level 0 itself."""

    ITERS = 6

    def __init__(self, model, video, interp_shape, weights: Optional[str] = None):
        frames = ingest.prepare_video(video, interp_shape, ingest.model_device(model))
        self.model, self.device, self.weights = model, frames.device, weights
        self.video_shape = torch.Size(video.shape)
        self.B = video.shape[0]
        BT, _, self.H, self.W = frames.shape
        self.T = BT // self.B
        self.interp_shape = (self.H, self.W)
        self.stride, self.loop, self.pad = model.stride, _loop(model), model._clip_pad(self.T)
        self.host = None
        self.pyr = model._encode_clip(frames, B=self.B)

    @property
    def input_hw(self):
        return tuple(self.video_shape[3:])

    @property
    def parked(self) -> bool:
        return self.pyr is None

    @property
    def nbytes(self) -> int:
        return 0 if self.pyr is None else self.pyr.numel() * self.pyr.element_size()

    def __repr__(self) -> str:
        where = "parked on the host" if self.parked else f"device={self.device}"
        return f"EncodedClip(video_shape={tuple(self.video_shape)}, interp_shape={self.interp_shape}, {where})"

    def to(self, device) -> "EncodedClip":
        """In place: park the clip on the host ("cpu") or bring it (back) to a CUDA device.  -> the clip."""
        device = torch.device(device)
        if device.type == "cuda" and device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        if device.type == "cpu":
            if not self.parked:
                self._park()
        elif device.type != "cuda":
            raise ValueError(f"an EncodedClip lives on a CUDA device or parked on the host (\"cpu\"), not {device}")
        elif self.parked:
            self._unpark(device)
        elif device != self.device:
            self.pyr, self.device = self.pyr.to(device), device
        return self

    def _level0(self, pyr) -> torch.Tensor:
        """[B, T + pad, H/s * W/s * 128] view of level 0 of `pyr`, the first level of the flat layout."""
        s = self.stride
        n = (self.H // s) * (self.W // s) * engine.LATENT
        return pyr[:self.B * (self.T + self.pad) * n].view(self.B, self.T + self.pad, n)

    def _park(self):
        lv0 = self._level0(self.pyr)
        keep = self.T + self.pad
        if self.pad and torch.equal(lv0[:, self.T:], lv0[:, self.T - 1:self.T].expand(-1, self.pad, -1)):
            keep = self.T   # the padding is copies of each clip's last frame: remade on return
        s = self.stride
        host = torch.empty((self.B, keep, self.H // s, self.W // s, engine.LATENT), dtype=lv0.dtype, pin_memory=True)
        with torch.cuda.device(self.device):
            for b in range(self.B):
                host[b].view(keep, -1).copy_(lv0[b, :keep], non_blocking=True)
            torch.cuda.current_stream().synchronize()
        self.host, self.pyr, self.device = host, None, torch.device("cpu")

    def _unpark(self, device):
        s, Tp, keep = self.stride, self.T + self.pad, self.host.shape[1]
        H4, W4 = self.H // s, self.W // s
        with torch.cuda.device(device):
            pyr = torch.empty(engine.pyramid_layout(self.B * Tp, H4, W4)[3], dtype=self.host.dtype, device=device)
            lv0 = self._level0(pyr)
            for b in range(self.B):
                lv0[b, :keep].copy_(self.host[b].view(keep, -1), non_blocking=True)
            if keep < Tp:
                lv0[:, keep:].copy_(lv0[:, keep - 1:keep].expand(-1, Tp - keep, -1))
            engine.pyramid_pools(pyr, self.B * Tp, H4, W4)
        self.pyr, self.host, self.device = pyr, None, device

    def track_groups(self, groups, reversed_groups, scores=False):
        """Query groups [B,n_g,3] (model resolution) of every clip in one pass, or, when the batch does not fit in
        device memory, in one pass per sub-batch of clips (`plan_clip_passes`; groups are independent, so the split
        does not change a bit).  A flagged group tracks the clip played backwards, with query frames in reversed-clip
        time.  -> [(tracks [B,T,n_g,2], visibility [B,T,n_g])] per group, with the confidence [B,T,n_g] third when
        `scores` (otherwise it is dropped at once)."""
        if any(q.shape[0] != self.B for q in groups):
            raise ValueError(f"every query group must hold the batch's {self.B} clips")
        sizes = [q.shape[1] for q in groups]
        flags = list(reversed_groups)
        queries = torch.cat(groups, dim=1)
        passes = [(0, 1)]
        if self.B > 1:
            T_loop, H4, W4, budget, _ = self.pass_shape(any(flags))
            passes = plan_clip_passes(self.B, sizes, T_loop, H4, W4, budget, lambda n: self.pass_frames(any(flags), n))
        keep = 3 if scores else 2
        outs = [self.model._track_pyramid(self.pyr, self.T, self.H, self.W, queries[b0:b1], self.ITERS, sizes,
                                          reversed_groups=flags, clips=None if len(passes) == 1 else range(b0, b1))[:keep]
                for b0, b1 in passes]
        res = outs[0] if len(outs) == 1 else tuple(torch.cat([o[i] for o in outs], dim=0) for i in range(len(outs[0])))
        out, a = [], 0
        for n in sizes:
            out.append(tuple(x[:, :, a:a + n] for x in res))
            a += n
        return out

    def loop_frames(self) -> int:
        """Frames of one update loop: the clip, or the window of the sliding-window model."""
        return self.model.window_len if hasattr(self.model, "init_video_online_processing") else self.T

    def pass_frames(self, backward: bool, n_clips: int = 1):
        """Pyramid frames a pass over n_clips clips reads through its frame map: the whole pyramid in place for the
        one-window model, a gather of at most two windows per clip (one without reversed groups) for the sliding-window
        model.  None: one clip without reversed groups has no frame map."""
        if self.B == 1 and not backward:
            return None
        T_loop = self.loop_frames()
        return self.B * self.T if T_loop == self.T else n_clips * (2 if backward else 1) * T_loop

    def pass_shape(self, backward: bool):
        """(T, H4, W4, budget, frames) of `plan_dense_passes`: one update loop's frames (the window of the
        sliding-window model), the feature map, the free-memory budget of a pass and the pyramid frames a one-clip pass
        reads (`pass_frames`)."""
        s = self.model.stride
        budget = pass_budget_bytes(self.model, self.device, self.B * self.T, self.H, self.W)
        return self.loop_frames(), self.H // s, self.W // s, budget, self.pass_frames(backward)


_EncodedClip = EncodedClip   # its name while it lived inside one call, kept for code that imports it


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
                grid_query_frame: int = 0, add_support_grid=False, return_scores: bool = False,
                segm_mask: torch.Tensor = None):
        """-> (tracks, visibility), or with return_scores=True (tracks, visibility, TrackScores) of the frames so far
        (module docstring); (None, None[, None]) at the first step.  segm_mask ([1,1,H,W] at the chunk's frame size,
        first step, with grid_size): track only the grid points inside it, selected as the offline predictor selects
        them; add_support_grid then appends the support grid as it does to queries."""
        _check_return_scores(return_scores)
        ingest.reject_encoded_clip(video_chunk, "CoTrackerOnlinePredictor")
        B, T, C, H, W = video_chunk.shape
        dev = ingest.model_device(self.model)
        if is_first_step:
            # (re)start a video: reset the model state and remember the queries (reference :242-274)
            queries, self.N = self._first_step_queries(B, (H, W), queries, grid_size, grid_query_frame,
                                                       add_support_grid, dev, segm_mask)
            self.model.init_video_online_processing()
            self.queries = queries
            return (None, None, None) if return_scores else (None, None)

        if self.queries.shape[0] != B:   # the B streams of the first step advance together
            raise ValueError(f"the video was started with {self.queries.shape[0]} streams, this chunk holds {B}")
        frames = ingest.prepare_video(video_chunk, self.interp_shape, dev)
        out = self.model._track_online(frames, self.queries, 6, predict=self._tail(add_support_grid, (H, W)),
                                       scores=return_scores)
        return (out[0], out[1], TrackScores(out[2], out[3])) if return_scores else out

    def _first_step_queries(self, B, frame_hw, queries, grid_size, grid_query_frame, add_support_grid, dev,
                            segm_mask=None):
        """The queries [B,N,3] at model resolution a video started with these first-step arguments tracks, and the
        number of them the output keeps (reference :242-274).  segm_mask keeps the grid points inside it (ValueError
        when none is) and then treats them as queries: add_support_grid appends the support grid."""
        H, W = frame_hw
        ih, iw = self.interp_shape
        N = None
        as_queries = queries is not None or segm_mask is not None
        if segm_mask is not None:
            if queries is not None or grid_size <= 0:
                raise ValueError("segm_mask selects grid points: it needs grid_size > 0 and no queries")
            corners.check_mask(segm_mask, 1, (H, W), "segm_mask")
            grid_pts = get_points_on_a_grid(grid_size, self.interp_shape, device=dev)
            grid_pts = corners.grid_in_mask(grid_pts, corners.model_masks(segm_mask, self.interp_shape, dev)[0])
            if grid_pts.shape[1] == 0:
                raise ValueError(f"segm_mask keeps none of the {grid_size}x{grid_size} grid points")
            N = grid_pts.shape[1]
            queries = torch.cat([torch.ones_like(grid_pts[:, :, :1]) * grid_query_frame, grid_pts], dim=2)
            queries = queries.repeat(B, 1, 1)
        elif queries is not None:
            B, N, D = queries.shape
            assert D == 3
            queries = queries.to(dev).clone()
            queries[:, :, 1:] *= queries.new_tensor([(iw - 1) / (W - 1), (ih - 1) / (H - 1)])
        elif grid_size > 0:
            grid_pts = get_points_on_a_grid(grid_size, self.interp_shape, device=dev)
            N = grid_size ** 2
            queries = torch.cat([torch.ones_like(grid_pts[:, :, :1]) * grid_query_frame, grid_pts], dim=2)
            queries = queries.repeat(B, 1, 1)
        if as_queries and add_support_grid:   # the reference appends no support grid to a plain grid
            sup = get_points_on_a_grid(self.support_grid_size, self.interp_shape, device=dev)
            sup = torch.cat([torch.zeros_like(sup[:, :, :1]), sup], dim=2).repeat(B, 1, 1)
            queries = torch.cat([queries, sup], dim=1)
        return queries, N

    def _tail(self, add_support_grid, frame_hw):
        """(n_keep, scale_xy) of the output of a call on H x W chunks: the support grid dropped when the call asks for
        it, the tracks scaled from the model's resolution to the chunk's (reference :276-309)."""
        H, W = frame_hw
        ih, iw = self.interp_shape
        n_keep = self.N if add_support_grid else self.queries.shape[1]
        return n_keep, ((W - 1) / (iw - 1), (H - 1) / (ih - 1))
