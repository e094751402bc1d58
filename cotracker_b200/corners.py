"""Where to put tracks: Shi-Tomasi corners of the frame the tracker sees, detected on the GPU.

    queries = detect_corners(video, 300)            # [1,n,3] (frame, x, y) in frame pixels, for B = 1
    tracks, visibility = model(video, queries=queries)

The detector is cv2.goodFeaturesToTrack(gray, max_corners, quality_level, min_distance, mask, block_size,
useHarrisDetector=False) restated exactly (ct3_detect_corners in include/ct3_b200.h).  It runs on the prepared fp32
model-resolution frame (interp_shape, values in [-1, 1]) the predictors track on, not on the original frame, so
min_distance and exclude_radius are model-resolution pixels.  The points come back in frame pixels, scaled by
(W-1)/(iw-1), (H-1)/(ih-1) as the predictors scale tracks, so they go straight back in as queries.
`OnlineStreams.seed_corners` adds such corners to a running stream, away from its own tracks.

A region mask keeps the corners on one object (cv2's `mask` argument, ct3_detect_corners_masked):

    queries = detect_corners(video, 300, mask=object_mask)   # object_mask [1,1,H,W] at frame size, nonzero = inside

Masks are resized to the model resolution on the device (ct3_prepare_masks), exactly as the offline predictor resizes
`segm_mask`: F.interpolate(mask.float(), interp_shape, mode="nearest") != 0.  `grid_in_mask` is the predictor's rule
for which grid points a mask keeps.
"""
from __future__ import annotations

import numbers

import torch

from . import engine, ingest


def _is_int(x) -> bool:
    return isinstance(x, numbers.Integral) and not isinstance(x, bool)


def _is_real(x) -> bool:
    return isinstance(x, numbers.Real) and not isinstance(x, bool) and x == x and abs(x) != float("inf")


def check_params(max_corners, quality_level, min_distance, block_size, exclude_radius=0) -> None:
    """Raise ValueError unless the detector's parameters are in range (what ct3_detect_corners accepts)."""
    if not _is_int(max_corners) or max_corners < 1:
        raise ValueError(f"max_corners must be an int >= 1, got {max_corners!r}")
    if not _is_real(quality_level) or not 0 < quality_level <= 1:
        raise ValueError(f"quality_level must be in (0, 1], got {quality_level!r}")
    if not _is_real(min_distance) or min_distance < 0:
        raise ValueError(f"min_distance must be a finite number >= 0, got {min_distance!r}")
    if not _is_int(block_size) or block_size not in (3, 5, 7):
        raise ValueError(f"block_size must be 3, 5 or 7, got {block_size!r}")
    if not _is_real(exclude_radius) or exclude_radius < 0:
        raise ValueError(f"exclude_radius must be a finite number >= 0, got {exclude_radius!r}")


def params(max_corners, quality_level=0.01, min_distance=10, block_size=3, exclude_radius=0) -> engine.CornerParams:
    """One frame's ct3_corner_params, range-checked."""
    check_params(max_corners, quality_level, min_distance, block_size, exclude_radius)
    return engine.CornerParams(int(max_corners), int(block_size), float(quality_level), float(min_distance),
                               float(exclude_radius))


def clip_frame(video, t: int):
    """Frame t of every clip of `video` ([B,T,3,H,W], a YUVClip or a Crop), as a one-frame clip of the same kind."""
    if isinstance(video, ingest.YUVClip):
        return video.with_data(video.data[:, t:t + 1])
    return video[:, t:t + 1]


def _exclusion_list(exclude, B: int):
    """exclude: None, a tensor [B,E,2] or a list of B tensors [E_b,2] -> a list of B fp32 tensors [E_b,2] or None."""
    if exclude is None:
        return None
    if torch.is_tensor(exclude):
        if exclude.dim() != 3 or exclude.shape[0] != B or exclude.shape[2] != 2:
            raise ValueError(f"exclude must be [B={B},E,2] or a list of B [E_b,2] tensors, got {tuple(exclude.shape)}")
        exclude = list(exclude)
    if not isinstance(exclude, (list, tuple)) or len(exclude) != B:
        raise ValueError(f"exclude must be [B={B},E,2] or a list of B [E_b,2] tensors")
    for e in exclude:
        if not torch.is_tensor(e) or e.dim() != 2 or e.shape[1] != 2 or e.dtype in (torch.bool, torch.complex64,
                                                                                     torch.complex128):
            raise ValueError("every exclusion entry must be a real tensor [E_b,2] of (x, y) frame pixels")
    return exclude


def check_mask(mask, B: int, frame_hw, name: str = "mask") -> None:
    """Raise ValueError unless `mask` is a real or bool tensor [B,1,H,W] or [1,1,H,W] at frame size (H, W)."""
    H, W = frame_hw
    if not torch.is_tensor(mask) or mask.dim() != 4 or mask.shape[0] not in (1, B) or mask.shape[1] != 1 \
            or tuple(mask.shape[2:]) != (H, W) or mask.is_complex():
        got = tuple(mask.shape) if torch.is_tensor(mask) else type(mask).__name__
        raise ValueError(f"{name} must be a real or bool tensor [{B},1,{H},{W}] or [1,1,{H},{W}] at frame size, "
                         f"got {got}")


def model_masks(mask: torch.Tensor, interp_shape, device) -> torch.Tensor:
    """Frame-size masks [B,1,H,W] (any real dtype or bool, host or device) -> [B,ih,iw] uint8 on `device`, 1 where
    F.interpolate(mask.float(), interp_shape, mode="nearest") != 0: the offline predictor's resize of segm_mask,
    computed by ct3_prepare_masks."""
    m = mask[:, 0].to(device)
    if m.dtype not in engine.MASK_DTYPES:   # nonzero-ness commutes with the nearest resize
        m = m != 0
    return engine.prepare_masks(m, interp_shape)


def grid_in_mask(grid_pts: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
    """Grid points [1,n,2] (x, y) at model resolution -> those inside mask [ih,iw] (`model_masks`), read at
    (round(y), round(x)) as the offline predictor selects them for segm_mask: [1,m,2], m may be 0."""
    keep = mask[grid_pts[0, :, 1].round().long(), grid_pts[0, :, 0].round().long()] != 0
    return grid_pts[:, keep]


@torch.no_grad()
def detect_corners(video, max_corners: int, *, frame: int = 0, quality_level: float = 0.01, min_distance: float = 10,
                   block_size: int = 3, exclude=None, exclude_radius: float = 0, interp_shape=(384, 512), mask=None):
    """Shi-Tomasi corners of frame `frame` of each clip of `video`, as queries for the predictors.

    video: anything `prepare_video` takes, [B,T,3,H,W] uint8 or float, host or device, a `YUVClip` or a `Crop`; only
    frame `frame` of each clip is prepared (at interp_shape) and searched.  max_corners, quality_level, min_distance and
    block_size are goodFeaturesToTrack's; min_distance is in model-resolution pixels.  exclude: points [B,E,2] or a
    list of B [E_b,2], (x, y) in frame pixels like queries; no corner lies closer than exclude_radius
    (model-resolution pixels) to one of its clip's points.  mask: None, or a region per clip [B,1,H,W] or one for
    every clip [1,1,H,W], at frame size, host or device, nonzero = inside: corners lie inside it, with cv2's `mask`
    semantics (the quality threshold is relative to the best response inside the mask; an empty mask gives none).
    -> queries [1,n,3] (frame, x, y) in frame pixels, best corner first, for B = 1; a list of B of them otherwise (the
    list-of-queries form CoTrackerPredictor takes).  Runs on the video's device, or the current CUDA device for a host
    video; only the B corner counts are copied to the host."""
    check_params(max_corners, quality_level, min_distance, block_size, exclude_radius)
    ingest.reject_encoded_clip(video, "detect_corners")
    if not (isinstance(video, (ingest.YUVClip, ingest.Crop)) or torch.is_tensor(video)) or video.dim() != 5 \
            or video.shape[2] != 3:
        raise ValueError(f"video must be [B,T,3,H,W], a YUVClip or a Crop, got {getattr(video, 'shape', type(video))}")
    B, T, _, H, W = video.shape
    if B < 1 or T < 1 or H < 2 or W < 2:
        raise ValueError(f"video must have B, T >= 1 and H, W >= 2, got {tuple(video.shape)}")
    if not _is_int(frame) or not 0 <= frame < T:
        raise ValueError(f"frame must be an int in [0, {T}), got {frame!r}")
    if len(interp_shape) != 2 or not all(_is_int(x) and x >= block_size for x in interp_shape):
        raise ValueError(f"interp_shape must be (ih, iw) ints >= block_size = {block_size}, got {interp_shape!r}")
    excl = _exclusion_list(exclude, B)
    if mask is not None:
        check_mask(mask, B, (H, W))
    ih, iw = interp_shape
    dev = video.device if video.is_cuda else torch.device("cuda", torch.cuda.current_device())
    frames = ingest.prepare_video(clip_frame(video, frame), (ih, iw), dev)
    points = None
    if excl is not None and max(e.shape[0] for e in excl) > 0:
        pts = torch.zeros(B, max(e.shape[0] for e in excl), 2, device=dev)
        for b, e in enumerate(excl):
            e = e.to(dev, torch.float32)
            pts[b, :e.shape[0]] = e * e.new_tensor([(iw - 1) / (W - 1), (ih - 1) / (H - 1)])
        points = (pts, [e.shape[0] for e in excl])
    region = None if mask is None else model_masks(mask, (ih, iw), dev).expand(B, ih, iw)
    found, counts = engine.detect_corners(frames, params(max_corners, quality_level, min_distance, block_size,
                                                         exclude_radius), points, mask=region)
    scale = found.new_tensor([(W - 1) / (iw - 1), (H - 1) / (ih - 1)])
    out = []
    for b, n in enumerate(counts.tolist()):
        xy = found[b, :n] * scale
        out.append(torch.cat([xy.new_full((n, 1), float(frame)), xy], 1)[None])
    return out[0] if B == 1 else out
