"""Mask test helpers, on top of tests/corner_cases.py: the float64 restatement of masked Shi-Tomasi selection (the
contract of ct3_detect_corners_masked, include/ct3_b200.h, i.e. cv2.goodFeaturesToTrack with a `mask`), ATen's
nearest-neighbour index rule (ct3_prepare_masks) in numpy fp32, and a few region masks."""
import numpy as np

import corner_cases as C


def select_masked(lam, max_corners, quality_level, min_distance, region, exclude=None):
    """corner_cases.select with a region: the threshold's maximum is taken over the region's pixels only, the 3x3
    maximum still over every pixel, and a candidate must lie in the region (and outside the exclusion discs, uint8
    `exclude`).  -> int64 [n,2] (x, y) in selection order."""
    H, W = lam.shape
    inside = np.asarray(region) != 0
    if not inside.any():
        return np.zeros((0, 2), np.int64)
    thr = float(quality_level) * lam[inside].max()
    inner = lam[1:-1, 1:-1]
    nbr = np.max(np.stack([lam[1 + a:H - 1 + a, 1 + b:W - 1 + b] for a in (-1, 0, 1) for b in (-1, 0, 1)]), 0)
    ok = (inner > thr) & (inner == nbr) & inside[1:-1, 1:-1]
    if exclude is not None:
        ok &= exclude[1:-1, 1:-1] != 0
    ys, xs = np.nonzero(ok)
    ys, xs = ys + 1, xs + 1
    vals = lam[ys, xs]
    idx = ys.astype(np.int64) * W + xs
    order = np.lexsort((-idx, -vals))                 # lambda descending, then raster index descending
    ys, xs = ys[order], xs[order]
    md2 = float(min_distance) * float(min_distance)
    kept = []
    for x, y in zip(xs.tolist(), ys.tolist()):
        if len(kept) == max_corners:
            break
        if md2 > 0 and any((x - kx) * (x - kx) + (y - ky) * (y - ky) < md2 for kx, ky in kept):
            continue
        kept.append((x, y))
    return np.asarray(kept, dtype=np.int64).reshape(-1, 2)


def corners_masked(frame, region, max_corners, quality_level=0.01, min_distance=10, block_size=3, exclude=None,
                   exclude_radius=0):
    """The whole masked contract on one prepared frame [3,H,W] fp32 and a region [H,W] -> (corners int64 [n,2],
    lambda [H,W] fp64)."""
    g = C.gray(frame)
    lam = C.response(g, block_size)
    excl = C.exclusion_mask(*g.shape, exclude, exclude_radius)
    return select_masked(lam, max_corners, quality_level, min_distance, region, excl), lam


def nearest_index(n_out, n_in):
    """ATen's nearest source index of every output index: min(floor(d * s), n_in - 1), s = fp32(n_in) / n_out and the
    product in fp32."""
    s = np.float32(n_in) / np.float32(n_out)
    d = np.arange(n_out, dtype=np.float32)
    return np.minimum(np.floor(d * s).astype(np.int64), n_in - 1)


def exact_index(n_out, n_in):
    """floor(d * n_in / n_out) in integers: what the fp32 rule approximates."""
    return np.minimum(np.arange(n_out, dtype=np.int64) * n_in // n_out, n_in - 1)


def resize_mask(mask, out_hw):
    """mask [H,W] (any dtype) -> uint8 [oh,ow], 1 where the nearest source pixel is nonzero (ct3_prepare_masks)."""
    m = np.asarray(mask)
    H, W = m.shape
    ys, xs = nearest_index(out_hw[0], H), nearest_index(out_hw[1], W)
    return (m[ys][:, xs] != 0).astype(np.uint8)


def disc(H, W, cy, cx, r):
    """uint8 [H,W]: 1 inside the disc of radius r around (cx, cy)."""
    ys, xs = np.mgrid[0:H, 0:W]
    return (((ys - cy) ** 2 + (xs - cx) ** 2) < r * r).astype(np.uint8)


def box(H, W, y0, y1, x0, x1):
    """uint8 [H,W]: 1 on rows [y0, y1) and columns [x0, x1)."""
    m = np.zeros((H, W), np.uint8)
    m[y0:y1, x0:x1] = 1
    return m


def without_global_max(lam, r=40):
    """A region that leaves out a disc of radius r around the frame's largest response: its own maximum is smaller, so
    the masked threshold is not the unmasked one."""
    H, W = lam.shape
    y, x = np.unravel_index(np.argmax(lam), lam.shape)
    return 1 - disc(H, W, y, x, r)
