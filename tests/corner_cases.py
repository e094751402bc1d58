"""Corner test helpers: a numpy float64 restatement of Shi-Tomasi corner selection (the contract of ct3_detect_corners,
include/ct3_b200.h, i.e. cv2.goodFeaturesToTrack with useHarrisDetector=False), and synthetic frames for it."""
import numpy as np
import torch


def gray(frame):
    """frame [3,H,W] fp32 -> g [H,W] fp32 = 0.299 R + 0.587 G + 0.114 B, evaluated left to right."""
    f = np.asarray(frame, dtype=np.float32)
    return np.float32(0.299) * f[0] + np.float32(0.587) * f[1] + np.float32(0.114) * f[2]


def response(g, block_size):
    """g [H,W] fp32 -> lambda [H,W] fp64: the smaller eigenvalue of the block's gradient covariance (unscaled)."""
    H, W = g.shape
    p = np.pad(g.astype(np.float64), 1, mode="reflect")      # numpy's "reflect" is reflect-101
    dx = ((p[:-2, 2:] - p[:-2, :-2]) + 2.0 * (p[1:-1, 2:] - p[1:-1, :-2])) + (p[2:, 2:] - p[2:, :-2])
    dy = ((p[2:, :-2] - p[:-2, :-2]) + 2.0 * (p[2:, 1:-1] - p[:-2, 1:-1])) + (p[2:, 2:] - p[:-2, 2:])
    r = block_size // 2
    px, py = np.pad(dx, r, mode="reflect"), np.pad(dy, r, mode="reflect")
    sxx, sxy, syy = np.zeros((H, W)), np.zeros((H, W)), np.zeros((H, W))
    for i in range(block_size):
        for j in range(block_size):
            u, v = px[i:i + H, j:j + W], py[i:i + H, j:j + W]
            sxx = sxx + u * u
            sxy = sxy + u * v
            syy = syy + v * v
    a, c = sxx * 0.5, syy * 0.5
    d = a - c
    return (a + c) - np.sqrt(d * d + sxy * sxy)


def exclusion_mask(H, W, points, radius):
    """uint8 [H,W]: 0 at pixels with (x - ex)^2 + (y - ey)^2 < radius^2 (fp64) from any point, 1 elsewhere."""
    mask = np.ones((H, W), np.uint8)
    if points is None or radius <= 0:
        return mask
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    r2 = float(radius) * float(radius)
    for ex, ey in np.asarray(points, dtype=np.float32).astype(np.float64):
        ddx, ddy = xs - ex, ys - ey
        mask[ddx * ddx + ddy * ddy < r2] = 0
    return mask


def select(lam, max_corners, quality_level, min_distance, mask=None):
    """Candidates of lambda [H,W] fp64 in order, then the greedy walk -> int64 [n,2] (x, y) in selection order."""
    H, W = lam.shape
    thr = float(quality_level) * lam.max()
    cand = []
    inner = lam[1:-1, 1:-1]
    nbr = np.max(np.stack([lam[1 + a:H - 1 + a, 1 + b:W - 1 + b] for a in (-1, 0, 1) for b in (-1, 0, 1)]), 0)
    ok = (inner > thr) & (inner == nbr)
    if mask is not None:
        ok &= mask[1:-1, 1:-1] != 0
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


def corners(frame, max_corners, quality_level=0.01, min_distance=10, block_size=3, exclude=None, exclude_radius=0):
    """The whole contract on one prepared frame [3,H,W] fp32 -> (corners int64 [n,2] (x, y), lambda [H,W] fp64)."""
    g = gray(frame)
    lam = response(g, block_size)
    mask = exclusion_mask(*g.shape, exclude, exclude_radius)
    return select(lam, max_corners, quality_level, min_distance, mask), lam


def textured_frame(H, W, seed=0):
    """A prepared-looking frame [3,H,W] fp32 in [-1, 1]: smooth blobs, edges and corners at several scales."""
    g = torch.Generator().manual_seed(seed)
    low = torch.rand(1, 3, max(2, H // 16), max(2, W // 16), generator=g)
    f = torch.nn.functional.interpolate(low, (H, W), mode="bilinear", align_corners=True)[0]
    ys, xs = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    for k in range(12):
        cy, cx = (torch.rand(2, generator=g) * torch.tensor([H, W])).tolist()
        hh, ww = (torch.rand(2, generator=g) * torch.tensor([H / 4, W / 4]) + 3).tolist()
        box = ((ys - cy).abs() < hh) & ((xs - cx).abs() < ww)
        f[k % 3] = torch.where(box, 1.0 - f[k % 3], f[k % 3])
    return (f * 2 - 1).float().contiguous()


def checkerboard(H, W, period=8):
    """[3,H,W] fp32 squares of `period` pixels in {-1, 1}: thousands of corners of exactly equal response."""
    ys, xs = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    c = (((ys // period) + (xs // period)) % 2).float() * 2 - 1
    return c[None].repeat(3, 1, 1).contiguous()
