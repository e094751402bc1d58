"""The flow_vis package (0.1, MIT; the Middlebury colour code of Baker et al., 2011) restated in numpy, as far as the
reference visualiser uses it: flow_vis.flow_to_color(flow) with its defaults.  It can stand in for the package:

    sys.modules["flow_vis"] = oracle.flow_vis_oracle

attainable(tracks, query_frame) bounds what a correct implementation may return for the reference's
flow_to_color(tracks - tracks[query_frame]): every operation of the colour code is pinned down by IEEE float64 except
arctan2, whose last bit differs between CPUs (numpy's SIMD path, glibc) and GPUs (CUDA documents 2 ulp).  The bounds
are the per-channel minimum and maximum of the colours obtained when the arctan2 result is moved by each of -4..+4 ulp.
"""
from __future__ import annotations

import numpy as np

ULPS = 4


def make_colorwheel() -> np.ndarray:
    """[55, 3] float64: RY, YG, GC, CB, BM, MR segments of 15, 6, 4, 11, 13 and 6 hues."""
    RY, YG, GC, CB, BM, MR = 15, 6, 4, 11, 13, 6
    wheel = np.zeros((RY + YG + GC + CB + BM + MR, 3))
    col = 0
    wheel[0:RY, 0] = 255
    wheel[0:RY, 1] = np.floor(255 * np.arange(0, RY) / RY)
    col += RY
    wheel[col:col + YG, 0] = 255 - np.floor(255 * np.arange(0, YG) / YG)
    wheel[col:col + YG, 1] = 255
    col += YG
    wheel[col:col + GC, 1] = 255
    wheel[col:col + GC, 2] = np.floor(255 * np.arange(0, GC) / GC)
    col += GC
    wheel[col:col + CB, 1] = 255 - np.floor(255 * np.arange(CB) / CB)
    wheel[col:col + CB, 2] = 255
    col += CB
    wheel[col:col + BM, 2] = 255
    wheel[col:col + BM, 0] = np.floor(255 * np.arange(0, BM) / BM)
    col += BM
    wheel[col:col + MR, 2] = 255 - np.floor(255 * np.arange(MR) / MR)
    wheel[col:col + MR, 0] = 255
    return wheel


def _colors(u, v, atan):
    """flow_uv_to_colors for normalised u, v and the arctan2(-v, -u) values `atan` -> uint8 [..., 3]."""
    wheel = make_colorwheel()
    ncols = wheel.shape[0]
    out = np.zeros(u.shape + (3,), np.uint8)
    rad = np.sqrt(np.square(u) + np.square(v))
    a = atan / np.pi
    fk = (a + 1) / 2 * (ncols - 1)
    k0 = np.floor(fk).astype(np.int32)
    k1 = k0 + 1
    k1[k1 == ncols] = 0
    f = fk - k0
    idx = rad <= 1
    for i in range(3):
        tmp = wheel[:, i]
        col = (1 - f) * (tmp[k0] / 255.0) + f * (tmp[k1] / 255.0)
        col[idx] = 1 - rad[idx] * (1 - col[idx])
        col[~idx] = col[~idx] * 0.75
        out[..., i] = np.floor(255 * col)
    return out


def _normalised(flow_uv):
    u, v = flow_uv[..., 0], flow_uv[..., 1]
    rad_max = np.max(np.sqrt(np.square(u) + np.square(v)))
    epsilon = 1e-5
    return u / (rad_max + epsilon), v / (rad_max + epsilon)


def flow_uv_to_colors(u, v, convert_to_bgr=False):
    out = _colors(u, v, np.arctan2(-v, -u))
    return out[..., ::-1].copy() if convert_to_bgr else out


def flow_to_color(flow_uv, clip_flow=None, convert_to_bgr=False):
    """flow [H, W, 2] (the reference passes int64 [T, N, 2]) -> uint8 [H, W, 3]."""
    assert flow_uv.ndim == 3, "input flow must have three dimensions"
    assert flow_uv.shape[2] == 2, "input flow must have shape [H,W,2]"
    if clip_flow is not None:
        flow_uv = np.clip(flow_uv, 0, clip_flow)
    u, v = _normalised(flow_uv)
    return flow_uv_to_colors(u, v, convert_to_bgr)


def attainable(tracks, query_frame: int, ulps: int = ULPS):
    """tracks: int64 [T, N, 2] as the reference holds them ((tracks + pad_value).long()).  -> (lo, hi) uint8 [T, N, 3]:
    the per-channel range of flow_to_color(tracks - tracks[query_frame]) over arctan2 results within +-ulps ulp of
    this host's."""
    tracks = np.asarray(tracks, dtype=np.int64)
    return attainable_uv(*_normalised(tracks - tracks[query_frame][None]), ulps=ulps)


def attainable_uv(u, v, ulps: int = ULPS):
    """attainable() for flow already normalised by rad_max + 1e-5 (float64 u, v of any shape)."""
    at = np.arctan2(-v, -u)
    lo = hi = _colors(u, v, at)
    for direction in (np.inf, -np.inf):
        p = at
        for _ in range(ulps):
            p = np.nextafter(p, direction)
            c = _colors(u, v, p)
            lo, hi = np.minimum(lo, c), np.maximum(hi, c)
    return lo, hi
