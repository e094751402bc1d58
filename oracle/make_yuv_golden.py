"""Generate tests/golden/yuv_cv2.npz: small YUV frames in each layout the library takes (nv12, i420, yuyv) and the
uint8 RGB OpenCV makes of them with cv2.cvtColor(frame, COLOR_YUV2RGB_{NV12|I420|YUYV}).  Needs cv2, which the tests
do not import:

    python oracle/make_yuv_golden.py

For each layout L and case C the file holds `L/C/yuv` (uint8 frames [T,H*3/2,W] or [T,H,W,2]) and `L/C/rgb` (uint8
[T,3,H,W]), plus `cv2_version`.  Cases:
    random   4 random frames of 24 x 32;
    odd      3 random frames of 30 x 46, whose chroma height 15 is odd;
    tiny     4 random frames of 2 x 2;
    flat     frames whose planes are all 0 or all 255, in every combination of Y, U and V;
    corners  every Y value 0..255 (a 16 x 16 frame) against each of the nine U, V pairs from {0, 128, 255}^2.
"""
from __future__ import annotations

import itertools
import os

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "yuv_cv2.npz")

CODES = {"nv12": cv2.COLOR_YUV2RGB_NV12, "i420": cv2.COLOR_YUV2RGB_I420, "yuyv": cv2.COLOR_YUV2RGB_YUYV}


def pack(layout: str, y: np.ndarray, u: np.ndarray, v: np.ndarray) -> np.ndarray:
    """One frame in `layout` from planes y [H,W], u and v [H/2,W/2] (4:2:0) or [H,W/2] (yuyv)."""
    H, W = y.shape
    if layout == "nv12":
        uv = np.stack([u, v], axis=-1).reshape(H // 2, W)
        return np.concatenate([y, uv], axis=0)
    if layout == "i420":
        return np.concatenate([y.reshape(-1), u.reshape(-1), v.reshape(-1)]).reshape(H * 3 // 2, W)
    out = np.empty((H, W, 2), np.uint8)
    out[..., 0] = y
    out[:, 0::2, 1] = u
    out[:, 1::2, 1] = v
    return out


def chroma_shape(layout: str, H: int, W: int):
    return (H, W // 2) if layout == "yuyv" else (H // 2, W // 2)


def frames(layout: str, planes) -> np.ndarray:
    return np.stack([pack(layout, *p) for p in planes])


def random_planes(rng, layout: str, T: int, H: int, W: int):
    ch = chroma_shape(layout, H, W)
    return [(rng.integers(0, 256, (H, W), dtype=np.uint8), rng.integers(0, 256, ch, dtype=np.uint8),
             rng.integers(0, 256, ch, dtype=np.uint8)) for _ in range(T)]


def cases(layout: str, rng):
    H, W = 4, 6
    ch = chroma_shape(layout, H, W)
    flat = [(np.full((H, W), a, np.uint8), np.full(ch, b, np.uint8), np.full(ch, c, np.uint8))
            for a, b, c in itertools.product((0, 255), repeat=3)]
    ys = np.arange(256, dtype=np.uint8).reshape(16, 16)
    ch = chroma_shape(layout, 16, 16)
    corners = [(ys, np.full(ch, b, np.uint8), np.full(ch, c, np.uint8))
               for b, c in itertools.product((0, 128, 255), repeat=2)]
    return {
        "random": random_planes(rng, layout, 4, 24, 32),
        "odd": random_planes(rng, layout, 3, 30, 46),
        "tiny": random_planes(rng, layout, 4, 2, 2),
        "flat": flat,
        "corners": corners,
    }


def main():
    rng = np.random.default_rng(20261018)
    out = {"cv2_version": np.array(cv2.__version__)}
    for layout, code in CODES.items():
        for name, planes in cases(layout, rng).items():
            yuv = frames(layout, planes)
            rgb = np.stack([cv2.cvtColor(np.ascontiguousarray(f), code).transpose(2, 0, 1) for f in yuv])
            out[f"{layout}/{name}/yuv"] = yuv
            out[f"{layout}/{name}/rgb"] = np.ascontiguousarray(rgb)
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}: {len(out) - 1} arrays, cv2 {cv2.__version__}")


if __name__ == "__main__":
    main()
