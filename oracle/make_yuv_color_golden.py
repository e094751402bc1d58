"""Generate tests/golden/yuv_color_cv2.npz: an outside anchor for the full-range BT.601 conversion of
ct3_prepare_frames_yuv_fmt.  OpenCV's cv2.cvtColor(frame, COLOR_YCrCb2RGB) is full-range BT.601 (JPEG) on 4:4:4 frames
whose channels are Y, Cr, Cb, for 8-bit and for 16-bit samples.  Needs cv2, which the tests do not import:

    python oracle/make_yuv_color_golden.py

For each depth d in (8, 16) the file holds the planes `d/y` [T,H,W], `d/u` and `d/v` [T,H/2,W/2] (4:2:0 chroma, uint8
or uint16) and `d/rgb` [T,3,H,W], what cv2 makes of the 4:4:4 frames that repeat each chroma sample over its 2x2 block
(uint8, or uint16 at 16 bits), plus `cv2_version`.  The frames are random, then the corners of the sample range: every
combination of 0, the midpoint and the maximum in Y, U and V.
"""
from __future__ import annotations

import itertools
import os

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "yuv_color_cv2.npz")
H, W = 24, 32


def planes(rng, bits: int):
    dtype = np.uint8 if bits == 8 else np.uint16
    top = (1 << bits) - 1
    y = [rng.integers(0, top + 1, (H, W)) for _ in range(3)]
    u = [rng.integers(0, top + 1, (H // 2, W // 2)) for _ in range(3)]
    v = [rng.integers(0, top + 1, (H // 2, W // 2)) for _ in range(3)]
    for a, b, c in itertools.product((0, 1 << (bits - 1), top), repeat=3):
        y.append(np.full((H, W), a))
        u.append(np.full((H // 2, W // 2), b))
        v.append(np.full((H // 2, W // 2), c))
    return [np.stack(p).astype(dtype) for p in (y, u, v)]


def main():
    rng = np.random.default_rng(20261019)
    out = {"cv2_version": np.array(cv2.__version__)}
    for bits in (8, 16):
        y, u, v = planes(rng, bits)
        up = lambda c: c.repeat(2, axis=1).repeat(2, axis=2)   # noqa: E731
        ycrcb = np.stack([y, up(v), up(u)], axis=-1)            # channel order Y, Cr, Cb
        rgb = np.stack([cv2.cvtColor(np.ascontiguousarray(f), cv2.COLOR_YCrCb2RGB).transpose(2, 0, 1) for f in ycrcb])
        out[f"{bits}/y"], out[f"{bits}/u"], out[f"{bits}/v"] = y, u, v
        out[f"{bits}/rgb"] = np.ascontiguousarray(rgb)
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}: {len(out) - 1} arrays, cv2 {cv2.__version__}")


if __name__ == "__main__":
    main()
