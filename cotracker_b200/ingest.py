"""One ingestion step for every predictor: the clip as the caller holds it -> normalised encoder input on the GPU.

    prepare_video(video [B,T,3,H,W], (ih, iw), device) -> frames [B*T,3,ih,iw] fp32 in [-1,1] on `device`

The frames of a batch come out clip after clip (clip b's at b*T ..), the order the encoder and the models take them in.

`video` may be uint8 (what decoders return) or float32 in 0..255, with any strides (a channels-last [T,H,W,3]
buffer seen through `permute` is read in place), on the device or on the host.  The resize and normalisation are one
library kernel (ct3_prepare_frames), bit-identical to the reference's
`2 * (F.interpolate(video, (ih, iw), mode="bilinear", align_corners=True) / 255) - 1`.

A device clip is one kernel call on the strided tensor.  A host clip is uploaded in chunks of k frames through two
pinned staging slots on a side stream: the host copy of chunk c+1 and its upload overlap the kernel on chunk c, and the
device never holds more than two raw chunks.  Staging memory is bounded: 2 * k * frame_bytes pinned host bytes plus
the same on the device, with k = max(1, min(T, STAGING_SLOT_BYTES // frame_bytes)) -- at most
2 * max(STAGING_SLOT_BYTES, frame_bytes) each (`staging_bytes`).  The clips of a host batch go through the same two
slots one after another, so the bound does not grow with B.

A `YUVClip` holds the clip as decoders and cameras emit it (NV12, I420, YUYV, 4:2:2 / 4:4:4 planar, and P010 / P016
/ 10-bit planar in 16-bit containers), with its colour matrix and range, and goes in wherever an RGB clip does.  Its
frames are converted, resized and normalised by one library kernel (ct3_prepare_frames_yuv[_fmt]), bit-identical to
the RGB path on the uint8 clip the header's integer formula makes of it (cv2.cvtColor(COLOR_YUV2RGB_*) for 8-bit
BT.601 limited range), and a host clip is uploaded as YUV bytes (1.5 bytes per pixel for 8-bit 4:2:0 instead of RGB's
3; a 16-bit 4:2:0 frame is 3) through the same two staging slots.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch

from . import engine

STAGING_SLOT_BYTES = 32 << 20   # one of the two staging slots; a frame larger than this gets a slot of its own


def chunk_frames(T: int, frame_bytes: int, slot_bytes: Optional[int] = None) -> int:
    """Frames per upload chunk: as many whole frames as fit in one staging slot (default STAGING_SLOT_BYTES), at least
    1, at most T."""
    if T < 1 or frame_bytes < 1:
        raise ValueError("T and frame_bytes must be >= 1")
    slot = STAGING_SLOT_BYTES if slot_bytes is None else slot_bytes
    return max(1, min(T, slot // frame_bytes))


def plan_chunks(T: int, frame_bytes: int, slot_bytes: Optional[int] = None) -> List[Tuple[int, int]]:
    """[t0, t1) frame ranges of the upload chunks, in order, covering 0..T-1."""
    k = chunk_frames(T, frame_bytes, slot_bytes)
    return [(t0, min(T, t0 + k)) for t0 in range(0, T, k)]


def staging_bytes(T: int, frame_bytes: int, slot_bytes: Optional[int] = None) -> int:
    """Pinned host bytes of a host-clip upload (the raw chunks on the device take the same): two slots of k frames."""
    return 2 * chunk_frames(T, frame_bytes, slot_bytes) * frame_bytes


def frame_is_dense(shape, strides) -> bool:
    """True when the 3*H*W elements of one frame [3,H,W] with these element strides fill a contiguous block (any
    dimension order, e.g. TCHW or THWC storage), so the frame can be copied as raw bytes."""
    dims = sorted((st, n) for n, st in zip(shape, strides) if n != 1)
    expect = 1
    for st, n in dims:
        if st != expect:
            return False
        expect *= n
    return True


def _dense_strides(shape, strides):
    """Strides of a dense frame seen from its first (lowest-address) element: unchanged for non-negative strides."""
    return tuple(st if n != 1 else 0 for n, st in zip(shape, strides))


class YUVClip:
    """A clip of YUV frames as decoders and cameras emit them, on the host or the device.  `layout` (FFmpeg's pix_fmt
    names) and `data`:
        "nv12"       uint8 [B,T,H*3/2,W]: H luma rows, then H/2 rows of interleaved U,V
        "i420"       uint8 [B,T,H*3/2,W]: the Y, U and V planes packed, as PyAV's `to_ndarray()` gives yuv420p
        "yuyv"       uint8 [B,T,H,W,2]: Y0 U Y1 V per pixel pair
        "yuv422p"    uint8 [B,T,2H,W]: the Y plane, then the H x W/2 U and V planes, packed
        "yuv444p"    uint8 [B,T,3H,W]: the Y, U and V planes of H x W, packed
        "p010", "p016"                          torch.uint16 [B,T,H*3/2,W]: nv12 with 16-bit samples, MSB-aligned (10
                                                or 16 significant bits; the low bits are ignored)
        "yuv420p10", "yuv422p10", "yuv444p10"   torch.uint16, planar as i420 / yuv422p / yuv444p, 10-bit LSB-aligned
                                                (the bits above bit 9 are ignored)
    H must be even for 4:2:0 and W for 4:2:0 / 4:2:2 (yuyv included).

    `matrix` ("bt601", "bt709" or "bt2020") and `full_range` describe the colour.  The clip stands for the uint8 RGB
    clip [B,T,3,H,W] that the integer formula of include/ct3_b200.h gives (a 10- or 16-bit frame rounded to 8 bits, as
    an rgb24 conversion rounds it).  With the defaults, BT.601 limited range, that is cv2.cvtColor(frame,
    COLOR_YUV2RGB_*) at 8 bits.  Only the matrix is applied: there is no PQ / HLG transfer function and no tone mapping.
    Every predictor and `OnlineStreams.push` take a YUVClip where they take that clip and give results `torch.equal` to
    it.  `shape` is that clip's logical (B, T, 3, H, W); `data` is read by `prepare_video` only."""

    def __init__(self, data: torch.Tensor, layout: str, *, matrix: str = "bt601", full_range: bool = False):
        if layout not in engine.YUV_FORMATS:
            raise ValueError(f"unknown YUV layout {layout!r}: one of {sorted(engine.YUV_FORMATS)}")
        engine.check_yuv_colour(matrix, full_range)
        want = f"[B,T,{engine.yuv_frame_shape(layout)[1:]}"
        dtype = engine.yuv_dtype(layout)
        if not torch.is_tensor(data) or data.dtype != dtype:
            raise ValueError(f"{layout} data must be a {dtype} tensor {want}, got "
                             f"{data.dtype if torch.is_tensor(data) else type(data).__name__}")
        hw = engine.yuv_frame_hw(layout, data.shape) if data.dim() == (5 if layout == "yuyv" else 4) else None
        if hw is None or min(data.shape[:2]) < 1 or min(hw) < 1:
            raise ValueError(f"{layout} data must be {want} with B, T, H, W >= 1, got {tuple(data.shape)}")
        xs, ys = engine.yuv_subsampling(layout)
        if (ys and hw[0] % 2) or (xs and hw[1] % 2):
            raise ValueError(f"{layout} frames must have an even {'width and height' if ys else 'width'}"
                             f", got H x W = {hw[0]} x {hw[1]}")
        self.data, self.layout, self.matrix, self.full_range = data, layout, matrix, full_range
        self.shape = torch.Size((data.shape[0], data.shape[1], 3) + tuple(hw))

    def dim(self) -> int:
        return 5

    @property
    def device(self) -> torch.device:
        return self.data.device

    @property
    def is_cuda(self) -> bool:
        return self.data.is_cuda

    def with_data(self, data: torch.Tensor) -> "YUVClip":
        """A clip of the same layout and colour over other frames (e.g. a slice of `data`)."""
        return YUVClip(data, self.layout, matrix=self.matrix, full_range=self.full_range)

    def to(self, device) -> "YUVClip":
        return self.with_data(self.data.to(device))

    def __repr__(self) -> str:
        colour = "" if (self.matrix, self.full_range) == ("bt601", False) else \
            f", {self.matrix}{' full range' if self.full_range else ''}"
        return f"YUVClip({self.layout}{colour}, shape={tuple(self.shape)}, device={self.device})"


def reject_encoded_clip(video, where: str):
    """TypeError when `video` is an `EncodedClip`: `where` takes pixels, and only CoTrackerPredictor takes a clip
    encoded already."""
    from .predictor import EncodedClip   # predictor imports this module
    if isinstance(video, EncodedClip):
        raise TypeError(f"{where} takes the video's pixels, not an EncodedClip (only CoTrackerPredictor calls take an "
                        "encoded clip)")


def model_device(model: torch.nn.Module) -> torch.device:
    p = next(model.parameters(), None)
    return p.device if p is not None else torch.device("cpu")


def prepare_video(video, out_hw, device, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """video [B,T,3,H,W] uint8 or float (0..255), host or device, any strides, or a `YUVClip` -> [B*T,3,oh,ow] fp32 in
    [-1,1] on device, clip after clip; each clip's frames are bit-identical to the call on that clip alone.
    out: an optional contiguous fp32 [B*T,3,oh,ow] destination on `device` (e.g. a slice of a larger frame batch).
    Other dtypes (float16, float64, ...) are cast to float32 first and then take the float32 path; for pixel values
    0..255 that cast is exact.  (Before this step existed they were resized in their own dtype, so results for them can
    differ from that in the last bits.)"""
    device = torch.device(device)
    if device.type != "cuda":
        raise engine.EngineError("cotracker_b200 runs on CUDA only; move the module to a GPU")
    if video.dim() != 5 or video.shape[0] < 1 or video.shape[1] < 1 or video.shape[2] != 3:
        raise ValueError(f"video must be [B,T,3,H,W] with B, T >= 1, got {tuple(video.shape)}")
    yuv = isinstance(video, YUVClip)
    if not yuv and video.dtype not in engine.FRAME_DTYPES:
        video = video.float()
    B, T = video.shape[:2]
    if video.is_cuda and video.device != device:
        video = video.to(device)
    shape = (B * T, 3, int(out_hw[0]), int(out_hw[1]))
    if out is None:
        out = torch.empty(shape, dtype=torch.float32, device=device)
    elif tuple(out.shape) != shape or out.dtype != torch.float32 or out.device != device or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous fp32 {shape} tensor on {device}")
    staging = None
    for b in range(B):
        clip = video.data[b] if yuv else video[b]
        if video.is_cuda and yuv:
            engine.prepare_frames_yuv(clip, video.layout, out_hw, out=out[b * T:(b + 1) * T], matrix=video.matrix,
                                      full_range=video.full_range)
        elif video.is_cuda:
            engine.prepare_frames(clip, out_hw, out=out[b * T:(b + 1) * T])
        else:
            staging = _prepare_host(clip, out_hw, out[b * T:(b + 1) * T], staging, video if yuv else None)
    return out


def _prepare_host(v: torch.Tensor, out_hw, out: torch.Tensor, staging=None, yuv: Optional[YUVClip] = None):
    """One host clip -> out [T,3,oh,ow] on the device: v [T,3,H,W], or the YUV frames of clip b of `yuv` (its
    data[b]), which are uploaded as they are, 1 or 2 bytes a sample, and converted on the device in its layout and
    colour.  Returns its staging buffers (pinned slots, device slots), which the next clip of a batch takes as
    `staging`."""
    layout = None if yuv is None else yuv.layout
    T, fshape = v.shape[0], tuple(v.shape[1:])
    oh, ow = int(out_hw[0]), int(out_hw[1])
    device = out.device
    fe = v[0].numel()                               # elements per frame
    esize = v.element_size()
    chunks = plan_chunks(T, fe * esize)
    k = chunks[0][1] - chunks[0][0]
    dense = frame_is_dense(fshape, v.stride()[1:]) and all(s >= 0 for s in v.stride())
    if layout is not None:   # the YUV kernel reads rows in their own order: a dense frame must be row-major
        dense = dense and v[0].is_contiguous()
    fstrides = _dense_strides(fshape, v.stride()[1:]) if dense else torch.empty(fshape, device="meta").stride()

    main = torch.cuda.current_stream(device)
    side = torch.cuda.Stream(device)
    if staging is None:
        staging = ([torch.empty(k * fe, dtype=v.dtype, pin_memory=True) for _ in range(2)],
                   [torch.empty(k * fe, dtype=v.dtype, device=device) for _ in range(2)])
    pinned, raw = staging
    copied = [torch.cuda.Event() for _ in range(2)]     # upload of the slot finished (side stream)
    consumed = [torch.cuda.Event() for _ in range(2)]   # kernel reading the slot finished (main stream)
    used = [False, False]
    # `raw` (and `out`) come from the caching allocator on the main stream, which only makes them safe to use in main-
    # stream order: main-stream work queued before this call may still use that memory.  The side stream's uploads
    # must therefore start after everything already queued on the main stream.
    side.wait_stream(main)
    for c, (t0, t1) in enumerate(chunks):
        slot, n = c % 2, t1 - t0
        if used[slot]:
            copied[slot].synchronize()                  # the pinned slot's previous upload must be done before reuse
        dst = pinned[slot][:n * fe].view(n, fe)
        if dense:
            # frame t starts at its lowest-address element: storage offset + t * stride_t for non-negative strides
            src = torch.as_strided(v, (n, fe), (v.stride(0), 1), v.storage_offset() + t0 * v.stride(0))
            dst.copy_(src)
        else:
            dst.copy_(v[t0:t1].contiguous().view(n, fe))
        with torch.cuda.stream(side):
            if used[slot]:
                side.wait_event(consumed[slot])         # the device slot is still read by the kernel of chunk c-2
            raw[slot][:n * fe].copy_(pinned[slot][:n * fe], non_blocking=True)
            copied[slot].record(side)
        main.wait_event(copied[slot])
        src_dev = torch.as_strided(raw[slot], (n,) + fshape, (fe,) + tuple(fstrides))
        if layout is None:
            engine.prepare_frames(src_dev, (oh, ow), out=out[t0:t1])
        else:
            engine.prepare_frames_yuv(src_dev, layout, (oh, ow), out=out[t0:t1], matrix=yuv.matrix,
                                      full_range=yuv.full_range)
        consumed[slot].record(main)
        used[slot] = True
    # the staging buffers go back to PyTorch's caches when this returns: uploads must be done with the pinned memory
    # (host wait below), and every side-stream use of the device slots is followed by a main-stream wait on `copied`,
    # so main-stream work that later reuses them is ordered after it
    for slot in range(2):
        if used[slot]:
            copied[slot].synchronize()
    return staging
