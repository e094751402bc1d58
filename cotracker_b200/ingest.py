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

A `YUVClip` holds the clip as decoders and cameras emit it (NV12, I420, YUYV) and goes in wherever an RGB clip does.
Its frames are converted, resized and normalised by one library kernel (ct3_prepare_frames_yuv), bit-identical to the
RGB path on the uint8 clip cv2.cvtColor(COLOR_YUV2RGB_*) makes of it, and a host clip is uploaded as YUV bytes (1.5
bytes per pixel for 4:2:0 instead of RGB's 3) through the same two staging slots.
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
    """A clip of uint8 YUV frames: data [B,T,H*3/2,W] for layout "nv12" (H luma rows, then H/2 rows of interleaved U,V)
    or "i420" (the Y, U and V planes packed, as PyAV's `to_ndarray()` gives yuv420p), or [B,T,H,W,2] for "yuyv"
    (Y0 U Y1 V per pixel pair); on the host or the device.  H and W must be even (W only, for yuyv).

    It stands for the RGB clip [B,T,3,H,W] whose frames are cv2.cvtColor(frame, COLOR_YUV2RGB_{NV12|I420|YUYV}): every
    predictor and `OnlineStreams.push` take it where they take that clip and give results `torch.equal` to it.  `shape`
    is that clip's logical (B, T, 3, H, W); `data` is read by `prepare_video` only."""

    def __init__(self, data: torch.Tensor, layout: str):
        if layout not in engine.YUV_LAYOUTS:
            raise ValueError(f"unknown YUV layout {layout!r}: one of {sorted(engine.YUV_LAYOUTS)}")
        want = "[B,T,H,W,2]" if layout == "yuyv" else "[B,T,H*3/2,W]"
        if not torch.is_tensor(data) or data.dtype != torch.uint8:
            raise ValueError(f"{layout} data must be a uint8 tensor {want}, got "
                             f"{data.dtype if torch.is_tensor(data) else type(data).__name__}")
        hw = engine.yuv_frame_hw(layout, data.shape) if data.dim() == (5 if layout == "yuyv" else 4) else None
        if hw is None or min(data.shape[:2]) < 1 or min(hw) < 1:
            raise ValueError(f"{layout} data must be {want} with B, T, H, W >= 1, got {tuple(data.shape)}")
        if hw[1] % 2 or (layout != "yuyv" and hw[0] % 2):
            raise ValueError(f"{layout} frames must have an even {'width' if layout == 'yuyv' else 'width and height'}"
                             f", got H x W = {hw[0]} x {hw[1]}")
        self.data, self.layout = data, layout
        self.shape = torch.Size((data.shape[0], data.shape[1], 3) + tuple(hw))

    def dim(self) -> int:
        return 5

    @property
    def device(self) -> torch.device:
        return self.data.device

    @property
    def is_cuda(self) -> bool:
        return self.data.is_cuda

    def to(self, device) -> "YUVClip":
        return YUVClip(self.data.to(device), self.layout)

    def __repr__(self) -> str:
        return f"YUVClip({self.layout}, shape={tuple(self.shape)}, device={self.device})"


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
    layout = video.layout if yuv else None
    for b in range(B):
        clip = video.data[b] if yuv else video[b]
        if video.is_cuda and yuv:
            engine.prepare_frames_yuv(clip, layout, out_hw, out=out[b * T:(b + 1) * T])
        elif video.is_cuda:
            engine.prepare_frames(clip, out_hw, out=out[b * T:(b + 1) * T])
        else:
            staging = _prepare_host(clip, out_hw, out[b * T:(b + 1) * T], staging, layout)
    return out


def _prepare_host(v: torch.Tensor, out_hw, out: torch.Tensor, staging=None, layout: Optional[str] = None):
    """One host clip -> out [T,3,oh,ow] on the device: v [T,3,H,W], or with a YUV `layout` the clip's YUV frames (a
    `YUVClip`'s data[b]), which are uploaded as they are and converted on the device.  Returns its staging buffers
    (pinned slots, device slots), which the next clip of a batch takes as `staging`."""
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
            engine.prepare_frames_yuv(src_dev, layout, (oh, ow), out=out[t0:t1])
        consumed[slot].record(main)
        used[slot] = True
    # the staging buffers go back to PyTorch's caches when this returns: uploads must be done with the pinned memory
    # (host wait below), and every side-stream use of the device slots is followed by a main-stream wait on `copied`,
    # so main-stream work that later reuses them is ordered after it
    for slot in range(2):
        if used[slot]:
            copied[slot].synchronize()
    return staging
