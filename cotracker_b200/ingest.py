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

A `Crop` stands for an h x w window of each frame of a clip or a `YUVClip`, at a top-left corner that may move from
frame to frame, and goes in wherever the clip does.  A device clip is read in place by the crop kernels
(ct3_prepare_frames_crop, ct3_prepare_frames_yuv_crop), which take the per-frame offsets from the device.  A host clip
stages only the windows through the two slots: an RGB window as it is, then the un-cropped kernel on it; a YUV window
as the smallest rectangle on the chroma grid that holds it (`yuv_window`), then the YUV crop kernel with the window's
residual offset (0 or 1) inside that rectangle.  Chunks are planned from the staged bytes, so a 1024 x 768 window of a
3840 x 2160 frame uploads about a tenth of the frame.
"""
from __future__ import annotations

import numbers
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


def _is_int(x) -> bool:
    return isinstance(x, numbers.Integral) and not isinstance(x, bool)


class Crop:
    """The h x w window of each frame of `video` whose top-left corner is `offset`, as a clip [B,T,3,h,w].

    video: anything `prepare_video` takes ([B,T,3,H,W] uint8 or float, host or device, any strides, or a `YUVClip`).
    size: (h, w) ints, 1 <= h <= H and 1 <= w <= W, the same in every frame.  offset: (top, left) ints for one window
    in every frame, or a CPU integer tensor [T,2] (one window per frame, shared by the B clips) or [B,T,2] of (top,
    left).  Every window lies inside its frame: 0 <= top <= H - h and 0 <= left <= W - w (ValueError otherwise,
    checked here on the host before any GPU work).  Frame (b, t) of the clip is video[b, t, :, top:top+h,
    left:left+w]; for a YUVClip, that window of the uint8 RGB clip it stands for.

    Every predictor, `OnlineStreams.push`, `EvaluationPredictor` and `detect_corners` take a Crop where they take that
    clip, with results `torch.equal` to the call on the materialised window and in window pixels; `to_frame` and
    `from_frame` convert to and from frame pixels.  `crop[b0:b1, t0:t1]` is the Crop of those clips and frames.
    `offsets` is the [B,T,2] int64 CPU tensor of (top, left); `shape` is (B, T, 3, h, w)."""

    def __init__(self, video, size, offset):
        from .predictor import EncodedClip   # predictor imports this module
        if isinstance(video, (Crop, EncodedClip)):
            raise TypeError(f"a Crop takes the video's pixels, not a {type(video).__name__}: crop the video itself")
        if not (torch.is_tensor(video) or isinstance(video, YUVClip)) or video.dim() != 5 or video.shape[2] != 3 \
                or min(video.shape[:2]) < 1:
            got = tuple(video.shape) if torch.is_tensor(video) else type(video).__name__
            raise ValueError(f"a Crop takes a video [B,T,3,H,W] with B, T >= 1 or a YUVClip, got {got}")
        B, T, _, H, W = video.shape
        if not isinstance(size, (tuple, list)) or len(size) != 2 or not all(_is_int(x) for x in size):
            raise ValueError(f"size must be (h, w) ints, got {size!r}")
        h, w = int(size[0]), int(size[1])
        if not (1 <= h <= H and 1 <= w <= W):
            raise ValueError(f"size (h, w) = {(h, w)} must lie in [1, {H}] x [1, {W}]")
        if torch.is_tensor(offset):
            if offset.device.type != "cpu" or offset.dtype.is_floating_point or offset.is_complex() \
                    or offset.dtype == torch.bool:
                raise ValueError(f"offset tensors must be CPU integer tensors, got {offset.dtype} on {offset.device}")
            if tuple(offset.shape) not in ((T, 2), (B, T, 2)):
                raise ValueError(f"offset must be (top, left), [T={T},2] or [B={B},T={T},2], got {tuple(offset.shape)}")
            offsets = offset.to(torch.int64).expand(B, T, 2)
        elif isinstance(offset, (tuple, list)) and len(offset) == 2 and all(_is_int(x) for x in offset):
            offsets = torch.tensor([int(offset[0]), int(offset[1])], dtype=torch.int64).expand(B, T, 2)
        else:
            raise ValueError(f"offset must be (top, left) ints or a CPU integer tensor, got {offset!r}")
        top, left = offsets[..., 0], offsets[..., 1]
        bad = (top < 0) | (top > H - h) | (left < 0) | (left > W - w)
        if bool(bad.any()):
            b, t = (int(i) for i in bad.nonzero()[0])
            raise ValueError(f"the {h} x {w} window at (top, left) = {tuple(offsets[b, t].tolist())} of clip {b}, "
                             f"frame {t} reaches outside the {H} x {W} frame")
        self.video, self.size, self.offsets = video, (h, w), offsets.contiguous()
        self.shape = torch.Size((B, T, 3, h, w))

    def dim(self) -> int:
        return 5

    @property
    def device(self) -> torch.device:
        return self.video.device

    @property
    def is_cuda(self) -> bool:
        return self.video.is_cuda

    def to(self, device) -> "Crop":
        return Crop(self.video.to(device), self.size, self.offsets)

    def __getitem__(self, key) -> "Crop":
        key = key if isinstance(key, tuple) else (key,)
        if len(key) > 2 or not all(isinstance(k, slice) for k in key):
            raise TypeError(f"a Crop is sliced over clips and frames only (crop[b0:b1, t0:t1]), got {key!r}")
        key = key + (slice(None),) * (2 - len(key))
        v = self.video
        return Crop(v.with_data(v.data[key]) if isinstance(v, YUVClip) else v[key], self.size, self.offsets[key])

    def to_frame(self, tracks: torch.Tensor, frames: Optional[slice] = None) -> torch.Tensor:
        """tracks [B,T',N,2] (x, y) in window pixels -> frame pixels: (left, top) of each frame added, one fp32 add
        on tracks' device.  frames: the frames of the clip tracks covers (default all T; e.g. slice(T - L, T) for the
        last L frames of an online result)."""
        off = self.offsets if frames is None else self.offsets[:, frames]
        if not torch.is_tensor(tracks) or tracks.dim() != 4 or tracks.shape[-1] != 2 \
                or tuple(tracks.shape[:2]) != tuple(off.shape[:2]):
            raise ValueError(f"tracks must be [{off.shape[0]},{off.shape[1]},N,2], got "
                             f"{tuple(tracks.shape) if torch.is_tensor(tracks) else type(tracks).__name__}")
        return tracks + off.flip(-1).to(device=tracks.device, dtype=torch.float32)[:, :, None]

    def from_frame(self, queries: torch.Tensor) -> torch.Tensor:
        """queries [B,N,3] (t, x, y) in frame pixels -> window pixels: the (left, top) of frame int(t) of the query's
        clip subtracted from (x, y), on queries' device.  ValueError for a query frame outside the clip."""
        B, T = self.shape[:2]
        if not torch.is_tensor(queries) or queries.dim() != 3 or queries.shape[0] != B or queries.shape[2] != 3:
            raise ValueError(f"queries must be [{B},N,3], got "
                             f"{tuple(queries.shape) if torch.is_tensor(queries) else type(queries).__name__}")
        t = queries[..., 0].long()
        if t.numel() and bool(((t < 0) | (t >= T)).any()):
            raise ValueError(f"a query frame lies outside the clip's {T} frames")
        off = self.offsets.to(queries.device)
        sel = off[torch.arange(B, device=queries.device)[:, None], t]   # [B,N,2] (top, left)
        out = queries.clone()
        out[..., 1:] -= sel.flip(-1).to(queries.dtype)
        return out

    def __repr__(self) -> str:
        inner = repr(self.video) if isinstance(self.video, YUVClip) else \
            f"tensor(shape={tuple(self.video.shape)}, dtype={self.video.dtype}, device={self.video.device})"
        return f"Crop({inner}, size={self.size}, shape={tuple(self.shape)})"


def yuv_window(layout: str, offsets: torch.Tensor, size):
    """Where the h x w windows at offsets [T,2] (top, left) of a YUV clip are staged from on the host: for each frame
    the smallest rectangle that holds its window and lies on the chroma grid (top / left rounded down to even on a
    subsampled axis, the end rounded up).  -> (origin [T,2] and extent [T,2] (rows, columns) of the rectangles,
    residual [T,2] = offsets - origin, 0 or 1: the window's offset inside its rectangle).  A staged frame holds the
    largest extent, extent.amax(0), so that every staged frame has one layout."""
    xs, ys = engine.yuv_subsampling(layout)
    grid = torch.tensor([2 if ys else 1, 2 if xs else 1], dtype=torch.int64)
    origin = offsets - offsets % grid
    end = offsets + torch.tensor(size, dtype=torch.int64)
    end = end + (-end) % grid
    return origin, end - origin, offsets - origin


def _yuv_planes(x: torch.Tensor, layout: str, H: int, W: int):
    """The planes of YUV frames x [n,<one H x W frame>] as views [(plane [n,rows,cols(,2)], ys, xs)]: a window's
    rows and columns in a plane are its frame rows >> ys and columns >> xs (NV12's interleaved chroma keeps the
    luma columns; YUYV is one [n,H,W,2] plane)."""
    n = x.shape[0]
    xs, ys = engine.yuv_subsampling(layout)
    if layout == "yuyv":
        return [(x, 0, 0)]
    if layout in ("nv12", "p010", "p016"):
        return [(x[:, :H], 0, 0), (x[:, H:H + H // 2], 1, 0)]
    flat = x.reshape(n, -1)
    cH, cW = H >> ys, W >> xs
    y, c = H * W, cH * cW
    return [(flat[:, :y].view(n, H, W), 0, 0), (flat[:, y:y + c].view(n, cH, cW), ys, xs),
            (flat[:, y + c:y + 2 * c].view(n, cH, cW), ys, xs)]


def _staged_strides(shape, strides):
    """Element strides of a dense frame of `shape` laid out in the dimension order of `strides` (by magnitude):
    a window of a channels-last frame is staged channels-last, so it is copied row by row."""
    out, acc = [0] * len(shape), 1
    for d in sorted(range(len(shape)), key=lambda d: abs(strides[d])):
        out[d] = acc
        acc *= shape[d]
    return tuple(out)


def _runs(rows: torch.Tensor, t0: int, t1: int):
    """[a, b) ranges of t0..t1 over which rows [T,k] does not change."""
    a = t0
    for t in range(t0 + 1, t1 + 1):
        if t == t1 or not torch.equal(rows[t], rows[a]):
            yield a, t
            a = t


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
    """video [B,T,3,H,W] uint8 or float (0..255), host or device, any strides, a `YUVClip` or a `Crop` of either ->
    [B*T,3,oh,ow] fp32 in [-1,1] on device, clip after clip; each clip's frames are bit-identical to the call on that
    clip alone (for a Crop, on its materialised window).
    out: an optional contiguous fp32 [B*T,3,oh,ow] destination on `device` (e.g. a slice of a larger frame batch).
    Other dtypes (float16, float64, ...) are cast to float32 first and then take the float32 path; for pixel values
    0..255 that cast is exact.  (Before this step existed they were resized in their own dtype, so results for them can
    differ from that in the last bits.)"""
    device = torch.device(device)
    if device.type != "cuda":
        raise engine.EngineError("cotracker_b200 runs on CUDA only; move the module to a GPU")
    if video.dim() != 5 or video.shape[0] < 1 or video.shape[1] < 1 or video.shape[2] != 3:
        raise ValueError(f"video must be [B,T,3,H,W] with B, T >= 1, got {tuple(video.shape)}")
    crop = video if isinstance(video, Crop) else None
    if crop is not None:
        video = crop.video
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
    kw = {}
    if crop is not None and video.is_cuda:   # the offsets of every clip, a few bytes, for the crop kernels
        offsets = crop.offsets.to(device=device, dtype=torch.int32)
    staging = None
    for b in range(B):
        clip = video.data[b] if yuv else video[b]
        if crop is not None and video.is_cuda:
            kw = dict(crop=(offsets[b], crop.size))
        if video.is_cuda and yuv:
            engine.prepare_frames_yuv(clip, video.layout, out_hw, out=out[b * T:(b + 1) * T], matrix=video.matrix,
                                      full_range=video.full_range, **kw)
        elif video.is_cuda:
            engine.prepare_frames(clip, out_hw, out=out[b * T:(b + 1) * T], **kw)
        else:
            staging = _prepare_host(clip, out_hw, out[b * T:(b + 1) * T], staging, video if yuv else None,
                                    None if crop is None else (crop.offsets[b], crop.size))
    return out


def _prepare_host(v: torch.Tensor, out_hw, out: torch.Tensor, staging=None, yuv: Optional[YUVClip] = None,
                  window=None):
    """One host clip -> out [T,3,oh,ow] on the device: v [T,3,H,W], or the YUV frames of clip b of `yuv` (its
    data[b]), which are uploaded as they are, 1 or 2 bytes a sample, and converted on the device in its layout and
    colour.  window: None, or (offsets [T,2] (top, left), (h, w)) of a `Crop`: only the windows are staged (an RGB
    window in the frame's dimension order; a YUV window as its `yuv_window` rectangle, then cropped on the device).
    Returns its staging buffers (pinned slots, device slots), which the next clip of a batch takes as `staging`."""
    layout = None if yuv is None else yuv.layout
    T, fshape = v.shape[0], tuple(v.shape[1:])
    oh, ow = int(out_hw[0]), int(out_hw[1])
    device = out.device
    if window is None:
        sshape = fshape                             # shape of one staged frame
    elif layout is None:
        offsets, (h, w) = window
        sshape = (3, h, w)
    else:
        offsets, (h, w) = window
        H, W = yuv.shape[3:]
        origin, extent, residual = yuv_window(layout, offsets, (h, w))
        hs, ws = (int(x) for x in extent.amax(0))
        sshape = (hs, ws, 2) if layout == "yuyv" else (hs * engine._YUV_ROWS[layout] // 2, ws)
    fe = 1                                          # elements per staged frame
    for n in sshape:
        fe *= n
    esize = v.element_size()
    chunks = plan_chunks(T, fe * esize)
    k = chunks[0][1] - chunks[0][0]
    if window is None:
        dense = frame_is_dense(fshape, v.stride()[1:]) and all(s >= 0 for s in v.stride())
        if layout is not None:   # the YUV kernel reads rows in their own order: a dense frame must be row-major
            dense = dense and v[0].is_contiguous()
        fstrides = _dense_strides(fshape, v.stride()[1:]) if dense else torch.empty(fshape, device="meta").stride()
    elif layout is None:
        fstrides = _staged_strides(sshape, v.stride()[1:])
    else:
        fstrides = torch.empty(sshape, device="meta").stride()
        crop = (residual.to(device=device, dtype=torch.int32), (h, w))

    main = torch.cuda.current_stream(device)
    side = torch.cuda.Stream(device)
    if staging is None or staging[0][0].numel() < k * fe:
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
        if window is not None:
            staged = torch.as_strided(pinned[slot], (n,) + sshape, (fe,) + tuple(fstrides))
            for a, b in _runs(offsets, t0, t1):         # one copy per run of frames with the same window
                if layout is None:
                    top, left = offsets[a].tolist()
                    staged[a - t0:b - t0].copy_(v[a:b, :, top:top + h, left:left + w])
                    continue
                (top, left), (r, q) = origin[a].tolist(), extent[a].tolist()
                for (sp, ys, xs), (dp, _, _) in zip(_yuv_planes(v[a:b], layout, H, W),
                                                    _yuv_planes(staged[a - t0:b - t0], layout, hs, ws)):
                    dp[:, :r >> ys, :q >> xs].copy_(sp[:, top >> ys:(top + r) >> ys, left >> xs:(left + q) >> xs])
        elif dense:
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
        src_dev = torch.as_strided(raw[slot], (n,) + sshape, (fe,) + tuple(fstrides))
        if layout is None:
            engine.prepare_frames(src_dev, (oh, ow), out=out[t0:t1])
        else:
            kw = {} if window is None else dict(crop=(crop[0][t0:t1], crop[1]))
            engine.prepare_frames_yuv(src_dev, layout, (oh, ow), out=out[t0:t1], matrix=yuv.matrix,
                                      full_range=yuv.full_range, **kw)
        consumed[slot].record(main)
        used[slot] = True
    # the staging buffers go back to PyTorch's caches when this returns: uploads must be done with the pinned memory
    # (host wait below), and every side-stream use of the device slots is followed by a main-stream wait on `copied`,
    # so main-stream work that later reuses them is ordered after it
    for slot in range(2):
        if used[slot]:
            copied[slot].synchronize()
    return staging
