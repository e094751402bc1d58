"""ctypes binding of libct3_b200.so (C ABI: include/ct3_b200.h).

PyTorch is plumbing here: it owns device memory and the CUDA stream; every tensor is handed to the
library as a raw device pointer.  There is NO fallback: if the shared library is missing or a call
fails, a RuntimeError is raised (the product path never routes through the oracle or eager PyTorch).
"""
from __future__ import annotations

import ctypes
import os
from typing import List, Optional, Sequence

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("CT3_B200_LIB", os.path.join(_HERE, "lib", "libct3_b200.so"))   # env override: A/B builds

LATENT, LEVELS, P, VOL, VOL_PAD = 128, 4, 49, 2401, 2432
HID, VIRT, XDIM, XDIM_PAD = 384, 64, 1110, 1152

_lib = None


class EngineError(RuntimeError):
    pass


class OnlineStream(ctypes.Structure):
    """ct3_online_stream (include/ct3_b200.h): one stream of a streaming window pass."""
    _fields_ = [("coords", ctypes.c_void_p), ("vis", ctypes.c_void_p), ("conf", ctypes.c_void_p),
                ("cap", ctypes.c_int64), ("len", ctypes.c_int64), ("tracks", ctypes.c_void_p),
                ("visibility", ctypes.c_void_p), ("ind", ctypes.c_int32), ("T", ctypes.c_int32), ("n", ctypes.c_int32),
                ("first", ctypes.c_int32), ("frame0", ctypes.c_int32), ("n_keep", ctypes.c_int32),
                ("scale_x", ctypes.c_float), ("scale_y", ctypes.c_float), ("out_first", ctypes.c_int64),
                ("ring", ctypes.c_int32), ("pad", ctypes.c_int32)]


class LoopShape(ctypes.Structure):
    """ct3_loop_shape (include/ct3_b200.h): one update-loop pass."""
    _fields_ = [("T", ctypes.c_int), ("N", ctypes.c_int), ("H4", ctypes.c_int), ("W4", ctypes.c_int),
                ("G", ctypes.c_int), ("group_sizes", ctypes.POINTER(ctypes.c_int32)), ("T_pyr", ctypes.c_int),
                ("group_frames", ctypes.POINTER(ctypes.c_int32)), ("slab_tracks", ctypes.c_int),
                ("group_T", ctypes.POINTER(ctypes.c_int32))]


def _signatures():
    """name -> (restype, argtypes) of every entry point of include/ct3_b200.h"""
    c_int, c_size_t, c_void_p, c_char_p = ctypes.c_int, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_char_p
    i64, i64p = ctypes.c_int64, ctypes.POINTER(ctypes.c_int64)
    intp = ctypes.POINTER(ctypes.c_int)
    return {
        "ct3_version": (c_int, []),
        "ct3_last_error": (c_char_p, []),
        "ct3_set_option": (c_int, [c_char_p, c_int]),
        "ct3_get_option": (c_int, [c_char_p, intp]),
        "ct3_precision_info": (c_int, [c_int, c_int, c_int, intp, intp, intp]),
        "ct3_volume_is_support_major": (c_int, [c_int, c_int, c_int, intp]),
        "ct3_num_weight_tensors": (c_int, []),
        "ct3_weight_name": (c_char_p, [c_int]),
        "ct3_packed_weights_bytes": (c_int, [ctypes.POINTER(c_size_t)]),
        "ct3_pack_weights": (c_int, [ctypes.POINTER(c_void_p), c_int, c_void_p, c_size_t, c_void_p]),
        "ct3_pyramid_layout": (c_int, [c_int, c_int, c_int, i64p, intp, intp, i64p]),
        "ct3_prepare_pyramid": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
        "ct3_prepare_frames": (c_int, [c_void_p, c_int, c_int, c_int, c_int, i64, i64, i64, i64, c_int, c_int, c_void_p,
                                       c_void_p]),
        "ct3_finish_tracks": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                      ctypes.c_float, ctypes.c_float, ctypes.c_float, c_void_p, c_void_p, c_void_p]),
        "ct3_online_window_begin": (c_int, [ctypes.POINTER(OnlineStream), c_int, c_int, c_int, c_int, c_int, c_void_p,
                                            c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                            c_void_p, c_size_t, c_void_p]),
        "ct3_online_window_end": (c_int, [ctypes.POINTER(OnlineStream), c_int, c_int, c_int, c_void_p, c_void_p,
                                          c_void_p, c_int, ctypes.c_float, c_void_p, c_size_t, c_void_p]),
        "ct3_render_prepare": (c_int, [c_void_p, c_int, c_int, c_int, c_int, i64, i64, i64, i64, c_int, c_int, c_void_p,
                                       c_void_p]),
        "ct3_render_workspace_bytes": (c_int, [c_int, c_int, c_int, c_int, c_int, ctypes.POINTER(c_size_t)]),
        "ct3_render_tracks": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                      c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
        "ct3_render_flow_workspace_bytes": (c_int, [c_int, c_int, ctypes.POINTER(c_size_t)]),
        "ct3_render_flow_colors": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
        "ct3_sample_support": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
        "ct3_workspace_bytes": (c_int, [ctypes.POINTER(LoopShape), ctypes.POINTER(c_size_t)]),
        "ct3_update_loop": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_int, ctypes.POINTER(LoopShape), c_void_p, c_size_t, c_void_p]),
        "ct3_corr_sample": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p,
                                    c_size_t, c_void_p]),
        "ct3_loop_tokens": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
        "ct3_linear": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
        "ct3_split_rows": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
        "ct3_split_rows_fp16": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
        "ct3_linear_prec": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
        "ct3_linear_ex": (c_int, [c_void_p, i64, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int,
                                  c_void_p, i64, c_int, c_void_p, i64, c_int, c_int, c_void_p]),
        "ct3_layernorm": (c_int, [c_void_p, c_int, c_void_p, c_void_p, ctypes.c_float, c_void_p, c_void_p]),
        "ct3_time_block_attention_workspace_bytes": (c_int, [c_int, c_int, ctypes.POINTER(c_size_t)]),
        "ct3_time_block_attention": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p, c_size_t,
                                             c_void_p]),
        "ct3_updateformer": (c_int, [c_void_p, c_void_p, c_int, c_int, ctypes.POINTER(ctypes.c_int32), c_int, c_void_p,
                                     c_void_p, c_size_t, c_void_p]),
        "ct3_attention_workspace_bytes": (c_int, [c_int, c_int, c_int, ctypes.POINTER(c_size_t)]),
        "ct3_attention": (c_int, [c_int, c_void_p, c_void_p, c_int, c_int, ctypes.POINTER(ctypes.c_int32), c_int, c_void_p,
                                  c_void_p, c_size_t, c_void_p]),
        "ct3_upsample_concat": (c_int, [ctypes.POINTER(c_void_p), intp, intp, intp, c_int, c_int, c_int, c_void_p, c_void_p]),
        "ct3_enc_tail_packed_bytes": (c_int, [ctypes.POINTER(c_size_t)]),
        "ct3_enc_tail_pack": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
        "ct3_enc_tail_workspace_bytes": (c_int, [c_int, c_int, c_int, ctypes.POINTER(c_size_t)]),
        "ct3_enc_tail": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
        "ct3_encoder_num_weight_tensors": (c_int, []),
        "ct3_encoder_weight_name": (c_char_p, [c_int]),
        "ct3_encoder_packed_bytes": (c_int, [ctypes.POINTER(c_size_t)]),
        "ct3_encoder_pack": (c_int, [ctypes.POINTER(c_void_p), c_int, c_void_p, c_size_t, c_void_p]),
        "ct3_encoder_workspace_bytes": (c_int, [c_int, c_int, c_int, ctypes.POINTER(c_size_t)]),
        "ct3_encoder": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
        "ct3_profile_enable": (c_int, [c_int]),
        "ct3_profile_read": (c_int, [ctypes.POINTER(ctypes.c_double), intp, ctypes.POINTER(ctypes.c_double)]),
    }


_SIGNATURES = _signatures()
EXPORTED_SYMBOLS = list(_SIGNATURES)


def lib():
    """Load (once) and return the shared library; raises EngineError if it is not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise EngineError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(or `make -C cotracker_b200/csrc`). There is no CPU/eager fallback.")
        try:
            handle = ctypes.CDLL(LIB_PATH)
        except OSError as e:  # pragma: no cover
            raise EngineError(f"cannot load {LIB_PATH}: {e}") from e
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(handle, name)  # AttributeError if the symbol is missing -> loud
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


def _check(rc: int, what: str):
    if rc != 0:
        msg = lib().ct3_last_error().decode("utf-8", "replace")
        raise EngineError(f"{what} failed (code {rc}): {msg}")


def _call(name: str, device, *args):
    """lib().<name>(*args) with `device` current; raises EngineError naming the entry point if it fails."""
    with torch.cuda.device(device):
        _check(getattr(lib(), name)(*args), name)


def _size(name: str, *args) -> int:
    """A size query: lib().<name>(*args, &out) -> out."""
    n = ctypes.c_size_t(0)
    _check(getattr(lib(), name)(*args, ctypes.byref(n)), name)
    return n.value


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _stream(device) -> ctypes.c_void_p:
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _req(t: torch.Tensor, dtype, name: str):
    if not t.is_cuda:
        raise EngineError(f"{name} must be a CUDA tensor (no CPU fallback)")
    if t.dtype != dtype:
        raise EngineError(f"{name} must be {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise EngineError(f"{name} must be contiguous")
    return t


def set_option(name: str, value: int):
    _check(lib().ct3_set_option(name.encode(), int(value)), f"ct3_set_option({name})")


def get_option(name: str) -> int:
    v = ctypes.c_int(0)
    _check(lib().ct3_get_option(name.encode(), ctypes.byref(v)), f"ct3_get_option({name})")
    return v.value


def precision_info(T: int = 16, H4: int = 96, W4: int = 128):
    """-> (corr_products, fc1_products, volume_bytes_per_element) in effect for this thread's options."""
    a, b, c = ctypes.c_int(0), ctypes.c_int(0), ctypes.c_int(0)
    _check(lib().ct3_precision_info(T, H4, W4, ctypes.byref(a), ctypes.byref(b), ctypes.byref(c)), "ct3_precision_info")
    return a.value, b.value, c.value


def precision_summary(T: int = 16, H4: int = 96, W4: int = 128) -> dict:
    """What bench.py prints as `dtype`: the arithmetic each GEMM group computes in (no precision claim beyond it)."""
    corr, fc1, vb = precision_info(T, H4, W4)
    name = {3: "x3 (split x split: hi*hi+lo*hi+hi*lo)", 2: "x2 (fp16 plane x split fp16)", 1: "x1 (single fp16 product)"}
    return {
        "dtype": (f"transformer + corr_mlp.fc2 + input_transform: bf16x3; correlation einsum: "
                  f"{'bf16' if corr == 3 else 'fp16'}{name[corr][:2]}; corr_mlp.fc1: {'bf16' if fc1 == 3 else 'fp16'}"
                  f"{name[fc1][:2]}; fp32 accumulate, fp32 softmax/LayerNorm/GELU"),
        "products": f"3 (bf16 split) except correlation einsum {corr} and corr_mlp.fc1 {fc1}",
        "corr_products": corr, "fc1_products": fc1, "volume_bytes_per_element": vb,
    }


def weight_names() -> List[str]:
    L = lib()
    return [L.ct3_weight_name(i).decode() for i in range(L.ct3_num_weight_tensors())]


def packed_weights_bytes() -> int:
    return _size("ct3_packed_weights_bytes")


def pack_weights(state: dict, device) -> torch.Tensor:
    """state: mapping state-dict key -> tensor (any device); returns the packed device buffer."""
    names = weight_names()
    tensors = []
    for k in names:
        if k not in state:
            raise EngineError(f"missing weight '{k}'")
        tensors.append(state[k].detach().to(device=device, dtype=torch.float32).contiguous())
    arr = (ctypes.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])
    nbytes = packed_weights_bytes()
    packed = torch.empty(nbytes, dtype=torch.uint8, device=device)
    _call("ct3_pack_weights", device, arr, len(tensors), _ptr(packed), nbytes, _stream(device))
    torch.cuda.current_stream(device).synchronize()  # `tensors` may be temporaries
    return packed


def pyramid_layout(T: int, H4: int, W4: int):
    off = (ctypes.c_int64 * 4)()
    h = (ctypes.c_int * 4)()
    w = (ctypes.c_int * 4)()
    tot = ctypes.c_int64(0)
    _check(lib().ct3_pyramid_layout(T, H4, W4, off, h, w, ctypes.byref(tot)), "ct3_pyramid_layout")
    return list(off), list(h), list(w), tot.value


def prepare_pyramid(fmaps: torch.Tensor) -> torch.Tensor:
    """fmaps [T,128,H4,W4] fp32 (raw fnet output) -> flat channels-last normalised 4-level pyramid."""
    _req(fmaps, torch.float32, "fmaps")
    T, C, H4, W4 = fmaps.shape
    if C != LATENT:
        raise EngineError("fmaps must have 128 channels")
    *_, total = pyramid_layout(T, H4, W4)
    pyr = torch.empty(total, dtype=torch.float32, device=fmaps.device)
    _call("ct3_prepare_pyramid", fmaps.device, _ptr(fmaps), T, H4, W4, _ptr(pyr), _stream(fmaps.device))
    return pyr


FRAME_DTYPES = {torch.uint8: 0, torch.float32: 1}   # CT3_FRAMES_U8, CT3_FRAMES_F32


def prepare_frames(src: torch.Tensor, out_hw, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """src [T,3,H,W] uint8 or float32 CUDA tensor with any strides (e.g. a permuted [T,H,W,3] decoder buffer) ->
    [T,3,oh,ow] fp32 = 2 * (bilinear(align_corners=True) resize / 255) - 1, bit-identical to the ATen expression.
    out: optional contiguous fp32 destination of that shape."""
    if not src.is_cuda:
        raise EngineError("src must be a CUDA tensor (no CPU fallback)")
    if src.dtype not in FRAME_DTYPES:
        raise EngineError(f"src must be uint8 or float32, got {src.dtype}")
    if src.dim() != 4 or src.shape[1] != 3:
        raise EngineError(f"src must be [T,3,H,W], got {tuple(src.shape)}")
    T, _, H, W = src.shape
    oh, ow = int(out_hw[0]), int(out_hw[1])
    if out is None:
        out = torch.empty(T, 3, oh, ow, dtype=torch.float32, device=src.device)
    _req(out, torch.float32, "out")
    if tuple(out.shape) != (T, 3, oh, ow) or out.device != src.device:
        raise EngineError(f"out must be [{T},3,{oh},{ow}] on {src.device}")
    _call("ct3_prepare_frames", src.device, _ptr(src), FRAME_DTYPES[src.dtype], T, H, W, *src.stride(), oh, ow, _ptr(out),
          _stream(src.device))
    return out


def finish_tracks(fwd, bwd, queries: torch.Tensor, n_keep: int, threshold: float, scale_xy):
    """The predictor's tail in one kernel (ct3_finish_tracks in include/ct3_b200.h).  fwd = (tracks [B,T,N,2],
    visibility probabilities [B,T,N]) of the forward pass, bwd = the same of the pass on the clip played backwards (in
    reversed-clip time) or None, queries [B,N,3] at model resolution; all fp32 on one device.
    -> (tracks [B,T,n_keep,2] fp32 scaled by scale_xy, visibility [B,T,n_keep] bool)."""
    tensors = [("fwd tracks", fwd[0]), ("fwd visibility", fwd[1]), ("queries", queries)]
    if bwd is not None:
        tensors += [("bwd tracks", bwd[0]), ("bwd visibility", bwd[1])]
    for name, t in tensors:
        _req(t, torch.float32, name)
    if queries.dim() != 3 or queries.shape[2] != 3:
        raise EngineError(f"queries must be [B,N,3], got {tuple(queries.shape)}")
    B, N, _ = queries.shape
    dev = queries.device
    T = fwd[0].shape[1] if fwd[0].dim() == 4 else -1
    for name, t in tensors:
        want = (B, N, 3) if name == "queries" else (B, T, N, 2) if name.endswith("tracks") else (B, T, N)
        if tuple(t.shape) != want or t.device != dev:
            raise EngineError(f"{name} must be {want} on {dev}, got {tuple(t.shape)} on {t.device}")
    n_keep = int(n_keep)
    tracks = torch.empty(B, T, max(n_keep, 0), 2, dtype=torch.float32, device=dev)
    visibility = torch.empty(B, T, max(n_keep, 0), dtype=torch.bool, device=dev)
    _call("ct3_finish_tracks", dev, _ptr(fwd[0]), _ptr(fwd[1]), _ptr(None if bwd is None else bwd[0]),
          _ptr(None if bwd is None else bwd[1]), _ptr(queries), B, T, N, n_keep, float(threshold), float(scale_xy[0]),
          float(scale_xy[1]), _ptr(tracks), _ptr(visibility), _stream(dev))
    return tracks, visibility


QUERY_FRAME_LIMIT = 1 << 30   # ct3_online_window_begin compares query frames clamped to +-2^30
STREAM_FRAME_LIMIT = 1 << 30  # ct3_online_window_* take a window at stream frame ind only while ind + S <= 2^30


def online_stream(hist, length: int, ind: int, T: int, first: int, frame0: int, out=None, n_keep: int = 0,
                  scale_xy=(1.0, 1.0), *, out_first: int = 0, ring: bool = False) -> OnlineStream:
    """One entry of a streaming window pass (ct3_online_stream): hist = (coords [cap,n,2], vis [cap,n], conf [cap,n])
    fp32 histories with `length` frames written, the window at stream frame `ind` with T real frames, the stream's
    tracks from `first` in the pass and its window at pyramid frame `frame0`; out = (tracks [ind+T-out_first,n_keep,2]
    fp32, visibility [ind+T-out_first,n_keep] bool or uint8) for window_end's predictor output of stream frames
    [out_first, ind+T), or None.  ring: the history holds frame f at row f mod cap (its last cap frames only)."""
    c, v, q = hist
    for t, dtype, name in ((c, torch.float32, "history coords"), (v, torch.float32, "history vis"),
                           (q, torch.float32, "history conf")):
        _req(t, dtype, name)
    cap, n = v.shape
    if tuple(c.shape) != (cap, n, 2) or tuple(q.shape) != (cap, n):
        raise EngineError(f"histories must be [cap,n,2], [cap,n], [cap,n], got {tuple(c.shape)}, {tuple(v.shape)}, "
                          f"{tuple(q.shape)}")
    e = OnlineStream(c.data_ptr(), v.data_ptr(), q.data_ptr(), cap, int(length), None, None, int(ind), int(T), n,
                     int(first), int(frame0), 0, float(scale_xy[0]), float(scale_xy[1]), int(out_first), int(bool(ring)))
    if out is not None:
        tr, vi = out
        _req(tr, torch.float32, "tracks")
        if not vi.is_cuda or vi.dtype not in (torch.bool, torch.uint8) or not vi.is_contiguous():
            raise EngineError("visibility must be a contiguous CUDA bool or uint8 tensor")
        rows = int(ind) + int(T) - int(out_first)
        if tuple(tr.shape) != (rows, int(n_keep), 2) or tuple(vi.shape) != (rows, int(n_keep)):
            raise EngineError(f"output must be [{rows},{n_keep},2] and [{rows},{n_keep}], got {tuple(tr.shape)} and "
                              f"{tuple(vi.shape)}")
        e.tracks, e.visibility, e.n_keep = tr.data_ptr(), vi.data_ptr(), int(n_keep)
    return e


def _online_table(streams, device):
    """Host array of the entries and the device scratch the library copies it into."""
    table = (OnlineStream * max(1, len(streams)))(*streams)
    ws = torch.empty(ctypes.sizeof(table), dtype=torch.uint8, device=device)
    return table, ws


def online_window_begin(streams, S: int, step: int, stride: int, T_pyr: int, qframes: torch.Tensor,
                        qcoords: torch.Tensor):
    """ct3_online_window_begin: streams = `online_stream` entries of one pass, qframes [N] int32 (stream time, within
    +-QUERY_FRAME_LIMIT), qcoords [N,2] fp32 (feature-grid units) -> (valid [N] uint8, entering [N] uint8, rel [N]
    int32, coords_init [S,N,2], vis_init [S,N], conf_init [S,N])."""
    _req(qframes, torch.int32, "qframes")
    _req(qcoords, torch.float32, "qcoords")
    N = qframes.shape[0]
    dev = qframes.device
    if tuple(qcoords.shape) != (N, 2) or qcoords.device != dev:
        raise EngineError(f"qcoords must be [{N},2] on {dev}")
    valid = torch.empty(N, dtype=torch.uint8, device=dev)
    entering = torch.empty(N, dtype=torch.uint8, device=dev)
    rel = torch.empty(N, dtype=torch.int32, device=dev)
    coords = torch.empty(S, N, 2, dtype=torch.float32, device=dev)
    vis = torch.empty(S, N, dtype=torch.float32, device=dev)
    conf = torch.empty(S, N, dtype=torch.float32, device=dev)
    table, ws = _online_table(streams, dev)
    _call("ct3_online_window_begin", dev, table, len(streams), int(S), int(step), int(stride), int(T_pyr),
          _ptr(qframes), _ptr(qcoords), N, _ptr(valid), _ptr(entering), _ptr(rel), _ptr(coords), _ptr(vis), _ptr(conf),
          _ptr(ws), ws.numel(), _stream(dev))
    return valid, entering, rel, coords, vis, conf


def online_window_end(streams, S: int, stride: int, coords: torch.Tensor, vis: torch.Tensor, conf: torch.Tensor,
                      threshold: float = 0.6):
    """ct3_online_window_end: the loop's coords [S,N,2] / vis / conf [S,N] of one pass into the streams' histories,
    and each entry's predictor output where it has one (see `online_stream`)."""
    for t, name in ((coords, "coords"), (vis, "vis"), (conf, "conf")):
        _req(t, torch.float32, name)
    N = vis.shape[1]
    dev = coords.device
    if tuple(coords.shape) != (S, N, 2) or tuple(vis.shape) != (S, N) or tuple(conf.shape) != (S, N):
        raise EngineError(f"coords, vis, conf must be [{S},N,2], [{S},N], [{S},N]")
    table, ws = _online_table(streams, dev)
    _call("ct3_online_window_end", dev, table, len(streams), int(S), int(stride), _ptr(coords), _ptr(vis), _ptr(conf),
          N, float(threshold), _ptr(ws), ws.numel(), _stream(dev))


def render_prepare(src: torch.Tensor, pad: int, grayscale: bool) -> torch.Tensor:
    """src [T,3,H,W] uint8 or float32 CUDA tensor, any strides -> [T,H+2p,W+2p,3] uint8: the visualiser's pad with
    255, optional Grayscale (repeated to 3 channels) and .byte(), bit-identical to the reference's CPU ops."""
    if not src.is_cuda:
        raise EngineError("src must be a CUDA tensor (no CPU fallback)")
    if src.dtype not in FRAME_DTYPES:
        raise EngineError(f"src must be uint8 or float32, got {src.dtype}")
    if src.dim() != 4 or src.shape[1] != 3:
        raise EngineError(f"src must be [T,3,H,W], got {tuple(src.shape)}")
    T, _, H, W = src.shape
    p = int(pad)
    out = torch.empty(T, H + 2 * p, W + 2 * p, 3, dtype=torch.uint8, device=src.device)
    _call("ct3_render_prepare", src.device, _ptr(src), FRAME_DTYPES[src.dtype], T, H, W, *src.stride(), p,
          int(bool(grayscale)), _ptr(out), _stream(src.device))
    return out


def render_workspace_bytes(T: int, H: int, W: int, N: int, trail: int) -> int:
    return _size("ct3_render_workspace_bytes", T, H, W, N, trail)


def render_tracks(frames: torch.Tensor, pts: torch.Tensor, colors: torch.Tensor, radius: int, linewidth: int,
                  trail: int = 0, query_frame: int = 0, visible: Optional[torch.Tensor] = None,
                  draw_mask: Optional[torch.Tensor] = None, alphas: Optional[torch.Tensor] = None,
                  diff: Optional[torch.Tensor] = None, workspace: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Draw trails and points in place on frames [T,H,W,3] uint8 (see ct3_render_tracks in include/ct3_b200.h).
    pts [T,N,2] fp32, colors [T,N,3] uint8, visible [T,N] uint8, draw_mask [N] uint8, alphas [T,S,2] / diff [T,S+1,2]
    fp64; all on the frames' device.  Returns frames."""
    _req(frames, torch.uint8, "frames")
    if frames.dim() != 4 or frames.shape[3] != 3:
        raise EngineError(f"frames must be [T,H,W,3], got {tuple(frames.shape)}")
    T, H, W, _ = frames.shape
    dev = frames.device
    N = pts.shape[1] if pts.dim() == 3 else -1
    want = {"pts": (pts, torch.float32, (T, N, 2)), "colors": (colors, torch.uint8, (T, N, 3)),
            "visible": (visible, torch.uint8, (T, N)), "draw_mask": (draw_mask, torch.uint8, (N,)),
            "alphas": (alphas, torch.float64, None), "diff": (diff, torch.float64, None)}
    for name, (t, dtype, shape) in want.items():
        if t is None:
            continue
        _req(t, dtype, name)
        if t.device != dev or (shape is not None and tuple(t.shape) != shape):
            raise EngineError(f"{name} must be {shape} on {dev}, got {tuple(t.shape)} on {t.device}")
    nbytes = render_workspace_bytes(T, H, W, N, trail)
    if workspace is None:
        workspace = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    _call("ct3_render_tracks", dev, _ptr(frames), T, H, W, _ptr(pts), _ptr(visible), _ptr(colors), _ptr(draw_mask), N,
          int(radius), int(linewidth), int(trail), int(query_frame), _ptr(alphas), _ptr(diff), _ptr(workspace),
          workspace.numel(), _stream(dev))
    return frames


def render_flow_workspace_bytes(T: int, N: int) -> int:
    return _size("ct3_render_flow_workspace_bytes", T, N)


def render_flow_colors(pts: torch.Tensor, query_frame: int) -> torch.Tensor:
    """pts [T,N,2] fp32 CUDA tensor (the frame pixel coordinates render_tracks takes) -> [T,N,3] uint8 on its device:
    flow_vis.flow_to_color(pts.long() - pts[query_frame].long()), the colours of the visualiser's optical_flow mode
    (see ct3_render_flow_colors in include/ct3_b200.h for the atan2 tolerance)."""
    _req(pts, torch.float32, "pts")
    if pts.dim() != 3 or pts.shape[2] != 2:
        raise EngineError(f"pts must be [T,N,2], got {tuple(pts.shape)}")
    T, N, _ = pts.shape
    dev = pts.device
    workspace = torch.empty(render_flow_workspace_bytes(T, N), dtype=torch.uint8, device=dev)
    colors = torch.empty(T, N, 3, dtype=torch.uint8, device=dev)
    _call("ct3_render_flow_colors", dev, _ptr(pts), T, N, int(query_frame), _ptr(colors), _ptr(workspace),
          workspace.numel(), _stream(dev))
    return colors


def pyramid_levels(pyr: torch.Tensor, T: int, H4: int, W4: int) -> List[torch.Tensor]:
    """Views [T,Hl,Wl,128] into the flat pyramid (tests / debugging)."""
    off, h, w, _ = pyramid_layout(T, H4, W4)
    return [pyr[off[l]: off[l] + T * h[l] * w[l] * LATENT].view(T, h[l], w[l], LATENT) for l in range(LEVELS)]


def sample_support(pyr, T, H4, W4, qframes, qcoords, support=None, accumulate_mask=None) -> torch.Tensor:
    _req(pyr, torch.float32, "pyr")
    _req(qframes, torch.int32, "queried_frames")
    _req(qcoords, torch.float32, "queried_coords")
    N = qframes.shape[0]
    if support is None:
        support = torch.zeros(LEVELS, P, N, LATENT, dtype=torch.float32, device=pyr.device)
    _req(support, torch.float32, "support")
    if accumulate_mask is not None:
        _req(accumulate_mask, torch.uint8, "accumulate_mask")
    _call("ct3_sample_support", pyr.device, _ptr(pyr), T, H4, W4, _ptr(qframes), _ptr(qcoords), N, _ptr(accumulate_mask),
          _ptr(support), _stream(pyr.device))
    return support


def _loop_shape(T, N, H4, W4, G=1, sizes=None, T_pyr=None, frames=None, slab_tracks=None, lengths=None) -> LoopShape:
    """ct3_loop_shape of a pass; None = the field's default (no map, no slabs, every group of length T)."""
    return LoopShape(int(T), int(N), int(H4), int(W4), int(G), sizes, int(T_pyr or 0), frames, int(slab_tracks or 0),
                     lengths)


def workspace_bytes(T: int, N: int, H4: int = 0, W4: int = 0, groups: int = 1, frames: Optional[int] = None,
                    slab_tracks: Optional[int] = None, group_T: Optional[Sequence[int]] = None) -> int:
    """Scratch of ct3_update_loop for T frames of H4 x W4 feature maps and N tracks (H4 = W4 = 0: updateformer only),
    split into `groups` track groups.  frames: the T_pyr pyramid frames of a pass with a frame map.  slab_tracks: the
    loop in track slabs of that many tracks.  group_T: the `groups` group lengths of a pass whose groups differ in
    length (ct3_loop_shape.group_T)."""
    lengths = None
    if group_T is not None:
        lengths, n_len = _group_array(group_T)
        if n_len != groups:
            raise EngineError(f"group_T has {n_len} entries for {groups} groups")
    shape = _loop_shape(T, N, H4, W4, groups, None, frames, None, slab_tracks, lengths)
    return _size("ct3_workspace_bytes", ctypes.byref(shape))


def pyramid_frames(pyr: torch.Tensor, H4: int, W4: int) -> int:
    """Number of frames of a flat pyramid (its size is linear in the frame count)."""
    per = pyramid_layout(1, H4, W4)[3]
    if pyr.numel() % per or pyr.numel() == 0:
        raise EngineError(f"a pyramid of {pyr.numel()} floats is not a whole number of {H4}x{W4} frames")
    return pyr.numel() // per


def _group_array(group_sizes):
    """Host int32 array of the group sizes (ct3_loop_shape.group_sizes); the library validates the values."""
    try:
        sizes = [int(g) for g in group_sizes]
    except (TypeError, ValueError) as e:
        raise EngineError(f"group_sizes must be a sequence of integers: {e}") from e
    if any(not (-2 ** 31 <= g < 2 ** 31) for g in sizes):
        raise EngineError("group sizes must fit in int32")
    return (ctypes.c_int32 * max(1, len(sizes)))(*sizes), len(sizes)


class WorkspaceCache:
    """Caller-owned scratch, grown on demand (the library never allocates)."""

    def __init__(self):
        self.buf: Optional[torch.Tensor] = None

    def get(self, T: int, N: int, device, H4: int = 0, W4: int = 0, groups: int = 1,
            frames: Optional[int] = None, slab_tracks: Optional[int] = None,
            group_T: Optional[Sequence[int]] = None) -> torch.Tensor:
        need = workspace_bytes(T, N, H4, W4, groups, frames, slab_tracks, group_T)
        if self.buf is None or self.buf.numel() < need or self.buf.device != torch.device(device):
            self.buf = None
            self.buf = torch.empty(need, dtype=torch.uint8, device=device)
        return self.buf


def _frame_array(group_frames, G: int, T: int):
    """Host int32 array [G*T] of a frame map given as a [G, T] nested sequence, array or tensor."""
    try:
        fr = torch.as_tensor(group_frames, dtype=torch.int64, device="cpu")
    except (TypeError, ValueError, RuntimeError) as e:
        raise EngineError(f"group_frames must be a [G, T] table of integers: {e}") from e
    if tuple(fr.shape) != (G, T):
        raise EngineError(f"group_frames must be [{G}, {T}], got {tuple(fr.shape)}")
    if fr.numel() and (int(fr.min()) < -2 ** 31 or int(fr.max()) >= 2 ** 31):
        raise EngineError("frame indices must fit in int32")
    return (ctypes.c_int32 * max(1, fr.numel()))(*fr.reshape(-1).tolist())


def update_loop(packed, pyr, H4, W4, support, track_valid, coords, vis, conf, time_emb, iters, workspace,
                group_sizes: Optional[Sequence[int]] = None, group_frames=None, slab_tracks: Optional[int] = None,
                group_T: Optional[Sequence[int]] = None):
    """In-place refinement of coords [T,N,2], vis [T,N], conf [T,N] (fp32, feature-grid units / logits).
    One ct3_update_loop call with the ct3_loop_shape the arguments describe.
    group_sizes: the N tracks as contiguous independent groups; each group's result is bit-identical to a call on its
    tracks alone.  None = one group.
    group_frames: [G, T] frame map: group g reads frame group_frames[g][t] of `pyr` (which may hold any number of
    frames) at time step t; each group's result is bit-identical to a call on a pyramid of exactly those frames.
    None = frame t.
    slab_tracks: run in track slabs of that many tracks in a workspace of workspace_bytes(..., slab_tracks=);
    bit-identical to the call without.  None = no slabs.
    group_T: G group lengths in [1, T]: group g tracks a clip of group_T[g] frames padded to T, and its rows t < group_T[g]
    are bit-identical to a call on its tracks alone with T = group_T[g]; time_emb is then [G, T, 1110], group g's time
    embedding in rows [0, group_T[g]).  None = every group has length T."""
    _req(coords, torch.float32, "coords"); _req(vis, torch.float32, "vis"); _req(conf, torch.float32, "conf")
    _req(pyr, torch.float32, "pyr"); _req(support, torch.float32, "support"); _req(time_emb, torch.float32, "time_emb")
    T, N, _ = coords.shape
    arr, G = _group_array(group_sizes if group_sizes is not None else [N])
    lengths = None
    if group_T is not None:
        lengths, n_len = _group_array(group_T)
        if n_len != G:
            raise EngineError(f"group_T has {n_len} entries for {G} groups")
    want = (T, XDIM) if group_T is None else (G, T, XDIM)
    if tuple(time_emb.shape) != want:
        raise EngineError(f"time_emb must be [{','.join(map(str, want))}]")
    if track_valid is not None:
        _req(track_valid, torch.uint8, "track_valid")
    if group_frames is None:
        T_pyr, fr = None, None
    else:
        T_pyr, fr = pyramid_frames(pyr, H4, W4), _frame_array(group_frames, G, T)
    shape = _loop_shape(T, N, H4, W4, G, arr, T_pyr, fr, slab_tracks, lengths)
    _call("ct3_update_loop", coords.device, _ptr(packed), _ptr(pyr), _ptr(support), _ptr(track_valid), _ptr(coords),
          _ptr(vis), _ptr(conf), _ptr(time_emb), int(iters), ctypes.byref(shape), _ptr(workspace), workspace.numel(),
          _stream(coords.device))


# ---- stage-level wrappers (tests, profiles) -----------------------------------------------------------
def corr_sample(pyr, H4, W4, support, track_valid, coords, scratch: bool = True) -> torch.Tensor:
    """-> fp32 correlation volume [N, T, 4, 2401] reconstructed from the split-bf16 device layout.
    scratch=False withholds the split-pyramid scratch, i.e. selects the sample-then-correlate kernel."""
    T, N, _ = coords.shape
    vol = torch.zeros(N * T * LEVELS, 2 * VOL_PAD, dtype=torch.bfloat16, device=coords.device)
    scr = torch.empty(pyr.numel() * 4, dtype=torch.uint8, device=coords.device) if scratch else None
    _call("ct3_corr_sample", coords.device, _ptr(pyr), H4, W4, _ptr(support), _ptr(track_valid), _ptr(coords), T, N,
          _ptr(vol), _ptr(scr), scr.numel() if scratch else 0, _stream(coords.device))
    return volume_planes(vol, T, N, H4, W4, scratch).sum(0).reshape(N, T, LEVELS, VOL)


def volume_planes(vol: torch.Tensor, T: int, N: int, H4: int, W4: int, patch: bool = True) -> torch.Tensor:
    """Decode a correlation volume in the device layout of ct3_corr_sample / ct3_loop_tokens (`vol`: the bytes as a
    [N*T*4, 2*2432] 16-bit tensor) -> fp32 [planes, N*T*4, 2401] in the reference's element order, planes = (hi, lo) of
    the split bf16 volume or the one fp16 plane; their sum is the volume.  patch: the split pyramid was available, so
    the correlate-then-interpolate kernels could run and this thread's options decide the format and element order."""
    rows = N * T * LEVELS
    # a single fp16 plane [rows, 2432] when the correlate-then-interpolate kernel runs with prec.fc1 < 3
    vb = precision_info(T, H4, W4)[2] if (patch and get_option("corr") == 0) else 4
    if vb == 2:
        planes = vol.reshape(-1).view(torch.float16)[:rows * VOL_PAD].reshape(1, rows, VOL_PAD).float()
    else:
        planes = vol.reshape(rows, 2, VOL_PAD).transpose(0, 1).float()
    assert bool((planes[:, :, VOL:] == 0).all()), "K padding of the correlation volume must be zero"
    planes = planes[:, :, :VOL]
    flag = ctypes.c_int(0)
    _check(lib().ct3_volume_is_support_major(T, H4, W4, ctypes.byref(flag)), "ct3_volume_is_support_major")
    if patch and flag.value:   # corr_tc3.cu: rows are [k][a*7+b]; hand back the reference order [(a*7+b)][k]
        planes = planes.reshape(len(planes), rows, P, P).transpose(2, 3).reshape(len(planes), rows, VOL)
    return planes


def x_src_col(dst: int) -> int:
    """Reference column of device X column `dst` (x_src_col in csrc/common.cuh): the correlation embeddings first, then
    vis, conf, posenc and zero padding; -1 = padding."""
    if dst < 1024:
        return dst + 2
    if dst in (1024, 1025):
        return dst - 1024
    return dst if dst < XDIM else -1


def x_planes(xs: torch.Tensor) -> torch.Tensor:
    """Split X rows [R, 2*1152] (bf16 hi | lo, device column order) -> fp32 [2, R, 1110] in the reference's column
    order; their sum is X."""
    dst = [c for c in range(XDIM_PAD) if x_src_col(c) >= 0]
    src = torch.tensor([x_src_col(c) for c in dst], device=xs.device)
    planes = xs.reshape(-1, 2, XDIM_PAD).transpose(0, 1).float()
    out = torch.empty(2, planes.shape[1], XDIM, dtype=torch.float32, device=xs.device)
    out[:, :, src] = planes[:, :, dst]
    return out


def loop_tokens(packed, pyr, H4, W4, support, track_valid, coords, vis, conf, time_emb, workspace=None,
                raw: bool = False):
    """ct3_loop_tokens: the first half of one update-loop iteration, from the state (read only) to the point tokens,
    under this thread's options -> fp32 (volume [N,T,4,2401] in reference order, X [N,T,1110] = hi + lo in reference
    column order without the time embedding, tokens [N,T,384]).  raw=True returns the device buffers instead: the
    volume bytes as [N*T*4, 2*2432] bf16 (volume_planes decodes them), X [N*T, 2*1152] bf16 (x_planes), tokens
    [N*T, 384]."""
    for t, name in ((coords, "coords"), (vis, "vis"), (conf, "conf"), (pyr, "pyr"), (support, "support"),
                    (time_emb, "time_emb")):
        _req(t, torch.float32, name)
    T, N, _ = coords.shape
    if time_emb.shape != (T, XDIM):
        raise EngineError(f"time_emb must be [{T},{XDIM}]")
    if track_valid is not None:
        _req(track_valid, torch.uint8, "track_valid")
    dev = coords.device
    if workspace is None:
        workspace = torch.empty(workspace_bytes(T, N, H4, W4), dtype=torch.uint8, device=dev)
    vol = torch.zeros(N * T * LEVELS, 2 * VOL_PAD, dtype=torch.bfloat16, device=dev)
    xs = torch.empty(N * T, 2 * XDIM_PAD, dtype=torch.bfloat16, device=dev)
    tokens = torch.empty(N * T, HID, dtype=torch.float32, device=dev)
    _call("ct3_loop_tokens", dev, _ptr(packed), _ptr(pyr), H4, W4, _ptr(support), _ptr(track_valid), _ptr(coords),
          _ptr(vis), _ptr(conf), _ptr(time_emb), T, N, _ptr(vol), _ptr(xs), _ptr(tokens), _ptr(workspace),
          workspace.numel(), _stream(dev))
    if raw:
        return vol, xs, tokens
    return (volume_planes(vol, T, N, H4, W4).sum(0).reshape(N, T, LEVELS, VOL),
            x_planes(xs).sum(0).reshape(N, T, XDIM), tokens.reshape(N, T, HID))


def split_rows(x: torch.Tensor, Kpad: int, fp16: bool = False) -> torch.Tensor:
    _req(x, torch.float32, "x")
    rows, K = x.shape
    out = torch.empty(rows, 2 * Kpad, dtype=torch.bfloat16, device=x.device)   # 16-bit planes (bf16 or fp16 bits)
    _call("ct3_split_rows_fp16" if fp16 else "ct3_split_rows", x.device, _ptr(x), rows, K, Kpad, _ptr(out),
          _stream(x.device))
    return out


def linear(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], act: int = 0, products: int = 3,
           fp16: bool = False) -> torch.Tensor:
    """Y = act(x w^T + b) through the wgmma GEMM engine; x [M,K], w [Nout,K] fp32.  products / fp16: the
    precision switches (3 = split x split, 2 = x_hi x split w, 1 = x_hi x w_hi; bf16 or fp16 planes)."""
    M, K = x.shape
    Nout = w.shape[0]
    Kpad = (K + 63) // 64 * 64
    xs, ws = split_rows(x.contiguous(), Kpad, fp16), split_rows(w.contiguous(), Kpad, fp16)
    y = torch.empty(M, Nout, dtype=torch.float32, device=x.device)
    _call("ct3_linear_prec", x.device, _ptr(xs), _ptr(ws), _ptr(bias), M, Nout, Kpad, act, products, 1 if fp16 else 0,
          _ptr(y), _stream(x.device))
    return y


def _req16(t: torch.Tensor, name: str, dev):
    """a contiguous 16-bit CUDA tensor on dev (split planes: bf16 or fp16 bits)"""
    if not t.is_cuda or t.device != torch.device(dev) or t.element_size() != 2 or not t.is_contiguous():
        raise EngineError(f"{name} must be a contiguous 16-bit tensor on {dev}")
    return t


def linear_ex(x_split: torch.Tensor, w_split: torch.Tensor, bias: Optional[torch.Tensor], M: int, Nout: int, Kpad: int,
              *, x_ld: int = 0, products: int = 3, fp16: bool = False, act: int = 0,
              row_bias: Optional[torch.Tensor] = None, row_mod: int = 1, y: Optional[torch.Tensor] = None,
              ld_y: int = 0, residual: bool = False, y_split: Optional[torch.Tensor] = None, ld_split: int = 0,
              lo_off: int = 0, row_group: int = 1):
    """ct3_linear_ex (include/ct3_b200.h): the GEMM engine with its whole epilogue, written in place into the caller's
    y (fp32) and / or y_split (16-bit).  Every buffer is flat or shaped as the caller likes; each must hold the elements
    the pitches address, which is checked here (the library can only check the pitches)."""
    dev = x_split.device
    _req16(x_split, "x_split", dev)
    _req16(w_split, "w_split", dev)
    xl = int(x_ld) if x_ld else 2 * int(Kpad)
    need = {"x_split": (x_split, (M - 1) * xl + (2 if products == 3 else 1) * Kpad), "w_split": (w_split, Nout * 2 * Kpad)}
    for name, t, n in (("bias", bias, Nout), ("row_bias", row_bias, max(row_mod, 1) * Nout)):
        if t is not None:
            _req(t, torch.float32, name)
            need[name] = (t, n)
    if y is not None:
        _req(y, torch.float32, "y")
        need["y"] = (y, (M - 1) * ld_y + Nout)
    if y_split is not None:
        _req16(y_split, "y_split", dev)
        need["y_split"] = (y_split, ((M + row_group - 1) // max(row_group, 1) - 1) * ld_split + lo_off + row_group * Nout)
    for name, (t, n) in need.items():
        if t.device != dev or t.numel() < n:
            raise EngineError(f"{name} must hold at least {n} elements on {dev}, has {t.numel()} on {t.device}")
    _call("ct3_linear_ex", dev, _ptr(x_split), int(x_ld), _ptr(w_split), _ptr(bias), int(M), int(Nout), int(Kpad),
          int(products), 1 if fp16 else 0, int(act), _ptr(row_bias), int(row_mod), _ptr(y), int(ld_y), 1 if residual else 0,
          _ptr(y_split), int(ld_split), int(lo_off), int(row_group), _stream(dev))


def layernorm(x: torch.Tensor, gamma: Optional[torch.Tensor] = None, beta: Optional[torch.Tensor] = None,
              eps: float = 1e-6) -> torch.Tensor:
    """ct3_layernorm: x [rows, 384] fp32 -> split bf16 rows [rows, 768] (hi | lo) of LayerNorm(x) with the optional
    affine gamma / beta [384], the kernel the transformer body runs."""
    _req(x, torch.float32, "x")
    if x.dim() != 2 or x.shape[1] != HID:
        raise EngineError(f"x must be [rows, {HID}], got {tuple(x.shape)}")
    for name, t in (("gamma", gamma), ("beta", beta)):
        if t is not None and (_req(t, torch.float32, name).numel() != HID or t.device != x.device):
            raise EngineError(f"{name} must be [{HID}] on {x.device}")
    out = torch.empty(x.shape[0], 2 * HID, dtype=torch.bfloat16, device=x.device)
    _call("ct3_layernorm", x.device, _ptr(x), x.shape[0], _ptr(gamma), _ptr(beta), float(eps), _ptr(out),
          _stream(x.device))
    return out


def time_block_attention(packed, depth: int, x_split: torch.Tensor, T: int,
                         out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """ct3_time_block_attention: q|k|v projection and per-track attention of time block `depth` on the LayerNorm
    output x_split [rows, 768] (split bf16, rows n*T + t), routed as the transformer body routes it under this thread's
    options -> split bf16 [rows, 768].  out: a 16-bit buffer of at least rows rows of 768 to write into (rows beyond
    are left as they are)."""
    dev = x_split.device
    _req16(x_split, "x_split", dev)
    rows = x_split.shape[0]
    if x_split.dim() != 2 or x_split.shape[1] != 2 * HID:
        raise EngineError(f"x_split must be [rows, {2 * HID}], got {tuple(x_split.shape)}")
    if out is None:
        out = torch.empty(rows, 2 * HID, dtype=torch.bfloat16, device=dev)
    _req16(out, "out", dev)
    if out.numel() < rows * 2 * HID:
        raise EngineError(f"out must hold {rows} rows of {2 * HID}")
    workspace = torch.empty(_size("ct3_time_block_attention_workspace_bytes", int(T), rows), dtype=torch.uint8, device=dev)
    _call("ct3_time_block_attention", dev, _ptr(packed), int(depth), _ptr(x_split), int(T), rows, _ptr(out),
          _ptr(workspace), workspace.numel(), _stream(dev))
    return out


def updateformer(packed, x: torch.Tensor, workspace: Optional[torch.Tensor] = None,
                 group_sizes: Optional[Sequence[int]] = None) -> torch.Tensor:
    """x [N,T,1110] fp32 (reference column order, time embedding added) -> delta [N,T,4].
    group_sizes: contiguous independent track groups, None = one group."""
    _req(x, torch.float32, "x")
    N, T, D = x.shape
    if D != XDIM:
        raise EngineError("x must be [N,T,1110]")
    delta = torch.empty(N, T, 4, dtype=torch.float32, device=x.device)
    arr, G = _group_array(group_sizes) if group_sizes is not None else (None, 1)
    if workspace is None:
        workspace = torch.empty(workspace_bytes(T, N, groups=G), dtype=torch.uint8, device=x.device)
    _call("ct3_updateformer", x.device, _ptr(packed), _ptr(x), T, N, arr, G, _ptr(delta), _ptr(workspace),
          workspace.numel(), _stream(x.device))
    return delta


# ct3_attention kinds (CT3_ATTN_*) and the column widths of their q and kv rows
ATTENTION_KINDS = {"time": 0, "virtual_from_point": 1, "virtual_self": 2, "point_from_virtual": 3}
_ATTENTION_WIDTHS = {0: (3 * HID, 3 * HID), 1: (HID, 2 * HID), 2: (3 * HID, 3 * HID), 3: (HID, 2 * HID)}


def attention(kind, q: torch.Tensor, kv: torch.Tensor, T: int, N: int,
              group_sizes: Optional[Sequence[int]] = None) -> torch.Tensor:
    """One attention core of the transformer body (ct3_attention in include/ct3_b200.h), dispatched as the body does
    under this thread's "attn" option.  kind: a name of ATTENTION_KINDS or its number.  q, kv: fp32 token rows
    [(N + 64 G) * T, width] (time / virtual_self: q|k|v rows of 1152, possibly the same tensor; the cross kinds: q rows
    of 384 and k|v rows of 768).  -> fp32 [(N + 64 G) * T, 384] = hi + lo of the split output; rows the kind does not
    write are 0."""
    k = ATTENTION_KINDS[kind] if isinstance(kind, str) else int(kind)
    _req(q, torch.float32, "q")
    _req(kv, torch.float32, "kv")
    arr, G = _group_array(group_sizes if group_sizes is not None else [N])
    rows = (int(N) + VIRT * G) * int(T)
    wq, wkv = _ATTENTION_WIDTHS.get(k, (q.shape[-1], kv.shape[-1]))
    if tuple(q.shape) != (rows, wq) or tuple(kv.shape) != (rows, wkv) or kv.device != q.device:
        raise EngineError(f"attention kind {kind}: q must be [{rows},{wq}] and kv [{rows},{wkv}] on one device, "
                          f"got {tuple(q.shape)} and {tuple(kv.shape)}")
    dev = q.device
    out = torch.zeros(rows, 2 * HID, dtype=torch.bfloat16, device=dev)
    workspace = torch.empty(_size("ct3_attention_workspace_bytes", int(T), int(N), G), dtype=torch.uint8, device=dev)
    _call("ct3_attention", dev, k, _ptr(q), _ptr(kv), int(T), int(N), arr, G, _ptr(out), _ptr(workspace),
          workspace.numel(), _stream(dev))
    return out[:, :HID].float() + out[:, HID:].float()


PROFILE_CATEGORIES = ["corr_sample", "gemm", "attention", "layernorm", "misc", "encoder", "qkv_time_attention"]


def profile_enable(on: bool):
    _check(lib().ct3_profile_enable(1 if on else 0), "ct3_profile_enable")


def profile_read():
    """-> ({category: ms}, {category: launches}, gemm_flops) accumulated since profile_enable(True)."""
    ms = (ctypes.c_double * len(PROFILE_CATEGORIES))()
    n = (ctypes.c_int * len(PROFILE_CATEGORIES))()
    fl = ctypes.c_double(0)
    _check(lib().ct3_profile_read(ms, n, ctypes.byref(fl)), "ct3_profile_read")
    return dict(zip(PROFILE_CATEGORIES, list(ms))), dict(zip(PROFILE_CATEGORIES, list(n))), fl.value


# ---- encoder tail -------------------------------------------------------------------------------------
def enc_tail_pack(conv2_w, conv2_b, conv3_w, conv3_b, device) -> torch.Tensor:
    n = _size("ct3_enc_tail_packed_bytes")
    ts = [x.detach().to(device=device, dtype=torch.float32).contiguous() for x in (conv2_w, conv2_b, conv3_w, conv3_b)]
    packed = torch.empty(n, dtype=torch.uint8, device=device)
    _call("ct3_enc_tail_pack", device, *[_ptr(t) for t in ts], _ptr(packed), n, _stream(device))
    torch.cuda.current_stream(device).synchronize()
    return packed


def enc_tail_workspace_bytes(T: int, H4: int, W4: int) -> int:
    return _size("ct3_enc_tail_workspace_bytes", T, H4, W4)


def enc_tail(packed, cat: torch.Tensor, workspace: torch.Tensor) -> torch.Tensor:
    """cat [T,416,H4,W4] fp32 -> flat channels-last normalised pyramid (same layout as prepare_pyramid)."""
    _req(cat, torch.float32, "cat")
    T, C, H4, W4 = cat.shape
    if C != 416:
        raise EngineError("cat must have 416 channels")
    *_, total = pyramid_layout(T, H4, W4)
    pyr = torch.empty(total, dtype=torch.float32, device=cat.device)
    _call("ct3_enc_tail", cat.device, _ptr(packed), _ptr(cat), T, H4, W4, _ptr(pyr), _ptr(workspace), workspace.numel(),
          _stream(cat.device))
    return pyr


# ---- whole encoder (enc_front.cu + GEMM engine) -----------------------------------------------------------
def encoder_weight_names() -> List[str]:
    L = lib()
    return [L.ct3_encoder_weight_name(i).decode() for i in range(L.ct3_encoder_num_weight_tensors())]


def encoder_pack(state: dict, device) -> torch.Tensor:
    """state: mapping `fnet` state-dict key (without the `fnet.` prefix) -> tensor; returns the packed device buffer."""
    names = encoder_weight_names()
    ts = [state[k].detach().to(device=device, dtype=torch.float32).contiguous() for k in names]
    n = _size("ct3_encoder_packed_bytes")
    packed = torch.empty(n, dtype=torch.uint8, device=device)
    ptrs = (ctypes.c_void_p * len(ts))(*[t.data_ptr() for t in ts])
    _call("ct3_encoder_pack", device, ptrs, len(ts), _ptr(packed), n, _stream(device))
    torch.cuda.current_stream(device).synchronize()   # `ts` may be temporaries
    return packed


def encoder_workspace_bytes(T: int, H: int, W: int) -> int:
    return _size("ct3_encoder_workspace_bytes", T, H, W)


def encoder(packed: torch.Tensor, frames: torch.Tensor, workspace: torch.Tensor) -> torch.Tensor:
    """frames [T,3,H,W] fp32 in [-1,1] -> flat channels-last L2-normalised 4-level pyramid (stride 4)."""
    _req(frames, torch.float32, "frames")
    T, C, H, W = frames.shape
    if C != 3:
        raise EngineError("frames must be [T,3,H,W]")
    *_, total = pyramid_layout(T, H // 4, W // 4)
    pyr = torch.empty(total, dtype=torch.float32, device=frames.device)
    _call("ct3_encoder", frames.device, _ptr(packed), _ptr(frames), T, H, W, _ptr(pyr), _ptr(workspace), workspace.numel(),
          _stream(frames.device))
    return pyr


def slice_pyramid(pyr: torch.Tensor, T: int, H4: int, W4: int, t0: int, S: int) -> torch.Tensor:
    """Frames [t0, t0+S) of every level as a new flat pyramid (sliding-window mode)."""
    off, h, w, _ = pyramid_layout(T, H4, W4)
    parts = []
    for l in range(LEVELS):
        per = h[l] * w[l] * LATENT
        parts.append(pyr[off[l] + t0 * per: off[l] + (t0 + S) * per])
    return torch.cat(parts)


def reverse_pyramid_(pyr: torch.Tensor, T: int, H4: int, W4: int, pad: int = 0, block: int = 4) -> torch.Tensor:
    """In place: turn the flat pyramid of a clip's T frames plus `pad` copies of frame T-1 into the pyramid of the clip
    played backwards, frames T-1 .. 0 plus `pad` copies of (original) frame 0.  The encoder is strictly per frame, so
    this is the pyramid of the reversed, likewise padded clip, without encoding it again.  Applying it twice restores
    the original bit for bit.  Frames are swapped `block` mirrored pairs at a time, so the scratch is at most 3 * block
    frames of level 0, never a second pyramid."""
    for lv in pyramid_levels(pyr, T + pad, H4, W4):
        half = T // 2
        for i in range(0, half, block):
            m = min(block, half - i)
            a, b = lv[i:i + m], lv[T - i - m:T - i]      # disjoint: i + m <= T // 2 <= T - i - m
            tmp = a.clone()
            a.copy_(b.flip(0))
            b.copy_(tmp.flip(0))
        if pad > 0:
            lv[T:].copy_(lv[T - 1:T].expand(pad, -1, -1, -1))
    return pyr


def concat_pyramid_runs(runs, H4: int, W4: int) -> torch.Tensor:
    """Flat pyramid of the frame runs (pyr, T, a, b) = frames [a, b) of the T-frame flat pyramid `pyr`, concatenated in
    order: one copy, whatever the number of runs and source pyramids."""
    parts = []
    layouts = {}
    for l in range(LEVELS):
        for pyr, T, a, b in runs:
            if T not in layouts:
                layouts[T] = pyramid_layout(T, H4, W4)
            off, h, w, _ = layouts[T]
            per = h[l] * w[l] * LATENT
            parts.append(pyr[off[l] + a * per: off[l] + b * per])
    return torch.cat(parts)


def upsample_concat(feats: Sequence[torch.Tensor], H: int, W: int) -> torch.Tensor:
    """4 stage outputs [T,Cs,Hs,Ws] -> bilinear(align_corners=True) to HxW, concatenated on channels [T,sum Cs,H,W]."""
    if len(feats) != 4:
        raise EngineError("upsample_concat expects 4 stage tensors")
    fs = [_req(f, torch.float32, "stage feature") for f in feats]
    T = fs[0].shape[0]
    out = torch.empty(T, sum(f.shape[1] for f in fs), H, W, dtype=torch.float32, device=fs[0].device)
    src = (ctypes.c_void_p * 4)(*[f.data_ptr() for f in fs])
    ch = (ctypes.c_int * 4)(*[f.shape[1] for f in fs])
    hh = (ctypes.c_int * 4)(*[f.shape[2] for f in fs])
    ww = (ctypes.c_int * 4)(*[f.shape[3] for f in fs])
    _call("ct3_upsample_concat", out.device, src, ch, hh, ww, T, H, W, _ptr(out), _stream(out.device))
    return out
