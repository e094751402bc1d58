"""Independent online streams in one update-loop pass.

    hub = OnlineStreams(predictor)                  # a CoTrackerOnlinePredictor; the hub shares its model
    a = hub.open(frame_size=(720, 1280), grid_size=10)
    b = hub.open(frame_size=(480, 640), queries=q, add_support_grid=True)
    hub.push(a, chunk_a)                            # [1,T,3,H,W], T <= window_len, uint8 or float, host or device
    hub.push(b, chunk_b)
    out = hub.step()                                # {stream id: (tracks [1,T_so_far,N,2], visibility [1,T_so_far,N])}
    hub.close(a)
    c = hub.open(frame_size=(720, 1280), grid_size=10, history=64)   # bounded: results of the last 64 frames only

Each stream has its own frame size, queries, start and pace.  `step()` advances every stream with a pushed chunk by one
window: their chunks are resized into one frame batch, their new frames go through one encoder pass, and their tracks
run as query groups of one update loop (or of a few, when they do not fit in device memory at once).  For every stream,
the results of the steps that advanced it are bit-identical to a fresh predictor on the same model called with
`is_first_step=True` and the `open()` arguments, then with that stream's chunks in order and the same
`add_support_grid`; whatever the other streams do.

A stream opened with `history=h` runs in bounded memory: its history is a ring allocated once, each `step()` returns
its last L = min(h, frames so far) frames only, and a step's work does not grow with the stream's length.  Its result
is then exactly the last L frames of the unbounded result, `full[:, -L:]`; `length(sid)` gives the stream's frame
count, so the result covers frames [length - L, length).  A stream can advance until a window would pass frame
2^30 (about 414 days at 30 fps); `push()` reports that limit.

A stream's tracks can change between steps:

    hub.retire_tracks(c, [3, 7])                    # ids of track_ids(c); the support grid's points have none
    new = hub.add_tracks(c, q)                      # [1,m,3] (t, x, y), frame pixels, every t >= hub.length(c)
    hub.track_ids(c)                                # the columns of c's next results: open() gave 0..n-1, adds continue

An edit is the same edit of the reference online model's per-track state between two predictor calls, along its N
axis: retiring deletes the tracks' columns; adding inserts columns after the stream's own tracks (before its support
grid) with zero support features and, at every frame so far, the query point with vis and conf logits 0.  So at the
frames before the next window an added track reads as its query point, not visible, and the other tracks' frames
there are unchanged.  Edits take effect at the stream's next step and each call copies the track pool once.  A track
whose query frame lies ahead still takes part in the attention of the other tracks, so adding one mid-stream is not
the same as having opened the stream with it; before the first step it is, bit for bit.

A stream can be parked on the host and continued on any hub of the same model:

    snap = hub.snapshot(c)                          # CPU tensors and plain values; c runs on unchanged
    hub.close(c)                                    # frees c's device memory
    torch.save(snap, f)                             # loads with torch.load(f, weights_only=True)
    c2 = other_hub.restore(snap)                    # a new id on other_hub's device

From its next step on, a restored stream's results are `torch.equal` to those the snapshotted stream would have given
without the snapshot, fed the same chunks, whatever the other streams of either hub do.  This needs the same weights
and the same GPU model: some split-K choices depend on the SM count.  Restoring one snapshot twice gives two
independent streams.  A snapshot holds the stream's own state and nothing more: its columns of the pool (support
features, query frames and coordinates), its window start, length and bound, its history (the whole ring of a bounded
stream, frames [0, length) otherwise), its frame size, output width, track ids and next track id, the format version,
and the model's window_len, interp_shape, stride and weights fingerprint, which `restore` checks.  It leaves out the
encoder features of the overlap frames (67 MB at 384x512): the chunk after a restore holds those frames again, and
the first step encodes the stream's whole chunk, which gives the same features since the encoder is strictly per
frame.  `restore` validates everything it reads before it changes anything (`check_snapshot`).
"""
from __future__ import annotations

import numbers
from typing import Dict, List, Optional, Tuple

import torch

from . import engine, ingest
from .model import StreamPool, StreamState

SNAPSHOT_FORMAT = 1
_SNAPSHOT_FIELDS = ("model", "frame_size", "n_keep", "ids", "next_id", "n", "ind", "length", "history", "support",
                    "qframes", "qcoords", "hist")


def _is_int(x) -> bool:
    return isinstance(x, numbers.Integral) and not isinstance(x, bool)


def _check_tensor(name: str, t, dtype, shape):
    got = f"{t.dtype} {list(t.shape)}" if torch.is_tensor(t) else type(t).__name__
    if not torch.is_tensor(t) or t.dtype != dtype or tuple(t.shape) != tuple(shape):
        raise ValueError(f"snapshot field {name} must be a {dtype} tensor {list(shape)}, got {got}")


def check_snapshot(snap, identity: dict):
    """Raise ValueError unless `snap` is a stream state that `OnlineStreams.restore` can continue on a model of
    `identity` (`OnlineStreams.model_identity`): a known format, the same model, every field present with its type,
    dtype and shape, and a window start and length a stream can reach.  A snapshot comes from outside the program (a
    file), so everything is checked; this reads nothing but its arguments and needs no device."""
    if not isinstance(snap, dict):
        raise ValueError(f"a snapshot is a dict, got {type(snap).__name__}")
    fmt = snap.get("format")
    if not _is_int(fmt) or fmt != SNAPSHOT_FORMAT:
        raise ValueError(f"unknown snapshot format {fmt!r}: this version reads format {SNAPSHOT_FORMAT}")
    missing = [k for k in _SNAPSHOT_FIELDS if k not in snap]
    if missing:
        raise ValueError(f"the snapshot misses the fields {missing}")
    model = snap["model"]
    if not isinstance(model, dict):
        raise ValueError(f"snapshot field model must be a dict, got {type(model).__name__}")
    for k, v in identity.items():
        if model.get(k) != v:
            raise ValueError(f"the snapshot was taken on a model with {k} {model.get(k)!r}, this hub's has {v!r}")
    ints = {k: snap[k] for k in ("n_keep", "next_id", "n", "ind", "length")}
    for k, v in ints.items():
        if not _is_int(v):
            raise ValueError(f"snapshot field {k} must be an int, got {type(v).__name__}")
    hw, ids, history = snap["frame_size"], snap["ids"], snap["history"]
    if not isinstance(hw, (list, tuple)) or len(hw) != 2 or not all(_is_int(x) and x >= 2 for x in hw):
        raise ValueError(f"snapshot field frame_size must be [H, W] with H, W >= 2 ints, got {hw!r}")
    if history is not None and (not _is_int(history) or history < 1):
        raise ValueError(f"snapshot field history must be None or an int >= 1, got {history!r}")
    if not isinstance(ids, (list, tuple)) or not all(_is_int(i) for i in ids):
        raise ValueError("snapshot field ids must be a list of ints")
    n, n_keep, next_id, ind, length = (ints[k] for k in ("n", "n_keep", "next_id", "ind", "length"))
    if n < 1 or not 1 <= n_keep <= n:
        raise ValueError(f"a snapshot holds 1 <= n_keep <= n tracks, got n_keep {n_keep} of n {n}")
    if len(ids) != n_keep or len(set(ids)) != n_keep or any(not 0 <= i < next_id for i in ids):
        raise ValueError(f"snapshot field ids must be n_keep = {n_keep} distinct ids in [0, next_id = {next_id}), "
                         f"got {len(ids)} ids")
    _check_tensor("support", snap["support"], torch.float32, (4, 49, n, 128))
    _check_tensor("qframes", snap["qframes"], torch.int32, (n,))
    _check_tensor("qcoords", snap["qcoords"], torch.float32, (n, 2))
    if int(snap["qframes"].abs().max()) > engine.QUERY_FRAME_LIMIT:
        raise ValueError(f"snapshot field qframes holds query frames past +-{engine.QUERY_FRAME_LIMIT}")
    S = identity["window_len"]
    step = S // 2
    if ind < 0 or length < 0:
        raise ValueError(f"a stream's window start and length are >= 0, got ind {ind}, length {length}")
    # after k >= 1 windows of chunks of 1..S frames: ind = k * step, length = ind - step + T
    if ind % step or (length != 0 if ind == 0 else not ind - step + 1 <= length <= ind - step + S):
        raise ValueError(f"no stream reaches window start {ind} with length {length} (window_len {S})")
    if ind and ind - step + S > engine.STREAM_FRAME_LIMIT:
        raise ValueError(f"window start {ind} lies past the stream frame limit {engine.STREAM_FRAME_LIMIT}")
    hist = snap["hist"]
    if length == 0:
        if hist is not None:
            raise ValueError("a stream that has not advanced has no history: snapshot field hist must be None")
        return
    if not isinstance(hist, (list, tuple)) or len(hist) != 3 or not torch.is_tensor(hist[1]) or hist[1].dim() != 2:
        raise ValueError("snapshot field hist must be [coords [R,n,2], vis [R,n], conf [R,n]]")
    rows = hist[1].shape[0]
    cap = None if history is None else StreamState(n, 0, history).ring_frames(S, step)
    if history is not None and rows != cap:
        raise ValueError(f"a stream bounded at history={history} keeps a ring of {cap} frames, the snapshot "
                         f"holds {rows}")
    if history is None and rows < length:
        raise ValueError(f"the history of a stream of length {length} holds {length} frames, the snapshot {rows}")
    for name, t, shape in (("coords", hist[0], (rows, n, 2)), ("vis", hist[1], (rows, n)),
                           ("conf", hist[2], (rows, n))):
        _check_tensor(f"hist {name}", t, torch.float32, shape)


class OnlineStreams:
    def __init__(self, predictor):
        self.predictor = predictor
        self.model = predictor.model
        self.pool = StreamPool()
        self._streams: Dict[int, dict] = {}     # id -> the stream's state, open arguments and output shape
        self._pending: Dict[int, torch.Tensor] = {}
        self._next_id = 0

    @torch.no_grad()
    def open(self, frame_size: Tuple[int, int], queries: torch.Tensor = None, grid_size: int = 5,
             grid_query_frame: int = 0, add_support_grid: bool = False, history: Optional[int] = None) -> int:
        """Start a stream of frames of frame_size = (H, W): the arguments of the predictor's `is_first_step=True` call,
        with the frame size in place of the first chunk.  history: None keeps every frame and returns them all at each
        step; an int h >= 1 keeps the stream in fixed memory and returns its last min(h, frames so far) frames.
        -> the stream's id."""
        if history is not None and (isinstance(history, bool) or not isinstance(history, int) or history < 1):
            raise ValueError(f"history must be None or an int >= 1, got {history!r}")
        H, W = (int(x) for x in frame_size)
        if H < 2 or W < 2:
            raise ValueError(f"frame_size must be (H, W) with H, W >= 2, got {tuple(frame_size)}")
        if queries is None and grid_size <= 0:
            raise ValueError("open() needs queries or grid_size > 0")
        if queries is not None and (queries.dim() != 3 or queries.shape[0] != 1 or queries.shape[1] < 1
                                    or queries.shape[2] != 3):
            raise ValueError(f"queries must be [1,N,3] with N >= 1, got {tuple(queries.shape)}")
        dev = ingest.model_device(self.model)
        if dev.type != "cuda":
            raise ValueError("the predictor's model must be on a CUDA device")
        q, n_out = self.predictor._first_step_queries(1, (H, W), queries, grid_size, grid_query_frame,
                                                      add_support_grid, dev)
        state = self.pool.open(*self.model._stream_queries(q[0]), history=history)
        n_keep = n_out if add_support_grid else q.shape[1]
        return self._add(state, (H, W), n_keep, list(range(n_keep)), n_keep)

    def _add(self, state, hw, n_keep: int, ids: List[int], next_id: int) -> int:
        """Register a stream of the pool under a new id: its frame size, output width, track ids and next track id."""
        sid = self._next_id
        self._next_id += 1
        H, W = hw
        ih, iw = self.predictor.interp_shape
        self._streams[sid] = dict(state=state, hw=(H, W), out=(n_keep, ((W - 1) / (iw - 1), (H - 1) / (ih - 1))),
                                  ids=ids, next_id=next_id)
        return sid

    def _get(self, sid: int) -> dict:
        if sid not in self._streams:
            raise KeyError(f"no open stream {sid}")
        return self._streams[sid]

    def length(self, sid: int) -> int:
        """The frames stream `sid` has been advanced by so far: its last result covers frames [length - L, length),
        with L the result's frame count."""
        return self._get(sid)["state"].length

    def push(self, sid: int, chunk: torch.Tensor):
        """Queue the next chunk [1,T,3,H,W] of stream `sid` (T <= window_len) for the next `step()`."""
        s = self._get(sid)
        if sid in self._pending:
            raise ValueError(f"stream {sid} already has a chunk for this step")
        if chunk.dim() != 5 or chunk.shape[0] != 1 or chunk.shape[2] != 3 or tuple(chunk.shape[3:]) != s["hw"]:
            raise ValueError(f"stream {sid} takes chunks [1,T,3,{s['hw'][0]},{s['hw'][1]}], got {tuple(chunk.shape)}")
        err = self.model.stream_advance_error(s["state"], chunk.shape[1])
        if err:
            raise ValueError(f"stream {sid}: {err}")
        self._pending[sid] = chunk

    def close(self, sid: int):
        """End stream `sid`: its tracks leave the pool and its id is no longer valid."""
        s = self._get(sid)
        self._pending.pop(sid, None)
        self.pool.close(s["state"])
        del self._streams[sid]

    def model_identity(self) -> dict:
        """What a snapshot must have been taken on to be restored here: window_len, interp_shape, stride and the
        weights' fingerprint."""
        return dict(window_len=self.model.window_len, interp_shape=list(self.predictor.interp_shape),
                    stride=self.model.stride, weights=self.model.weights_fingerprint())

    def snapshot(self, sid: int) -> dict:
        """Stream `sid`'s state as CPU tensors and plain Python values (`torch.save` it, load it with
        `weights_only=True`); the stream runs on unchanged.  Taken between steps: a pushed chunk must be stepped first."""
        s = self._get(sid)
        if sid in self._pending:
            raise ValueError(f"stream {sid} has a chunk waiting for step(): take a snapshot between steps")
        return dict(self.pool.export(s["state"]), format=SNAPSHOT_FORMAT, model=self.model_identity(),
                    frame_size=list(s["hw"]), n_keep=s["out"][0], ids=list(s["ids"]), next_id=s["next_id"])

    @torch.no_grad()
    def restore(self, snap: dict) -> int:
        """Add the stream of `snapshot()`'s `snap` to this hub, on its device, as `open()` adds one.  From its next
        step on its results are `torch.equal` to those the snapshotted stream would have given, on the same model and
        device model.  Restoring one snapshot twice gives two independent streams.  -> the new stream's id."""
        check_snapshot(snap, self.model_identity())
        dev = ingest.model_device(self.model)
        if dev.type != "cuda":
            raise ValueError("the predictor's model must be on a CUDA device")
        state = self.pool.restore(snap, dev)
        return self._add(state, tuple(snap["frame_size"]), snap["n_keep"], list(snap["ids"]), snap["next_id"])

    def track_ids(self, sid: int) -> List[int]:
        """The ids of the tracks of stream `sid`'s results, in column order, from its next step on.  open() numbers
        its tracks 0..n-1 and each add_tracks() continues upward; a stream never reuses an id."""
        return list(self._get(sid)["ids"])

    @torch.no_grad()
    def add_tracks(self, sid: int, queries: torch.Tensor) -> List[int]:
        """Add the tracks of queries [1,m,3] (t, x, y) to stream `sid` from its next step on: frame pixels and stream
        time, as open() takes them.  Every t must be >= length(sid): a frame the stream has passed can no longer give
        a track its features.  The new tracks follow the others in the results (before the support grid).  At the
        frames before the next window they read as their query point, not visible.  -> their ids."""
        s = self._get(sid)
        if queries.dim() != 3 or queries.shape[0] != 1 or queries.shape[1] < 1 or queries.shape[2] != 3:
            raise ValueError(f"queries must be [1,m,3] with m >= 1, got {tuple(queries.shape)}")
        state = s["state"]
        t = queries[0, :, 0]
        if not bool((t >= state.length).all()):
            raise ValueError(f"stream {sid} has advanced {state.length} frames: query frames must be >= "
                             f"{state.length}, got {float(t.min())}")
        q, _ = self.predictor._first_step_queries(1, s["hw"], queries, 0, 0, False, ingest.model_device(self.model))
        n_keep, scale = s["out"]
        self.pool.edit(state, range(state.n), n_keep, *self.model._stream_queries(q[0]), self.model.stride)
        m = q.shape[1]
        ids = list(range(s["next_id"], s["next_id"] + m))
        s.update(ids=s["ids"] + ids, next_id=s["next_id"] + m, out=(n_keep + m, scale))
        return ids

    def retire_tracks(self, sid: int, ids):
        """Remove the tracks `ids` (ids of stream `sid`, see track_ids) from its next step on.  The support grid's
        points have no ids; a stream keeps at least one track of its own: close it instead."""
        s = self._get(sid)
        ids = ids.tolist() if torch.is_tensor(ids) else list(ids)
        col = {i: c for c, i in enumerate(s["ids"])}
        for i in ids:
            if isinstance(i, bool) or not isinstance(i, numbers.Integral) or i not in col:
                raise ValueError(f"stream {sid} has no track {i!r}: its track ids are track_ids({sid})")
        if len(set(ids)) != len(ids):
            raise ValueError(f"track ids to retire hold duplicates: {ids}")
        if len(ids) == len(col):
            raise ValueError(f"retiring every track of stream {sid} would leave it empty: close it instead")
        state = s["state"]
        gone = {col[i] for i in ids}
        n_keep, scale = s["out"]
        dev = self.pool.qframes.device
        self.pool.edit(state, [c for c in range(state.n) if c not in gone], n_keep - len(gone),
                       torch.empty(0, dtype=torch.int32, device=dev), torch.empty(0, 2, device=dev), self.model.stride)
        s.update(ids=[i for i in s["ids"] if col[i] not in gone], out=(n_keep - len(gone), scale))

    @torch.no_grad()
    def step(self) -> Dict[int, Tuple[torch.Tensor, torch.Tensor]]:
        """Advance every stream with a pushed chunk by one window, in one pass.  -> {id: (tracks [1,L,n,2] fp32,
        visibility [1,L,n] bool)} of the streams it advanced, for their frames [length - L, length) with L = length
        (frames so far), or min(h, length) for a stream opened with history=h; the others keep their state.
        Frames before length - (window_len - step) (step = window_len // 2) are final: the next window re-tracks the
        others."""
        order = {id(s): k for k, s in enumerate(self.pool.streams)}
        ids = sorted(self._pending, key=lambda i: order[id(self._streams[i]["state"])])
        if not ids:
            return {}
        S = self.model.window_len
        ih, iw = self.predictor.interp_shape
        dev = ingest.model_device(self.model)
        frames = torch.empty(len(ids) * S, 3, ih, iw, dtype=torch.float32, device=dev)
        Ts = []
        for k, sid in enumerate(ids):
            chunk = self._pending[sid]
            T = chunk.shape[1]
            ingest.prepare_video(chunk, (ih, iw), dev, out=frames[k * S:k * S + T])
            if T < S:   # the model pads a short chunk with copies of its last frame
                frames[k * S + T:(k + 1) * S] = frames[k * S + T - 1]
            Ts.append(T)
        self._pending.clear()
        states = [self._streams[i]["state"] for i in ids]
        outputs = [self._streams[i]["out"] if s.history is None else
                   (*self._streams[i]["out"], min(s.history, s.ind + T)) for i, s, T in zip(ids, states, Ts)]
        outs = self.model._stream_step(self.pool, states, frames, Ts, 6, outputs=outputs)
        return {sid: (tr[None], vi[None]) for sid, (tr, vi) in zip(ids, outs)}
