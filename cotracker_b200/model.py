"""CoTracker3 models whose iterative update loop runs in libct3_b200.so.

Drop-in mirror of the reference's inner model API (SURVEY.md §8b):
    CoTrackerThreeOffline.forward  -- reference cotracker3_offline.py:19-233
    CoTrackerThreeOnline.forward   -- reference cotracker3_online.py:266-541 (+ init_video_online_processing :163-169)
with the same constructor kwargs, attributes (`model_resolution`, `window_len`, `stride`) and the same
state-dict keys (SURVEY.md Appendix B), so `load_state_dict(strict=True)` of the released checkpoints works.

The nn.Module tree below is a *parameter container*: nothing executes through PyTorch modules.  The CNN
encoder, L2-normalisation + pyramid, support sampling, correlation sampling, the correlation MLP, the whole
EfficientUpdateFormer and the delta heads run as hand-written sm_90a CUDA behind the C ABI
(`cotracker_b200.engine`).  Inference only.  A batch of B clips (same length and size) is tracked in one pass: clip b's
queries are query groups of one update loop that read clip b's frames of one pyramid holding all B clips, and slot b of
the result is bit-identical to the call on `video[b:b+1]`, `queries[b:b+1]` (DESIGN.md 4.4.3).
"""
from __future__ import annotations

import hashlib
import math
from typing import List, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import engine
from .encoder import BasicEncoder
from .evaluation import pass_budget_bytes, plan_clip_passes, slab_tracks_for

HID, HEADS, VIRT, XDIM = 384, 8, 64, 1110


# ------------------------------------------------------------------------------------------------------
# parameter containers (names = checkpoint keys)
class _AttnParams(nn.Module):
    def __init__(self, dim: int = HID):
        super().__init__()
        self.to_q = nn.Linear(dim, dim)
        self.to_kv = nn.Linear(dim, 2 * dim)
        self.to_out = nn.Linear(dim, dim)


class _MlpParams(nn.Module):
    def __init__(self, din: int, dhid: int, dout: int):
        super().__init__()
        self.fc1 = nn.Linear(din, dhid)
        self.fc2 = nn.Linear(dhid, dout)


class _SelfBlockParams(nn.Module):  # reference AttnBlock (blocks.py:401-438); norm1/norm2 carry no parameters
    def __init__(self):
        super().__init__()
        self.attn = _AttnParams()
        self.mlp = _MlpParams(HID, 4 * HID, HID)


class _CrossBlockParams(nn.Module):  # reference CrossAttnBlock (cotracker.py:534-577)
    def __init__(self):
        super().__init__()
        self.norm_context = nn.LayerNorm(HID)
        self.cross_attn = _AttnParams()
        self.mlp = _MlpParams(HID, 4 * HID, HID)


class UpdateFormerParams(nn.Module):
    """Weights of EfficientUpdateFormer (reference cotracker.py:387-531); compute lives in csrc/."""

    def __init__(self, depth: int = 3):
        super().__init__()
        self.input_transform = nn.Linear(XDIM, HID)
        self.flow_head = nn.Linear(HID, 2)
        self.vis_conf_head = nn.Linear(HID, 2)
        self.virual_tracks = nn.Parameter(torch.randn(1, VIRT, 1, HID))  # (sic) checkpoint key
        self.time_blocks = nn.ModuleList(_SelfBlockParams() for _ in range(depth))
        self.space_virtual_blocks = nn.ModuleList(_SelfBlockParams() for _ in range(depth))
        self.space_point2virtual_blocks = nn.ModuleList(_CrossBlockParams() for _ in range(depth))
        self.space_virtual2point_blocks = nn.ModuleList(_CrossBlockParams() for _ in range(depth))
        for m in self.modules():
            if isinstance(m, nn.Linear):
                nn.init.xavier_uniform_(m.weight)
                nn.init.zeros_(m.bias)
        nn.init.trunc_normal_(self.flow_head.weight, std=0.001)
        nn.init.trunc_normal_(self.vis_conf_head.weight, std=0.001)


def sincos_time_embedding(dim: int, length: int) -> torch.Tensor:
    """[1, length, dim] buffer: sin half | cos half with 10000^(-i/(dim/2)) frequencies
    (reference embeddings.py:59-84, computed in float64 then cast)."""
    omega = 1.0 / 10000 ** (torch.arange(dim // 2, dtype=torch.float64) / (dim / 2.0))
    ang = torch.arange(length, dtype=torch.float64)[:, None] * omega[None, :]
    return torch.cat([ang.sin(), ang.cos()], dim=1)[None].float()


# ------------------------------------------------------------------------------------------------------
# frame maps (ct3_loop_shape.group_frames): which pyramid frame each group reads at each time step
def clip_frame_map(T: int, reversed_groups) -> List[List[int]]:
    """Offline model: a forward group reads frame t, a group on the clip played backwards frame T-1-t."""
    return [list(range(T - 1, -1, -1)) if r else list(range(T)) for r in reversed_groups]


def window_frame_map(T: int, S: int, ind: int, reversed_groups) -> List[List[int]]:
    """Sliding-window model, window starting at `ind` (non-streaming): frames of the clip padded to a multiple of S with
    copies of frame T-1.  A forward group reads ind+t.  The reversed clip is padded with copies of the original frame 0,
    so a reversed group reads max(T-1-ind-t, 0)."""
    return [[max(T - 1 - ind - t, 0) for t in range(S)] if r else [ind + t for t in range(S)] for r in reversed_groups]


def ragged_frame_map(T: int, groups) -> List[List[int]]:
    """Pass of clips of different lengths in one pyramid: groups = (first pyramid frame f0 of the clip, its length T_g,
    reversed) per group.  A group reads f0 + t (f0 + T_g-1-t reversed) and, at its padded steps t >= T_g, the frame of
    its last real step, as the sliding-window model clamps its padded window."""
    rows = []
    for f0, T_g, rev in groups:
        row = [f0 + (T_g - 1 - t if rev else t) for t in range(T_g)]
        rows.append(row + [row[-1]] * (T - T_g))
    return rows


def gather_plan(frame_map):
    """The runs [a, b) of consecutive frames a frame map references, in order, and the map remapped into the pyramid
    that concatenates those runs (each referenced frame once)."""
    used = sorted({f for row in frame_map for f in row})
    pos = {f: i for i, f in enumerate(used)}
    runs = []
    for f in used:
        if runs and runs[-1][1] == f:
            runs[-1][1] = f + 1
        else:
            runs.append([f, f + 1])
    return [tuple(r) for r in runs], [[pos[f] for f in row] for row in frame_map]


def gather_pyramid(pyr, T: int, H4: int, W4: int, runs) -> torch.Tensor:
    """Flat pyramid of the frame runs [a, b) of the T-frame pyramid `pyr`, concatenated in order."""
    return engine.concat_pyramid_runs([(pyr, T, a, b) for a, b in runs], H4, W4)


# A batch is stored clip after clip: clip c's frames are frames c * T_clip ... of one pyramid, its tracks follow clip
# c-1's, and its query groups are groups of the same update loop.  `clips` names the clips a pass tracks (all of them,
# or a sub-batch when the whole batch does not fit in device memory).
def batch_frame_map(frame_map, clips, T_clip: int) -> List[List[int]]:
    """The one-clip frame map repeated for each of `clips`: the groups of clip c read the same frames plus c * T_clip."""
    return [[f + c * T_clip for f in row] for c in clips for row in frame_map]


def batch_gather_plan(frame_map, clips, T_clip: int):
    """`gather_plan` of `batch_frame_map(frame_map, clips, T_clip)` with every run inside one clip: the one-clip plan
    repeated per clip, so clip number i of `clips` owns frames [i * n, (i + 1) * n) of the gathered pyramid."""
    runs, remap = gather_plan(frame_map)
    n = sum(b - a for a, b in runs)
    return ([(a + c * T_clip, b + c * T_clip) for c in clips for a, b in runs],
            [[p + i * n for p in row] for i in range(len(clips)) for row in remap])


def _reversed_flags(reversed_groups, G: int) -> List[bool]:
    flags = [False] * G if reversed_groups is None else [bool(r) for r in reversed_groups]
    if len(flags) != G:
        raise engine.EngineError(f"reversed_groups has {len(flags)} entries for {G} groups")
    return flags


# ------------------------------------------------------------------------------------------------------
# streaming: streams that each hold their own window start (CoTrackerThreeOnline._stream_step)
class StreamState:
    """One stream of the streaming model: its window start, the history of its tracks and the encoder features of its
    last chunk's overlap frames.  Its tracks are rows [first, first + n) of the `StreamPool` it belongs to.

    history=None keeps every frame (frame f at row f).  A bound h keeps the history in a ring that holds frame f at row
    f mod cap and only the last cap frames; the stream's results then cover its last h frames at most, and its memory
    does not grow with its length."""

    def __init__(self, n: int, first: int, history: Optional[int] = None):
        self.n, self.first = n, first
        self.history = history    # None, or the bound on the frames of each result
        self.ind = 0              # window start (the reference's online_ind)
        self.length = 0           # frames of history (written so far; a ring holds the last cap of them)
        self.hist = None          # (coords * stride [cap,n,2], vis [cap,n], conf [cap,n] logits); frames >= length unset
        self.enc = None           # (signatures [S-step,2], frame shape, pyramid) of the last chunk's overlap frames

    def ring_frames(self, S: int, step: int) -> int:
        """The ring of a bounded state, in frames.  A window at ind reads frames [ind + T - L, ind) for a result of
        L <= h frames (T >= 1 real frames) when the history holds frames up to ind + S - step, so h + S - step frames
        always suffice; the library takes S at least."""
        return max(S, self.history + S - step)

    def reserve(self, frames: int, device):
        """Room for `frames` history frames: the buffers at least double when they grow, so a stream reallocates
        O(log length) times.  A bounded state calls this once, with its `ring_frames`."""
        cap = 0 if self.hist is None else self.hist[1].shape[0]
        if frames <= cap:
            return
        cap = max(frames, 2 * cap)
        new = (torch.empty(cap, self.n, 2, device=device), torch.empty(cap, self.n, device=device),
               torch.empty(cap, self.n, device=device))
        if self.length:
            for a, b in zip(new, self.hist):
                a[:self.length] = b[:self.length]
        self.hist = new

    def edit(self, keep: torch.Tensor, at: int, coords: torch.Tensor):
        """The history side of `StreamPool.edit`: keep columns `keep` [k] (int64, in order) and insert m new columns
        after the first `at` of them that hold coords [m,2] (model resolution) with vis and conf logits 0 at every row:
        every frame of the history, and every row a ring holds.  The buffers keep their size."""
        m = coords.shape[0]
        if self.hist is not None:
            cap = self.hist[1].shape[0]
            new = (coords.expand(cap, m, 2), coords.new_zeros(cap, m), coords.new_zeros(cap, m))
            self.hist = tuple(torch.cat([h.index_select(1, keep[:at]), x, h.index_select(1, keep[at:])], 1)
                              for h, x in zip(self.hist, new))
        self.n = keep.shape[0] + m

    def export_history(self) -> Optional[List[torch.Tensor]]:
        """Host copies of the history rows a later window can read: the whole ring of a bounded state (frame f stays
        at row f mod cap), rows [0, length) otherwise; None before the first step."""
        if self.hist is None:
            return None
        rows = self.hist[1].shape[0] if self.history is not None else self.length
        return [h[:rows].to("cpu", copy=True) for h in self.hist]


class StreamPool:
    """The tracks of a set of streams, stream after stream: support features [4,49,N,128] (accumulated as queries enter
    the window), query frames [N] int32 (stream time) and query coordinates [N,2] (feature-grid units).  `open` appends
    a stream's tracks; `close` removes them and `edit` changes them, each with one copy of the pool.  `export` copies a
    stream's state to the host and `restore` appends it back, to this pool or another."""

    def __init__(self):
        self.streams: List[StreamState] = []
        self.support = self.qframes = self.qcoords = None

    def open(self, qframes: torch.Tensor, qcoords: torch.Tensor, history: Optional[int] = None,
             support: Optional[torch.Tensor] = None) -> StreamState:
        """Append a stream of the tracks qframes [n] / qcoords [n,2], with zero support features or `support`
        [4,49,n,128]."""
        n = qframes.shape[0]
        state = StreamState(n, 0 if self.qframes is None else self.qframes.shape[0], history)
        sup = torch.zeros(4, 49, n, 128, device=qframes.device) if support is None else support.contiguous()
        if self.support is None:
            self.support, self.qframes, self.qcoords = sup, qframes.contiguous(), qcoords.contiguous()
        else:
            self.support = torch.cat([self.support, sup], 2)
            self.qframes = torch.cat([self.qframes, qframes])
            self.qcoords = torch.cat([self.qcoords, qcoords])
        self.streams.append(state)
        return state

    def close(self, state: StreamState):
        a, b = state.first, state.first + state.n
        self.streams.remove(state)
        if not self.streams:
            self.support = self.qframes = self.qcoords = None
            return
        self.support = torch.cat([self.support[:, :, :a], self.support[:, :, b:]], 2)
        self.qframes = torch.cat([self.qframes[:a], self.qframes[b:]])
        self.qcoords = torch.cat([self.qcoords[:a], self.qcoords[b:]])
        for s in self.streams:
            if s.first >= b:
                s.first -= state.n

    def edit(self, state: StreamState, keep, at: int, qframes: torch.Tensor, qcoords: torch.Tensor, stride: int):
        """A column edit of `state`'s tracks, the way the reference's per-track tensors would be edited along their N
        axis: keep its tracks `keep` (indices into its n, in order), and insert the tracks of qframes [m] / qcoords [m,2]
        (as `open` takes them) after the first `at` kept ones.  A new track has zero support features and, at every frame
        of the history, its query point (qcoords * stride) with vis and conf logits 0."""
        a, b = state.first, state.first + state.n
        keep = torch.as_tensor(list(keep), dtype=torch.long).to(self.qframes.device)
        qframes, qcoords = qframes.to(self.qframes), qcoords.to(self.qcoords)
        head, tail = keep[:at] + a, keep[at:] + a

        def cols(x, dim, new):
            return torch.cat([x.narrow(dim, 0, a), x.index_select(dim, head), new, x.index_select(dim, tail),
                              x.narrow(dim, b, x.shape[dim] - b)], dim)

        support = cols(self.support, 2, self.support.new_zeros(4, 49, qframes.shape[0], 128))
        qf, qc = cols(self.qframes, 0, qframes), cols(self.qcoords, 0, qcoords)
        state.edit(keep, at, qcoords * float(stride))
        self.support, self.qframes, self.qcoords = support, qf, qc
        for s in self.streams:
            if s.first >= b:
                s.first += state.n - (b - a)

    def export(self, state: StreamState) -> dict:
        """`state`'s own values as host tensors and ints: its columns of the pool, its window start, length and bound,
        and its history (`StreamState.export_history`).  The encoder cache is left out: the first window after a
        `restore` encodes its chunk whole, which gives the same features (the encoder is strictly per frame)."""
        a, b = state.first, state.first + state.n
        return dict(n=state.n, ind=state.ind, length=state.length, history=state.history,
                    support=self.support[:, :, a:b].to("cpu", copy=True),
                    qframes=self.qframes[a:b].to("cpu", copy=True), qcoords=self.qcoords[a:b].to("cpu", copy=True),
                    hist=state.export_history())

    def restore(self, snap: dict, device) -> StreamState:
        """Append the stream of `export`'s `snap` on `device`, as `open` appends one; the state owns copies of the
        snapshot's tensors, so one snapshot can be restored any number of times."""
        state = self.open(snap["qframes"].to(device, copy=True), snap["qcoords"].to(device, copy=True),
                          snap["history"], support=snap["support"].to(device, copy=True))
        state.ind, state.length = snap["ind"], snap["length"]
        if snap["hist"] is not None:
            rows = snap["hist"][1].shape[0] if state.history is not None else state.length
            state.hist = tuple(h[:rows].to(device, copy=True).contiguous() for h in snap["hist"])
        return state


class CoTrackerThreeBase(nn.Module):
    def __init__(self, window_len=8, stride=4, corr_radius=3, corr_levels=4, num_virtual_tracks=64,
                 model_resolution=(384, 512), add_space_attn=True, linear_layer_for_vis_conf=True):
        super().__init__()
        if (stride, corr_radius, corr_levels, num_virtual_tracks) != (4, 3, 4, 64) or not add_space_attn \
                or not linear_layer_for_vis_conf:
            raise NotImplementedError("libct3_b200 implements the released CoTracker3 configuration only "
                                      "(stride 4, radius 3, 4 levels, 64 virtual tracks)")
        if tuple(model_resolution) != (384, 512):
            # the relative-motion posenc is normalised by model_resolution/stride = (128, 96) inside tokens.cu
            raise NotImplementedError("libct3_b200 hard-codes model_resolution=(384, 512) (posenc scale 128/96)")
        self.window_len = window_len
        self.stride = stride
        self.corr_radius = corr_radius
        self.corr_levels = corr_levels
        self.hidden_dim = 256
        self.latent_dim = 128
        self.num_virtual_tracks = num_virtual_tracks
        self.model_resolution = model_resolution
        self.input_dim = XDIM
        self.fnet = BasicEncoder(input_dim=3, output_dim=self.latent_dim, stride=stride)
        self.updateformer = UpdateFormerParams()
        self.corr_mlp = _MlpParams(49 * 49, 384, 256)
        self.register_buffer("time_emb", sincos_time_embedding(XDIM, window_len))
        self._packed: Optional[torch.Tensor] = None
        self._packed_key = None
        self._enc_packed: Optional[torch.Tensor] = None
        self._enc_key = None
        self._fingerprint: Optional[str] = None
        self._fingerprint_key = None
        self._ws = engine.WorkspaceCache()
        self._enc_ws: Optional[torch.Tensor] = None

    # -- engine plumbing ----------------------------------------------------------------------------------
    def _hot_state(self):
        sd = {}
        for k, v in self.named_parameters():
            if k.startswith("updateformer.") or k.startswith("corr_mlp."):
                sd[k] = v
        return sd

    def packed_weights(self, device) -> torch.Tensor:
        sd = self._hot_state()
        key = (str(device), tuple((v.data_ptr(), v._version) for v in sd.values()))
        if self._packed is None or self._packed_key != key:
            self._packed = engine.pack_weights(sd, device)
            self._packed_key = key
        return self._packed

    def weights_fingerprint(self) -> str:
        """sha256 over the names, dtypes, shapes and bytes of every parameter and buffer: the same string for the same
        weights on any device.  Computed once per weights version, like `packed_weights`."""
        tensors = sorted(self.state_dict(keep_vars=True).items())
        key = tuple((k, v.data_ptr(), v._version) for k, v in tensors)
        if self._fingerprint_key != key:
            h = hashlib.sha256()
            for k, v in tensors:
                h.update(f"{k}|{v.dtype}|{tuple(v.shape)};".encode())
                h.update(v.detach().reshape(-1).to("cpu").contiguous().view(torch.uint8).numpy())
            self._fingerprint, self._fingerprint_key = h.hexdigest(), key
        return self._fingerprint

    TIME_EMBED_CACHE = 64   # lengths whose interpolated time embedding is kept (a list call needs one per length)

    def interpolate_time_embed(self, t: int) -> torch.Tensor:
        """[t, 1110] time embedding (reference cotracker3_online.py:145-156); constant per (buffer, t): cached per
        length, for the last TIME_EMBED_CACHE lengths."""
        buf = (self.time_emb.data_ptr(), self.time_emb._version, str(self.time_emb.device))
        cache = getattr(self, "_te_cache", None)
        if not isinstance(cache, dict) or getattr(self, "_te_key", None) != buf:
            cache, self._te_key = {}, buf
            self._te_cache = cache
        if t not in cache:
            te = self.time_emb.float()
            if t != te.shape[1]:
                te = F.interpolate(te.permute(0, 2, 1), size=t, mode="linear").permute(0, 2, 1)
            if len(cache) >= self.TIME_EMBED_CACHE:
                del cache[next(iter(cache))]
            cache[t] = te[0].contiguous()
        return cache[t]

    def _encode(self, video: torch.Tensor, chunk: int) -> torch.Tensor:
        """video [T,3,H,W] already scaled to [-1,1] -> L2-normalised channels-last 4-level pyramid (flat fp32).

        The whole BasicEncoder (reference blocks.py:141-219) runs in libct3_b200.so (csrc/enc_front.cu + the GEMM
        engine): conv1 as fp32 SIMT, every other convolution as split-bf16x3 wgmma GEMMs, channels-last.  The
        library walks the clip in chunks of 16 frames itself (`chunk` = the reference's fmaps_chunk_size only bounds
        memory there and has no numerical effect: the encoder is strictly per frame)."""
        dev = video.device
        sd = {k: v for k, v in self.fnet.state_dict().items()}
        key = (str(dev), tuple((v.data_ptr(), v._version) for v in self.fnet.parameters()))
        if self._enc_packed is None or self._enc_key != key:
            self._enc_packed = engine.encoder_pack(sd, dev)
            self._enc_key = key
        T, _, H, W = video.shape
        need = engine.encoder_workspace_bytes(T, H, W)
        if self._enc_ws is None or self._enc_ws.numel() < need or self._enc_ws.device != dev:
            self._enc_ws = None
            self._enc_ws = torch.empty(need, dtype=torch.uint8, device=dev)
        return engine.encoder(self._enc_packed, video.contiguous(), self._enc_ws)

    def _check_inputs(self, video, queries, is_train):
        if is_train:
            raise NotImplementedError("cotracker_b200 is inference-only (training is out of scope, SURVEY.md §2)")
        B, T, C, H, W = video.shape
        if B < 1 or queries.dim() != 3 or queries.shape[0] != B:
            raise ValueError(f"video [B,T,3,H,W] and queries [B,N,3] must hold the same B >= 1 clips, got "
                             f"{tuple(video.shape)} and {tuple(queries.shape)}")
        assert H % self.stride == 0 and W % self.stride == 0
        if not video.is_cuda:
            raise engine.EngineError("cotracker_b200 runs on CUDA only; move the module and inputs to a GPU")

    def _refine(self, pyr, H4, W4, support, track_valid, coords, vis, conf, iters, group_sizes, group_frames=None,
                group_T=None):
        """group_frames: [G, T] frame map into `pyr` (ct3_loop_shape.group_frames), None = frame t.
        group_T: G group lengths (ct3_loop_shape.group_T), None = every group has T frames.
        A pass whose full workspace exceeds the pass budget runs in the largest track slabs that fit
        (ct3_loop_shape.slab_tracks, bit-identical); every other pass runs as it always did."""
        T, N, _ = coords.shape
        dev = coords.device
        G = len(group_sizes)
        T_all = engine.pyramid_frames(pyr, H4, W4)
        T_pyr = None if group_frames is None else T_all
        budget = pass_budget_bytes(self, dev, T_all, H4 * self.stride, W4 * self.stride)
        slab = slab_tracks_for(T, N, G, H4, W4, T_pyr, budget, group_T)
        if group_T is None:
            time_emb = self.interpolate_time_embed(T).to(dev)
        else:   # each group's own embedding, zero rows past its length
            time_emb = torch.zeros(G, T, XDIM, device=dev)
            for g, t in enumerate(group_T):
                time_emb[g, :t] = self.interpolate_time_embed(t).to(dev)
        ws = (self._ws.get(T, N, dev, H4, W4, G, T_pyr, slab) if group_T is None
              else self._ws.get(T, N, dev, H4, W4, G, T_pyr, slab, group_T))
        engine.update_loop(self.packed_weights(dev), pyr, H4, W4, support, track_valid, coords, vis, conf,
                           time_emb, iters, ws,
                           group_sizes=group_sizes, group_frames=group_frames, slab_tracks=slab, group_T=group_T)

    @staticmethod
    def _track_reversed(group_sizes, flags, device) -> torch.Tensor:
        """[N] bool: the tracks of the groups flagged as reversed."""
        return torch.repeat_interleave(torch.tensor(flags, dtype=torch.bool),
                                       torch.tensor(group_sizes, dtype=torch.int64)).to(device)

    @torch.no_grad()
    def forward_groups(self, video, queries, group_sizes, iters=4, fmaps_chunk_size=200, reversed_groups=None):
        """Track G independent query sets over one clip in one pass.

        queries [1, sum(group_sizes), 3] holds the groups one after another.  The clip is encoded once and the support
        features are sampled once; each window runs one update loop for all groups together (ct3_loop_shape.G),
        where every group keeps its own virtual tokens.  Returns the 4-tuple of `forward`; the columns of each group
        are bit-identical to `forward(video, that group's queries)`.  Streaming (is_online=True) is not grouped.
        reversed_groups: G flags; a flagged group is tracked on the clip played backwards (its query frames and its
        output are in reversed-clip time) and its columns are bit-identical to `forward(video.flip(1), its queries)`.
        The reversed clip is never encoded: those groups read the forward pyramid through a frame map."""
        sizes = [int(g) for g in group_sizes]
        if not sizes or any(g < 1 for g in sizes) or sum(sizes) != queries.shape[1]:
            raise engine.EngineError(f"group_sizes {sizes} must be >= 1 each and sum to the {queries.shape[1]} queries")
        _reversed_flags(reversed_groups, len(sizes))
        self._check_inputs(video, queries, False)
        return self._track(video, queries, iters, fmaps_chunk_size, sizes, reversed_groups=reversed_groups)

    # -- internal entry points of the predictors: frames already resized and normalised (cotracker_b200.ingest) --------
    def _check_frames(self, frames, queries):
        B = queries.shape[0] if queries.dim() == 3 else 0
        if frames.dim() != 4 or frames.shape[1] != 3 or B < 1 or frames.shape[0] % B or frames.shape[0] < B:
            raise ValueError(f"frames must be [B*T,3,H,W] (clip after clip) and queries [B,N,3], got "
                             f"{tuple(frames.shape)} and {tuple(queries.shape)}")
        if not frames.is_cuda:
            raise engine.EngineError("cotracker_b200 runs on CUDA only; move the module and inputs to a GPU")
        assert frames.shape[2] % self.stride == 0 and frames.shape[3] % self.stride == 0

    def _clip_pad(self, T: int) -> int:
        """Frames the model appends (copies of the last frame) before encoding a T-frame clip."""
        return 0

    def _encode_clip(self, frames, fmaps_chunk_size=200, B: int = 1) -> torch.Tensor:
        """frames [B*T,3,H,W] in [-1,1], clip after clip -> the pyramid `_track_pyramid` expects: every clip's frames
        followed by the model's padding frames, in one encoder pass."""
        pad = self._clip_pad(frames.shape[0] // B)
        if pad > 0:
            v = frames.unflatten(0, (B, -1))
            frames = torch.cat([v, v[:, -1:].expand(-1, pad, -1, -1, -1)], 1).flatten(0, 1)
        return self._encode(frames.contiguous(), fmaps_chunk_size)

    def _reverse_clip_pyramid_(self, pyr, T: int, H: int, W: int) -> torch.Tensor:
        """In place: `_encode_clip` of a T-frame clip -> `_encode_clip` of the clip played backwards (no encoder pass,
        no second pyramid); applying it again restores the original."""
        return engine.reverse_pyramid_(pyr, T, H // self.stride, W // self.stride, self._clip_pad(T))

    def _track_frames(self, frames, queries, iters=4, group_sizes=None, fmaps_chunk_size=200):
        """`forward` on frames [B*T,3,H,W] (clip after clip) already scaled to [-1,1] (the predictors' path)."""
        self._check_frames(frames, queries)
        B = queries.shape[0]
        BT, _, H, W = frames.shape
        return self._track_pyramid(self._encode_clip(frames, fmaps_chunk_size, B), BT // B, H, W, queries, iters,
                                   group_sizes or [queries.shape[1]])

    # -- batches: B clips in one pyramid, tracks and groups clip after clip ---------------------------------------------
    @staticmethod
    def _pass_clips(B: int, clips):
        """(clips a pass tracks, whether it is today's one-clip pass that needs neither clip offsets nor a frame map)."""
        if clips is None:
            return list(range(B)), B == 1
        clips = [int(c) for c in clips]
        if len(clips) != B:
            raise engine.EngineError(f"{B} query sets for clips {clips}")
        return clips, False

    @staticmethod
    def _clip_offsets(clips, T_clip: int, N: int, device) -> torch.Tensor:
        """[B*N] int64: the first pyramid frame of each track's clip."""
        return torch.tensor([c * T_clip for c in clips], dtype=torch.int64).repeat_interleave(N).to(device)

    @staticmethod
    def _batched(x: torch.Tensor, B: int) -> torch.Tensor:
        """[T, B*N, ...] (tracks clip after clip) -> [B, T, N, ...]; no copy for B = 1."""
        return x.unflatten(1, (B, -1)).transpose(0, 1).contiguous()


class CoTrackerThreeOffline(CoTrackerThreeBase):
    """Whole clip = one window (reference cotracker3_offline.py)."""

    @torch.no_grad()
    def forward(self, video, queries, iters=4, is_train=False, add_space_attn=True, fmaps_chunk_size=200):
        self._check_inputs(video, queries, is_train)
        return self._track(video, queries, iters, fmaps_chunk_size, [queries.shape[1]])

    def _track(self, video, queries, iters, fmaps_chunk_size, group_sizes, reversed_groups=None):
        B, T, C, H, W = video.shape
        assert T >= 1
        frames = 2.0 * (video.flatten(0, 1).float() / 255.0) - 1.0
        pyr = self._encode(frames, fmaps_chunk_size)
        return self._track_pyramid(pyr, T, H, W, queries, iters, group_sizes, reversed_groups)

    def _track_pyramid(self, pyr, T, H, W, queries, iters, group_sizes, reversed_groups=None, clips=None):
        """The model after the encoder: pyr = the pyramid of the clips (`_encode_clip`), T frames of H x W pixels each.
        group_sizes, reversed_groups: the G groups of one clip's N queries (every clip has the same), G flags; a
        flagged group tracks the clip played backwards (see `forward_groups`).
        clips: the clip of the pyramid each of the B rows of `queries` tracks (None: 0 .. B-1, the whole pyramid)."""
        B, N = queries.shape[:2]
        dev = pyr.device
        H4, W4 = H // self.stride, W // self.stride
        group_sizes = list(group_sizes)
        flags = _reversed_flags(reversed_groups, len(group_sizes))
        clips, plain = self._pass_clips(B, clips)
        qframes = queries[:, :, 0].long().reshape(-1)
        if any(flags):   # a reversed group's query frame q is frame T-1-q of the forward pyramid
            qframes = torch.where(self._track_reversed(group_sizes * B, flags * B, dev), T - 1 - qframes, qframes)
        if not plain:
            qframes = qframes + self._clip_offsets(clips, T, N, dev)
        qframes = qframes.to(torch.int32).contiguous()
        qcoords = (queries[:, :, 1:3].float() / self.stride).reshape(-1, 2).contiguous()
        support = engine.sample_support(pyr, T if plain else engine.pyramid_frames(pyr, H4, W4), H4, W4, qframes, qcoords)
        coords = qcoords[None].expand(T, B * N, 2).contiguous()
        vis = torch.zeros(T, B * N, device=dev)
        conf = torch.zeros(T, B * N, device=dev)
        frame_map = clip_frame_map(T, flags) if any(flags) or not plain else None
        if not plain:
            frame_map = batch_frame_map(frame_map, clips, T)
        self._refine(pyr, H4, W4, support, None, coords, vis, conf, iters, group_sizes * B, frame_map)
        return (self._batched(coords * float(self.stride), B), self._batched(torch.sigmoid(vis), B),
                self._batched(torch.sigmoid(conf), B), None)


    def _track_ragged(self, pyr, H, W, groups, iters):
        """One update-loop pass over query groups of clips of different lengths in one pyramid (`_encode_clip` of
        the clips one after another, H x W frames).  groups: (queries [1,n,3] at model resolution in the group's own
        clip time, first pyramid frame f0 of its clip, clip length T_g, reversed) per group; a reversed group tracks its
        clip played backwards and reads the forward pyramid through its frame map.  The pass pads every group to the
        longest T_g (ct3_loop_shape.group_T); a padded step reads its group's last frame.
        -> [(tracks [1,T_g,n,2] at model resolution, visibility [1,T_g,n])] per group, each bit-identical to the
        one-clip pass on that group (`_track_pyramid`)."""
        dev = pyr.device
        H4, W4 = H // self.stride, W // self.stride
        T = max(g[2] for g in groups)
        sizes = [q.shape[1] for q, *_ in groups]
        lengths = [int(T_g) for _, _, T_g, _ in groups]
        qframes = []
        for q, f0, T_g, rev in groups:
            qf = q[0, :, 0].long()
            qframes.append((T_g - 1 - qf if rev else qf) + f0)
        frame_map = ragged_frame_map(T, [(f0, T_g, rev) for _, f0, T_g, rev in groups])
        qframes = torch.cat(qframes).to(torch.int32).contiguous()
        qcoords = (torch.cat([q[0, :, 1:3] for q, *_ in groups]).float() / self.stride).contiguous()
        support = engine.sample_support(pyr, engine.pyramid_frames(pyr, H4, W4), H4, W4, qframes, qcoords)
        N = qcoords.shape[0]
        coords = qcoords[None].expand(T, N, 2).contiguous()
        vis = torch.zeros(T, N, device=dev)
        conf = torch.zeros(T, N, device=dev)
        self._refine(pyr, H4, W4, support, None, coords, vis, conf, iters, sizes, frame_map, lengths)
        out, a = [], 0
        for n, T_g in zip(sizes, lengths):
            out.append(((coords[:T_g, a:a + n] * float(self.stride))[None], torch.sigmoid(vis[:T_g, a:a + n])[None]))
            a += n
        return out


class CoTrackerThreeOnline(CoTrackerThreeBase):
    """Sliding windows of `window_len` frames, stride window_len/2 (reference cotracker3_online.py)."""

    def init_video_online_processing(self):
        self.online_ind = 0
        # B streams that advance in lockstep: the pool of their tracks, clip after clip, and one state per stream
        self._online_pool: Optional[StreamPool] = None
        self._online_streams: List[StreamState] = []

    def _encode_online(self, frames, chunk, step, H4, W4, streams):
        """frames [K*S,3,H,W]: the S-frame chunks of the K `streams`.  Consecutive online chunks of a stream overlap by
        window_len - step frames and the encoder is strictly per-frame (InstanceNorm statistics are per sample), so the
        features of the overlap are reused bit-for-bit from the stream's previous window and only the new frames are
        encoded (SURVEY.md 8(f1): the reference re-encodes all 16).  A stream whose overlap does not match its cache is
        encoded whole, in the same encoder pass as the other streams' new frames.  Each stream then keeps the features
        of its chunk's last window_len - step frames, and only those."""
        K = len(streams)
        S = frames.shape[0] // K
        keep = S - step
        shape = tuple(frames.shape[1:])
        # [K,S,2] float64: one pass over the chunks; one flag per stream goes to the host
        sig = self._frame_signatures(frames).unflatten(0, (K, S))
        same = [False] * K
        cand = [k for k, s in enumerate(streams) if keep > 0 and s.ind > 0 and s.enc is not None and s.enc[1] == shape]
        if cand:
            prev = torch.stack([streams[k].enc[0] for k in cand])
            for k, eq in zip(cand, (sig[cand, :keep] == prev).flatten(1).all(1).tolist()):
                same[k] = eq
        if any(same):
            v = frames.unflatten(0, (K, S))
            fresh = [v[k, keep:] if same[k] else v[k] for k in range(K)]
            fresh = fresh[0] if K == 1 else torch.cat(fresh, 0)
            new = self._encode(fresh.contiguous(), chunk)
            runs, n = [], 0
            for k in range(K):
                if same[k]:
                    runs.append((streams[k].enc[2], keep, 0, keep))
                m = step if same[k] else S
                runs.append((new, fresh.shape[0], n, n + m))
                n += m
            pyr = engine.concat_pyramid_runs(runs, H4, W4)
        else:
            pyr = self._encode(frames, chunk)
        if keep > 0:
            for k, s in enumerate(streams):
                s.enc = (sig[k, step:], shape, engine.concat_pyramid_runs([(pyr, K * S, k * S + step, (k + 1) * S)],
                                                                          H4, W4))
        return pyr

    def stream_advance_error(self, state: "StreamState", T: int) -> Optional[str]:
        """Why `state` cannot advance by a chunk of T frames (None: it can).  The history of a stream is the window
        results of its frames so far; a window at `ind` > 0 needs the previous window's overlap and extends the history
        by min(step, T - step) frames, to ind + T.  After a chunk shorter than the window that no longer holds."""
        S = self.window_len
        step = S // 2
        if not 1 <= T <= S:
            return f"a chunk must hold 1 to window_len = {S} frames, got {T}"
        if state.ind > 0 and (state.length != state.ind + S - step or state.length + min(step, T - step) != state.ind + T):
            return "the stream has ended: its last chunk was shorter than the window"
        if state.ind + S > engine.STREAM_FRAME_LIMIT:   # the library's window start limit, checked before any work
            return "the stream has reached the frame limit: a window must end by frame 2^30"
        return None

    def _stream_step(self, pool: "StreamPool", streams, frames, Ts, iters, chunk=200, outputs=None):
        """Advance each of `streams` (states of `pool`, in pool order) by one window, in as few update-loop passes as
        fit in device memory.  frames [K*S,3,H,W] in [-1,1]: stream k's chunk of Ts[k] frames, padded to S frames with
        copies of its last frame.  outputs: per stream None, or (n_keep, scale_xy) for the online predictor's output
        of all its frames so far, or (n_keep, scale_xy, L) for that of its last L frames only (L <= ind + T; a bounded
        state's results need L <= its bound).  -> per stream None or (tracks [L,n_keep,2] fp32, visibility [L,n_keep]
        bool), L = ind + T without a bound.  Every stream's result is bit-identical to advancing it alone: streams are
        independent query groups, each reading its own S frames of one pyramid."""
        K = len(streams)
        S = self.window_len
        step = S // 2
        _, _, H, W = frames.shape
        H4, W4 = H // self.stride, W // self.stride
        dev = frames.device
        for s, T in zip(streams, Ts):
            err = self.stream_advance_error(s, T)
            if err:
                raise ValueError(err)
        outputs = outputs or [None] * K
        pyr = self._encode_online(frames, chunk, step, H4, W4, streams)
        T_pyr = K * S
        for s, T in zip(streams, Ts):
            s.reserve(s.ind + T if s.history is None else s.ring_frames(S, step), dev)
        passes = [(0, K)]
        if K > 1:
            budget = pass_budget_bytes(self, dev, T_pyr, H, W)
            passes = plan_clip_passes(K, [[s.n] for s in streams], S, H4, W4, budget, lambda n: T_pyr)
        results = [None] * K
        for b0, b1 in passes:
            sub = streams[b0:b1]
            in_place = sub == pool.streams
            if in_place:
                support, qframes, qcoords = pool.support, pool.qframes, pool.qcoords
            else:   # the support rows of these streams in pass scratch, written back after the pass
                idx = torch.cat([torch.arange(s.first, s.first + s.n) for s in sub]).to(dev)
                support = pool.support.index_select(2, idx)
                qframes, qcoords = pool.qframes[idx], pool.qcoords[idx]
            entries, first = [], 0
            for k, s in enumerate(sub, b0):
                out, n_keep, scale, out_first = None, 0, (1.0, 1.0), 0
                if outputs[k] is not None:
                    n_keep, scale = outputs[k][:2]
                    rows = s.ind + Ts[k] if len(outputs[k]) < 3 else outputs[k][2]
                    out_first = s.ind + Ts[k] - rows
                    out = (torch.empty(rows, n_keep, 2, device=dev), torch.empty(rows, n_keep, dtype=torch.bool,
                                                                                 device=dev))
                    results[k] = out
                entries.append(engine.online_stream(s.hist, s.length, s.ind, Ts[k], first, k * S, out, n_keep, scale,
                                                    out_first=out_first, ring=s.history is not None))
                first += s.n
            valid, entering, rel, coords, vis, conf = engine.online_window_begin(entries, S, step, self.stride, T_pyr,
                                                                                 qframes, qcoords)
            engine.sample_support(pyr, T_pyr, H4, W4, rel, qcoords, support=support, accumulate_mask=entering)
            frame_map = None if K == 1 else [[k * S + t for t in range(S)] for k in range(b0, b1)]
            self._refine(pyr, H4, W4, support, valid, coords, vis, conf, iters, [s.n for s in sub], frame_map)
            engine.online_window_end(entries, S, self.stride, coords, vis, conf)
            if not in_place:
                pool.support.index_copy_(2, idx, support)
        for s, T in zip(streams, Ts):
            s.length = s.ind + T
            s.ind += step
        return results

    def _lockstep_streams(self, queries):
        """The pool and states of the B streams of queries [B,N,3] that advance in lockstep (opened at the first chunk
        after init_video_online_processing); the query points are taken from this call's queries."""
        B, N = queries.shape[:2]
        qframes, qcoords = self._stream_queries(queries.reshape(B * N, 3))
        if self._online_pool is None:
            self._online_pool = StreamPool()
            self._online_streams = [self._online_pool.open(qframes[b * N:(b + 1) * N], qcoords[b * N:(b + 1) * N])
                                    for b in range(B)]
        pool = self._online_pool
        if pool.qframes.shape[0] != B * N:
            raise ValueError(f"the video was started with {pool.qframes.shape[0]} tracks, these queries hold {B * N}")
        pool.qframes, pool.qcoords = qframes, qcoords
        return pool, self._online_streams

    def _stream_queries(self, queries):
        """queries [n,3] (t, x, y) at model resolution -> (query frames [n] int32 within +-QUERY_FRAME_LIMIT, query
        coordinates [n,2] fp32 in feature-grid units)."""
        lim = engine.QUERY_FRAME_LIMIT
        qframes = queries[:, 0].long().clamp(-lim, lim).to(torch.int32).contiguous()
        return qframes, (queries[:, 1:3].float() / self.stride).contiguous()

    def _track_online(self, frames, queries, iters, chunk=200, predict=None):
        """One streaming step of the B streams of queries [B,N,3] in lockstep; frames [B*T,3,H,W] in [-1,1], T <=
        window_len.  -> the model's (coords, vis, conf) [B, frames so far, N, ...], or with predict = (n_keep,
        scale_xy) the online predictor's (tracks [B,.,n_keep,2], visibility [B,.,n_keep] bool)."""
        B = queries.shape[0]
        T = frames.shape[0] // B
        S = self.window_len
        assert T <= S, "Online mode: video chunk must be <= window size."
        assert getattr(self, "online_ind", None) is not None, "Call model.init_video_online_processing() first."
        if S > T:
            v = frames.unflatten(0, (B, T))
            frames = torch.cat([v, v[:, -1:].expand(-1, S - T, -1, -1, -1)], 1).flatten(0, 1)
        pool, streams = self._lockstep_streams(queries)
        outs = self._stream_step(pool, streams, frames, [T] * B, iters, chunk, [predict] * B)
        self.online_ind += S // 2
        if predict is not None:
            return tuple(torch.stack([o[i] for o in outs]) for i in range(2))
        L = streams[0].length
        coords, vis, conf = (torch.stack([s.hist[i][:L] for s in streams]) for i in range(3))
        return coords, torch.sigmoid(vis), torch.sigmoid(conf), None

    def _frame_signatures(self, frames: torch.Tensor) -> torch.Tensor:
        """Two order-sensitive checksums per frame (plain sum and a position-weighted sum, float64 accumulators):
        frames whose signatures match the previous chunk's are taken to be the same frames.  Replaces a full
        `torch.equal` against a retained 38 MB copy of the previous chunk (ADVICE r1)."""
        S = frames.shape[0]
        flat = frames.reshape(S, -1)
        key = (flat.shape[1], str(flat.device))
        if getattr(self, "_sig_key", None) != key:
            g = torch.Generator().manual_seed(0x5eed)
            self._sig_w = torch.rand(flat.shape[1], generator=g, dtype=torch.float32).to(flat.device)
            self._sig_key = key
        a = flat.sum(dim=1, dtype=torch.float64)
        b = (flat * self._sig_w).sum(dim=1, dtype=torch.float64)
        return torch.stack([a, b], dim=1)

    @torch.no_grad()
    def forward(self, video, queries, iters=4, is_train=False, add_space_attn=True, fmaps_chunk_size=200,
                is_online=False):
        self._check_inputs(video, queries, is_train)
        return self._track(video, queries, iters, fmaps_chunk_size, [queries.shape[1]], is_online)

    def _clip_pad(self, T: int) -> int:
        S = self.window_len
        return (S - T % S) % S

    def _track(self, video, queries, iters, fmaps_chunk_size, group_sizes, is_online=False, reversed_groups=None):
        frames = 2.0 * (video.flatten(0, 1).float() / 255.0) - 1.0
        return self._track_normalised(frames, queries, iters, fmaps_chunk_size, group_sizes, is_online, reversed_groups)

    def _track_frames(self, frames, queries, iters=4, group_sizes=None, fmaps_chunk_size=200, is_online=False):
        self._check_frames(frames, queries)
        return self._track_normalised(frames, queries, iters, fmaps_chunk_size, group_sizes or [queries.shape[1]],
                                      is_online)

    def _track_normalised(self, frames, queries, iters, fmaps_chunk_size, group_sizes, is_online, reversed_groups=None):
        """frames [B*T,3,H,W], clip after clip, B = queries.shape[0]."""
        B = queries.shape[0]
        BT, _, H, W = frames.shape
        T = BT // B
        assert self.window_len >= 2
        if is_online:
            if any(_reversed_flags(reversed_groups, len(group_sizes))) or len(group_sizes) != 1:
                raise NotImplementedError("streaming (is_online=True) tracks one forward group per stream")
            return self._track_online(frames, queries, iters, fmaps_chunk_size)
        pyr_all = self._encode_clip(frames, fmaps_chunk_size, B)
        return self._track_pyramid(pyr_all, T, H, W, queries, iters, group_sizes, reversed_groups=reversed_groups)

    def _track_pyramid(self, pyr_all, T, H, W, queries, iters, group_sizes, reversed_groups=None, clips=None):
        """The model after the encoder, sliding windows over whole clips (streaming is `_stream_step`): pyr_all = the
        pyramid of the clips, each T frames and the padding (`_encode_clip`).  group_sizes, reversed_groups: the G
        groups of one clip's N queries (every clip has the same), G flags; a flagged group tracks the clip played
        backwards (see `forward_groups`).  With reversed groups or more than one clip each window runs on the frames its
        groups reference (at most 2 S per clip), gathered from pyr_all, through a frame map.
        clips: the clip of the pyramid each of the B rows of `queries` tracks (None: 0 .. B-1, the whole pyramid).
        Below, N counts the tracks of all B clips, clip after clip."""
        dev = pyr_all.device
        B = queries.shape[0]
        N = B * queries.shape[1]
        S = self.window_len
        step = S // 2
        H4, W4 = H // self.stride, W // self.stride
        T_pad = T + self._clip_pad(T)
        flags = _reversed_flags(reversed_groups, len(group_sizes))
        clips, plain = self._pass_clips(B, clips)
        T_all = T_pad if plain else engine.pyramid_frames(pyr_all, H4, W4)
        clip_off = None if plain else self._clip_offsets(clips, T_pad, queries.shape[1], dev)
        G1 = len(flags)                                   # groups of one clip
        group_sizes, flags = list(group_sizes) * B, flags * B
        qframes_l = queries[:, :, 0].long().reshape(-1)
        qcoords = (queries[:, :, 1:3].float() / self.stride).reshape(-1, 2).contiguous()

        coords_pred = torch.zeros(T, N, 2, device=dev)
        vis_pred = torch.zeros(T, N, device=dev)
        conf_pred = torch.zeros(T, N, device=dev)

        # support features of every track at its query frame
        qf = qframes_l.clamp(0, T_pad - 1)
        if any(flags):   # frame q of the reversed, padded clip is forward frame max(T-1-q, 0)
            qf = torch.where(self._track_reversed(group_sizes, flags, dev), (T - 1 - qf).clamp(min=0), qf)
        if not plain:
            qf = qf + clip_off
        support = engine.sample_support(pyr_all, T_all, H4, W4, qf.to(torch.int32).contiguous(), qcoords)

        coords_init = qcoords[None].expand(S, N, 2).contiguous()
        vis_init = torch.zeros(S, N, device=dev)
        conf_init = torch.zeros(S, N, device=dev)
        num_windows = (T - S + step - 1) // step + 1

        for ind in range(0, step * num_windows, step):
            if ind > 0:
                # warm start from the overlap with the previous window (reference :457-482)
                overlap = S - step
                carry = (qframes_l < ind + overlap)[None, :]                               # [1,N]
                prev_c = coords_pred[ind:ind + overlap] / self.stride
                prev_c = torch.cat([prev_c, prev_c[-1:].expand(step, -1, -1)], 0)
                prev_v = vis_pred[ind:ind + overlap]
                prev_v = torch.cat([prev_v, prev_v[-1:].expand(step, -1)], 0)
                prev_q = conf_pred[ind:ind + overlap]
                prev_q = torch.cat([prev_q, prev_q[-1:].expand(step, -1)], 0)
                coords_init = torch.where(carry[..., None], prev_c, coords_init)
                vis_init = torch.where(carry, prev_v, vis_init)
                conf_init = torch.where(carry, prev_q, conf_init)
            valid = (qframes_l < ind + S).to(torch.uint8).contiguous()                      # reference :484,:493-496
            frame_map = None
            if any(flags) or not plain:
                runs, frame_map = batch_gather_plan(window_frame_map(T, S, ind, flags[:G1]), clips, T_pad)
                pyr = gather_pyramid(pyr_all, T_all, H4, W4, runs)
            else:
                pyr = engine.slice_pyramid(pyr_all, T_pad, H4, W4, ind, S)
            coords = coords_init.clone().contiguous()
            vis = vis_init.clone().contiguous()
            conf = conf_init.clone().contiguous()
            self._refine(pyr, H4, W4, support, valid, coords, vis, conf, iters, group_sizes, frame_map)
            S_trim = min(T - ind, S)
            coords_pred[ind:ind + S] = (coords * float(self.stride))[:S_trim]
            vis_pred[ind:ind + S] = vis[:S_trim]
            conf_pred[ind:ind + S] = conf[:S_trim]

        return (self._batched(coords_pred, B), self._batched(torch.sigmoid(vis_pred), B),
                self._batched(torch.sigmoid(conf_pred), B), None)
