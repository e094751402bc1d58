"""CoTracker3 models whose iterative update loop runs in libct3_b200.so.

Drop-in mirror of the reference's inner model API (SURVEY.md §8b):
    CoTrackerThreeOffline.forward  -- reference cotracker3_offline.py:19-233
    CoTrackerThreeOnline.forward   -- reference cotracker3_online.py:266-541 (+ init_video_online_processing :163-169)
with the same constructor kwargs, attributes (`model_resolution`, `window_len`, `stride`) and the same
state-dict keys (SURVEY.md Appendix B), so `load_state_dict(strict=True)` of the released checkpoints works.

The nn.Module tree below is a *parameter container*: nothing executes through PyTorch modules.  The CNN
encoder, L2-normalisation + pyramid, support sampling, correlation sampling, the correlation MLP, the whole
EfficientUpdateFormer and the delta heads run as hand-written sm_90a CUDA behind the C ABI
(`cotracker_b200.engine`).  Inference only; B must be 1 (as in the reference, SURVEY.md §0).
"""
from __future__ import annotations

import math
from typing import List, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import engine
from .encoder import BasicEncoder

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
# frame maps (ct3_update_loop_frames): which pyramid frame each group reads at each time step
def clip_frame_map(T: int, reversed_groups) -> List[List[int]]:
    """Offline model: a forward group reads frame t, a group on the clip played backwards frame T-1-t."""
    return [list(range(T - 1, -1, -1)) if r else list(range(T)) for r in reversed_groups]


def window_frame_map(T: int, S: int, ind: int, reversed_groups) -> List[List[int]]:
    """Sliding-window model, window starting at `ind` (non-streaming): frames of the clip padded to a multiple of S with
    copies of frame T-1.  A forward group reads ind+t.  The reversed clip is padded with copies of the original frame 0,
    so a reversed group reads max(T-1-ind-t, 0)."""
    return [[max(T - 1 - ind - t, 0) for t in range(S)] if r else [ind + t for t in range(S)] for r in reversed_groups]


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
    out, n = None, 0
    for a, b in runs:
        part = engine.slice_pyramid(pyr, T, H4, W4, a, b - a)
        out = part if out is None else engine.concat_pyramid_frames(out, n, 0, part, b - a, H4, W4)
        n += b - a
    return out


def _reversed_flags(reversed_groups, G: int) -> List[bool]:
    flags = [False] * G if reversed_groups is None else [bool(r) for r in reversed_groups]
    if len(flags) != G:
        raise engine.EngineError(f"reversed_groups has {len(flags)} entries for {G} groups")
    return flags


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

    def interpolate_time_embed(self, t: int) -> torch.Tensor:
        """[t, 1110] time embedding (reference cotracker3_online.py:145-156); constant per (buffer, t): cached."""
        key = (t, self.time_emb.data_ptr(), self.time_emb._version, str(self.time_emb.device))
        if getattr(self, "_te_key", None) != key:
            te = self.time_emb.float()
            if t != te.shape[1]:
                te = F.interpolate(te.permute(0, 2, 1), size=t, mode="linear").permute(0, 2, 1)
            self._te_cache, self._te_key = te[0].contiguous(), key
        return self._te_cache

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
        if B != 1 or queries.shape[0] != 1:
            raise ValueError("CoTracker3 inference requires B == 1 (the reference fails for B > 1 as well)")
        assert H % self.stride == 0 and W % self.stride == 0
        if not video.is_cuda:
            raise engine.EngineError("cotracker_b200 runs on CUDA only; move the module and inputs to a GPU")

    def _refine(self, pyr, H4, W4, support, track_valid, coords, vis, conf, iters, group_sizes, group_frames=None):
        """group_frames: [G, T] frame map into `pyr` (ct3_update_loop_frames), None = frame t."""
        T, N, _ = coords.shape
        dev = coords.device
        G = len(group_sizes)
        T_pyr = None if group_frames is None else engine.pyramid_frames(pyr, H4, W4)
        engine.update_loop(self.packed_weights(dev), pyr, H4, W4, support, track_valid, coords, vis, conf,
                           self.interpolate_time_embed(T).to(dev), iters, self._ws.get(T, N, dev, H4, W4, G, T_pyr),
                           group_sizes=group_sizes if G > 1 or group_frames is not None else None,
                           group_frames=group_frames)

    @staticmethod
    def _track_reversed(group_sizes, flags, device) -> torch.Tensor:
        """[N] bool: the tracks of the groups flagged as reversed."""
        return torch.repeat_interleave(torch.tensor(flags, dtype=torch.bool),
                                       torch.tensor(group_sizes, dtype=torch.int64)).to(device)

    @torch.no_grad()
    def forward_groups(self, video, queries, group_sizes, iters=4, fmaps_chunk_size=200, reversed_groups=None):
        """Track G independent query sets over one clip in one pass.

        queries [1, sum(group_sizes), 3] holds the groups one after another.  The clip is encoded once and the support
        features are sampled once; each window runs one update loop for all groups together (ct3_update_loop_groups),
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
        if frames.dim() != 4 or frames.shape[1] != 3 or queries.shape[0] != 1:
            raise ValueError("frames must be [T,3,H,W] and queries [1,N,3] (B == 1)")
        if not frames.is_cuda:
            raise engine.EngineError("cotracker_b200 runs on CUDA only; move the module and inputs to a GPU")
        assert frames.shape[2] % self.stride == 0 and frames.shape[3] % self.stride == 0

    def _clip_pad(self, T: int) -> int:
        """Frames the model appends (copies of the last frame) before encoding a T-frame clip."""
        return 0

    def _encode_clip(self, frames, fmaps_chunk_size=200) -> torch.Tensor:
        """frames [T,3,H,W] in [-1,1] -> the pyramid `_track_pyramid` expects (with the model's padding frames)."""
        pad = self._clip_pad(frames.shape[0])
        if pad > 0:
            frames = torch.cat([frames, frames[-1:].expand(pad, -1, -1, -1)], 0)
        return self._encode(frames.contiguous(), fmaps_chunk_size)

    def _reverse_clip_pyramid_(self, pyr, T: int, H: int, W: int) -> torch.Tensor:
        """In place: `_encode_clip` of a T-frame clip -> `_encode_clip` of the clip played backwards (no encoder pass,
        no second pyramid); applying it again restores the original."""
        return engine.reverse_pyramid_(pyr, T, H // self.stride, W // self.stride, self._clip_pad(T))

    def _track_frames(self, frames, queries, iters=4, group_sizes=None, fmaps_chunk_size=200):
        """`forward` on frames [T,3,H,W] already scaled to [-1,1] (the predictors' path)."""
        self._check_frames(frames, queries)
        T, _, H, W = frames.shape
        return self._track_pyramid(self._encode_clip(frames, fmaps_chunk_size), T, H, W, queries, iters,
                                   group_sizes or [queries.shape[1]])


class CoTrackerThreeOffline(CoTrackerThreeBase):
    """Whole clip = one window (reference cotracker3_offline.py)."""

    @torch.no_grad()
    def forward(self, video, queries, iters=4, is_train=False, add_space_attn=True, fmaps_chunk_size=200):
        self._check_inputs(video, queries, is_train)
        return self._track(video, queries, iters, fmaps_chunk_size, [queries.shape[1]])

    def _track(self, video, queries, iters, fmaps_chunk_size, group_sizes, reversed_groups=None):
        B, T, C, H, W = video.shape
        assert T >= 1
        frames = 2.0 * (video[0].float() / 255.0) - 1.0
        pyr = self._encode(frames, fmaps_chunk_size)
        return self._track_pyramid(pyr, T, H, W, queries, iters, group_sizes, reversed_groups)

    def _track_pyramid(self, pyr, T, H, W, queries, iters, group_sizes, reversed_groups=None):
        """The model after the encoder: pyr = the clip's pyramid (`_encode_clip`), T frames of H x W pixels.
        reversed_groups: G flags; a flagged group tracks the clip played backwards (see `forward_groups`)."""
        N = queries.shape[1]
        H4, W4 = H // self.stride, W // self.stride
        flags = _reversed_flags(reversed_groups, len(group_sizes))
        qframes = queries[0, :, 0].long()
        if any(flags):   # a reversed group's query frame q is frame T-1-q of the forward pyramid
            qframes = torch.where(self._track_reversed(group_sizes, flags, qframes.device), T - 1 - qframes, qframes)
        qframes = qframes.to(torch.int32).contiguous()
        qcoords = (queries[0, :, 1:3].float() / self.stride).contiguous()
        support = engine.sample_support(pyr, T, H4, W4, qframes, qcoords)
        coords = qcoords[None].expand(T, N, 2).contiguous()
        vis = torch.zeros(T, N, device=pyr.device)
        conf = torch.zeros(T, N, device=pyr.device)
        self._refine(pyr, H4, W4, support, None, coords, vis, conf, iters, group_sizes,
                     clip_frame_map(T, flags) if any(flags) else None)
        return (coords * float(self.stride))[None], torch.sigmoid(vis)[None], torch.sigmoid(conf)[None], None


class CoTrackerThreeOnline(CoTrackerThreeBase):
    """Sliding windows of `window_len` frames, stride window_len/2 (reference cotracker3_online.py)."""

    def init_video_online_processing(self):
        self.online_ind = 0
        self.online_track_support = None          # [4,49,N,128], accumulated as queries enter the window
        self.online_coords_predicted = None
        self.online_vis_predicted = None
        self.online_conf_predicted = None
        self._online_enc_cache = None             # (per-frame checksums, pyramid) of the previous chunk

    def _encode_online(self, frames, chunk, step, H4, W4):
        """Consecutive online chunks overlap by window_len - step frames and the encoder is strictly per-frame
        (InstanceNorm statistics are per sample), so the features of the overlap are reused bit-for-bit from the
        previous call and only the new frames are encoded (SURVEY.md 8(f1): the reference re-encodes all 16)."""
        S = frames.shape[0]
        keep = S - step
        cache = getattr(self, "_online_enc_cache", None)
        sig = self._frame_signatures(frames)           # [S,2] float64: one pass over the chunk, 16 numbers to the host
        pyr = None
        if cache is not None and self.online_ind > 0 and keep > 0:
            prev_sig, prev_shape, prev_pyr = cache
            if prev_shape == frames.shape and torch.equal(sig[:keep], prev_sig[step:]):
                new = self._encode(frames[keep:].contiguous(), chunk)
                pyr = engine.concat_pyramid_frames(prev_pyr, S, step, new, S - keep, H4, W4)
        if pyr is None:
            pyr = self._encode(frames, chunk)
        self._online_enc_cache = (sig, frames.shape, pyr)
        return pyr

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
        frames = 2.0 * (video[0].float() / 255.0) - 1.0
        return self._track_normalised(frames, queries, iters, fmaps_chunk_size, group_sizes, is_online, reversed_groups)

    def _track_frames(self, frames, queries, iters=4, group_sizes=None, fmaps_chunk_size=200, is_online=False):
        self._check_frames(frames, queries)
        return self._track_normalised(frames, queries, iters, fmaps_chunk_size, group_sizes or [queries.shape[1]],
                                      is_online)

    def _track_normalised(self, frames, queries, iters, fmaps_chunk_size, group_sizes, is_online, reversed_groups=None):
        T, _, H, W = frames.shape
        S = self.window_len
        assert S >= 2
        if is_online:
            assert T <= S, "Online mode: video chunk must be <= window size."
            assert getattr(self, "online_ind", None) is not None, "Call model.init_video_online_processing() first."
            H4, W4 = H // self.stride, W // self.stride
            frames = torch.cat([frames, frames[-1:].expand(S - T, -1, -1, -1)], 0) if S > T else frames
            pyr_all = self._encode_online(frames, fmaps_chunk_size, S // 2, H4, W4)
        else:
            pyr_all = self._encode_clip(frames, fmaps_chunk_size)
        return self._track_pyramid(pyr_all, T, H, W, queries, iters, group_sizes, is_online, reversed_groups)

    def _track_pyramid(self, pyr_all, T, H, W, queries, iters, group_sizes, is_online=False, reversed_groups=None):
        """The model after the encoder: pyr_all = the pyramid of the T frames and the padding (`_encode_clip`).
        reversed_groups: G flags; a flagged group tracks the clip played backwards (see `forward_groups`).  Each window
        then runs on the frames its groups reference (at most 2 S), gathered from pyr_all, through a frame map."""
        dev = pyr_all.device
        N = queries.shape[1]
        S = self.window_len
        step = S // 2
        H4, W4 = H // self.stride, W // self.stride
        T_pad = T + ((S - T) if is_online else self._clip_pad(T))
        flags = _reversed_flags(reversed_groups, len(group_sizes))
        if is_online and any(flags):
            raise NotImplementedError("streaming (is_online=True) does not track reversed groups")
        qframes_l = queries[0, :, 0].long()
        qcoords = (queries[0, :, 1:3].float() / self.stride).contiguous()

        coords_pred = torch.zeros(T, N, 2, device=dev)
        vis_pred = torch.zeros(T, N, device=dev)
        conf_pred = torch.zeros(T, N, device=dev)
        if is_online and self.online_coords_predicted is not None:
            grow = min(step, T - step)
            coords_pred = F.pad(self.online_coords_predicted, (0, 0, 0, 0, 0, grow))
            vis_pred = F.pad(self.online_vis_predicted, (0, 0, 0, grow))
            conf_pred = F.pad(self.online_conf_predicted, (0, 0, 0, grow))

        # support features of every track at its query frame
        if is_online:
            left = 0 if self.online_ind == 0 else self.online_ind + step
            right = self.online_ind + S
            entering = ((qframes_l >= left) & (qframes_l < right)).to(torch.uint8).contiguous()
            if self.online_track_support is None:
                self.online_track_support = torch.zeros(4, 49, N, 128, device=dev)
            rel = (qframes_l - self.online_ind).clamp(0, T_pad - 1).to(torch.int32).contiguous()
            engine.sample_support(pyr_all, T_pad, H4, W4, rel, qcoords, support=self.online_track_support,
                                  accumulate_mask=entering)
            support = self.online_track_support
        else:
            qf = qframes_l.clamp(0, T_pad - 1)
            if any(flags):   # frame q of the reversed, padded clip is forward frame max(T-1-q, 0)
                qf = torch.where(self._track_reversed(group_sizes, flags, dev), (T - 1 - qf).clamp(min=0), qf)
            support = engine.sample_support(pyr_all, T_pad, H4, W4, qf.to(torch.int32).contiguous(), qcoords)

        coords_init = qcoords[None].expand(S, N, 2).contiguous()
        vis_init = torch.zeros(S, N, device=dev)
        conf_init = torch.zeros(S, N, device=dev)
        num_windows = (T - S + step - 1) // step + 1
        starts = [self.online_ind] if is_online else list(range(0, step * num_windows, step))

        for ind in starts:
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
            if is_online:
                pyr = pyr_all
            elif any(flags):
                runs, frame_map = gather_plan(window_frame_map(T, S, ind, flags))
                pyr = gather_pyramid(pyr_all, T_pad, H4, W4, runs)
            else:
                pyr = engine.slice_pyramid(pyr_all, T_pad, H4, W4, ind, S)
            coords = coords_init.clone().contiguous()
            vis = vis_init.clone().contiguous()
            conf = conf_init.clone().contiguous()
            self._refine(pyr, H4, W4, support, valid, coords, vis, conf, iters, group_sizes, frame_map)
            S_trim = T if is_online else min(T - ind, S)
            coords_pred[ind:ind + S] = (coords * float(self.stride))[:S_trim]
            vis_pred[ind:ind + S] = vis[:S_trim]
            conf_pred[ind:ind + S] = conf[:S_trim]

        if is_online:
            self.online_ind += step
            self.online_coords_predicted = coords_pred
            self.online_vis_predicted = vis_pred
            self.online_conf_predicted = conf_pred
        return coords_pred[None], torch.sigmoid(vis_pred)[None], torch.sigmoid(conf_pred)[None], None
