"""Track visualiser with the reference's interface (cotracker/utils/visualizer.py), drawn by library kernels.

    vis = Visualizer(save_dir="./saved_videos", pad_value=120, linewidth=3)
    frames = vis.visualize(video, pred_tracks, pred_visibility, save_video=False)   # uint8 [1,T',3,H',W'] on the host

The frames are bit-identical to the reference's PIL drawing.  The padding, grayscale, discs, outlines and trails run
as CUDA kernels (ct3_render_prepare / ct3_render_tracks, csrc/render.cu) on the device copy of the clip; the host only
computes colours ([T,N] numbers) and, with compensate_for_camera_motion, the per-frame camera offsets, exactly as the
reference does, and copies the finished frames back once.  mode="optical_flow" colours every (t, n) by its flow from
query_frame (flow_vis.flow_to_color); those colours come from a kernel too (ct3_render_flow_colors), so the tracks
never come to the host.  Every operation there is the reference's float64 one except atan2, the one IEEE leaves open
(numpy's own result depends on the CPU); a colour that depended on its last bits could differ by 1 (DESIGN.md §4.9.1).
On a host without a CUDA device the constructor raises NotImplementedError for this mode, as it has no host path.

Video may be on the host or the device, uint8 or float (other float dtypes are cast to float32 first); tracks and
visibility may be on either too.  matplotlib and imageio are imported only when a colour map or a video file is needed.
Not provided: gt_tracks (the reference's _draw_gt_tracks rebinds its own input inside the loop and fails for more than
one point, so it has no behaviour to match).
"""
from __future__ import annotations

import os
from typing import Optional

import numpy as np
import torch

from . import engine, ingest


def _get_cmap(name: str):
    import matplotlib
    try:
        return matplotlib.colormaps[name]
    except AttributeError:   # matplotlib < 3.5
        from matplotlib import cm
        return cm.get_cmap(name)


def read_video_from_path(path):
    """Frames [T,H,W,3] uint8 of a video file (imageio when installed, else OpenCV), or None when it cannot be read."""
    try:
        import imageio
    except ImportError:
        imageio = None
    if imageio is not None:
        try:
            reader = imageio.get_reader(path)
        except Exception as e:
            print("Error opening video file: ", e)
            return None
        return np.stack([np.array(im) for im in reader])
    try:
        import cv2
    except ImportError as e:
        raise ImportError("read_video_from_path needs imageio or opencv-python (cv2)") from e
    cap = cv2.VideoCapture(path)
    frames = []
    while cap.isOpened():
        ok, frame = cap.read()
        if not ok:
            break
        frames.append(cv2.cvtColor(frame, cv2.COLOR_BGR2RGB))
    cap.release()
    if not frames:
        print("Error opening video file: ", path)
        return None
    return np.stack(frames)


def _normalize(v, vmin, vmax):
    """plt.Normalize(vmin, vmax)(v) for finite values: (v - vmin) / (vmax - vmin) in float64, 0 when vmin == vmax."""
    v = np.asarray(v, dtype=np.float64)
    vmin, vmax = float(vmin), float(vmax)
    if vmin == vmax:
        return np.zeros_like(v)
    return (v - vmin) / (vmax - vmin)


def _cmap_rgb(cmap, values) -> np.ndarray:
    """cmap(v)[:3] for every v as float64 [n,3]: one vectorised call when the colour map takes arrays (matplotlib's
    do, with the same result per element), else one call per value as the reference makes."""
    values = np.asarray(values, dtype=np.float64)
    try:
        out = np.asarray(cmap(values), dtype=np.float64)
        if out.shape == (values.shape[0], 4) or out.shape == (values.shape[0], 3):
            return out[:, :3]
    except Exception:
        pass
    return np.array([np.asarray(cmap(float(v))[:3], dtype=np.float64) for v in values]).reshape(-1, 3)


def _device_for(*tensors) -> torch.device:
    for t in tensors:
        if isinstance(t, torch.Tensor) and t.is_cuda:
            return t.device
    if not torch.cuda.is_available():
        raise engine.EngineError("cotracker_b200's visualiser draws on CUDA only; no GPU is available")
    return torch.device("cuda", torch.cuda.current_device())


def _reject_crop(video, where: str):
    """TypeError for a `Crop`: drawing draws on whole frames; draw on the frame with `crop.to_frame(tracks)`."""
    if isinstance(video, ingest.Crop):
        raise TypeError(f"{where} draws on whole frames, not a Crop: pass the video and crop.to_frame(tracks)")


class Visualizer:
    def __init__(
        self,
        save_dir: str = "./results",
        grayscale: bool = False,
        pad_value: int = 0,
        fps: int = 10,
        mode: str = "rainbow",  # 'cool', 'optical_flow'
        linewidth: int = 2,
        show_first_frame: int = 10,
        tracks_leave_trace: int = 0,  # -1 for infinite
    ):
        if mode == "optical_flow" and not torch.cuda.is_available():
            # the colours of this mode exist only as a library kernel (no host flow_vis path), so say so at once
            raise NotImplementedError("mode='optical_flow' computes flow_vis's colour code on the GPU "
                                      "(ct3_render_flow_colors); no CUDA device is available")
        self.mode = mode
        self.save_dir = save_dir
        self._color_map = None   # resolved from matplotlib on first use unless a caller sets color_map
        self.show_first_frame = show_first_frame
        self.grayscale = grayscale
        self.tracks_leave_trace = tracks_leave_trace
        self.pad_value = pad_value
        self.linewidth = linewidth
        self.fps = fps

    @property
    def color_map(self):
        if self._color_map is None and self.mode in ("rainbow", "cool"):
            self._color_map = _get_cmap("gist_rainbow" if self.mode == "rainbow" else "cool")
        return self._color_map

    @color_map.setter
    def color_map(self, cmap):
        self._color_map = cmap

    def visualize(
        self,
        video: torch.Tensor,  # (B,T,C,H,W)
        tracks: torch.Tensor,  # (B,T,N,2)
        visibility: torch.Tensor = None,  # (B,T,N) or (B,T,N,1)
        gt_tracks: torch.Tensor = None,
        segm_mask: torch.Tensor = None,  # (B,1,H,W)
        filename: str = "video",
        writer=None,  # tensorboard SummaryWriter
        step: int = 0,
        query_frame=0,
        save_video: bool = True,
        compensate_for_camera_motion: bool = False,
        opacity: float = 1.0,
    ):
        ingest.reject_encoded_clip(video, "Visualizer.visualize")
        _reject_crop(video, "Visualizer.visualize")
        if gt_tracks is not None:
            raise NotImplementedError("gt_tracks is not provided (the reference cannot draw more than one of them)")
        if compensate_for_camera_motion:
            assert segm_mask is not None
        query_frame = self._query_frame(query_frame)
        if segm_mask is not None:
            coords = tracks[0, query_frame].round().long()
            segm_mask = segm_mask[0, query_frame][coords[:, 1].to(segm_mask.device), coords[:, 0].to(segm_mask.device)]
            segm_mask = segm_mask.long()
        dev = _device_for(video, tracks)
        frames = self._frames(video, dev, self.pad_value, self.grayscale)
        res_video = self._draw(frames, tracks, self.pad_value, visibility, segm_mask, query_frame,
                               compensate_for_camera_motion)
        if save_video:
            self.save_video(res_video, filename=filename, writer=writer, step=step)
        return res_video

    def save_video(self, video, filename, writer=None, step=0):
        if writer is not None:
            writer.add_video(filename, video.to(torch.uint8), global_step=step, fps=self.fps)
            return
        try:
            import imageio
        except ImportError as e:
            raise ImportError("Visualizer.save_video needs the imageio package (with imageio-ffmpeg for mp4)") from e
        os.makedirs(self.save_dir, exist_ok=True)
        wide_list = [wide[0].permute(1, 2, 0).cpu().numpy() for wide in video.unbind(1)]
        save_path = os.path.join(self.save_dir, f"{filename}.mp4")
        video_writer = imageio.get_writer(save_path, fps=self.fps)
        for frame in wide_list[2:-1]:   # the reference drops the first two frames and the last
            video_writer.append_data(frame)
        video_writer.close()
        print(f"Video saved to {save_path}")

    def draw_tracks_on_video(
        self,
        video: torch.Tensor,
        tracks: torch.Tensor,
        visibility: torch.Tensor = None,
        segm_mask: torch.Tensor = None,
        gt_tracks=None,
        query_frame=0,
        compensate_for_camera_motion=False,
        color_alpha: int = 255,
    ):
        """video (B,T,3,H,W) as drawn on (already padded), tracks (B,T,N,2) in its pixel coordinates, segm_mask [N]."""
        ingest.reject_encoded_clip(video, "Visualizer.draw_tracks_on_video")
        _reject_crop(video, "Visualizer.draw_tracks_on_video")
        if gt_tracks is not None:
            raise NotImplementedError("gt_tracks is not provided (the reference cannot draw more than one of them)")
        B, T, C, H, W = video.shape
        assert tracks.shape[-1] == 2
        assert C == 3
        dev = _device_for(video, tracks)
        frames = self._frames(video, dev, 0, False)
        return self._draw(frames, tracks, 0, visibility, segm_mask, self._query_frame(query_frame),
                          compensate_for_camera_motion)

    # ---- internals ----------------------------------------------------------------------------------------------
    @staticmethod
    def _query_frame(query_frame) -> int:
        if isinstance(query_frame, torch.Tensor):
            if query_frame.numel() != 1:
                raise NotImplementedError("a per-track query_frame tensor is not supported; pass one frame index")
            query_frame = query_frame.item()
        return int(query_frame)

    @staticmethod
    def _frames(video: torch.Tensor, dev, pad: int, grayscale: bool) -> torch.Tensor:
        """video [B,T,3,H,W] -> [T,H+2p,W+2p,3] uint8 on dev (pad with 255, optional grayscale, .byte())."""
        v = video[0]
        if v.dtype not in engine.FRAME_DTYPES:
            v = v.float()
        if v.device != dev:
            v = v.to(dev)
        return engine.render_prepare(v, pad, grayscale)

    def _colors(self, y_query: np.ndarray, y_first: np.ndarray, segm: Optional[np.ndarray], T: int) -> np.ndarray:
        """vector_colors of draw_tracks_on_video (visualizer.py:189-236) -> uint8 [T,N,3].  y_query / y_first: the
        truncated y of every track at query_frame / frame 0."""
        N = y_query.shape[0]
        if segm is None:
            if self.mode == "rainbow":
                rgb = _cmap_rgb(self.color_map, _normalize(y_query, y_query.min(), y_query.max())) * 255
                vc = np.repeat(rgb[None], T, axis=0)
            else:   # colour changes with time
                rgb = _cmap_rgb(self.color_map, [t / T for t in range(T)]) * 255
                vc = np.repeat(rgb[:, None], N, axis=1)
        elif self.mode == "rainbow":
            vc = np.zeros((T, N, 3))
            vc[:, segm <= 0, :] = 255
            fg = segm > 0
            ys = y_first[fg]
            rgb = _cmap_rgb(self.color_map, _normalize(ys, ys.min(), ys.max())) * 255
            vc[:, fg] = rgb[None]
        else:   # colour changes with segm class (float32, as the reference builds it)
            color = np.zeros((N, 3), dtype=np.float32)
            color[segm > 0] = np.array(self.color_map(1.0)[:3]) * 255.0
            color[segm <= 0] = np.array(self.color_map(0.0)[:3]) * 255.0
            vc = np.repeat(color[None], T, axis=0)
        # .astype(int) at draw time; PIL clips ink to 0..255
        return np.clip(np.asarray(vc).astype(np.int64), 0, 255).astype(np.uint8)

    def _draw(self, frames: torch.Tensor, tracks: torch.Tensor, pad: int, visibility, segm_mask, query_frame: int,
              compensate: bool) -> torch.Tensor:
        dev = frames.device
        T, Hp, Wp, _ = frames.shape
        N = tracks.shape[2]
        trace = max(-1, int(self.tracks_leave_trace))   # every negative value draws every earlier step unblended
        # tracks + pad_value in the tracks' own dtype, as the reference adds it, then fp32 for the kernel (which
        # truncates like .long()); other dtypes are truncated here first
        tp = tracks[0] + pad
        if tp.dtype != torch.float32:
            tp = torch.where(torch.isfinite(tp.double()), torch.trunc(tp.double()), tp.double()).float()
        pts = tp.to(dev).contiguous()
        segm = None if segm_mask is None else torch.as_tensor(segm_mask).reshape(-1).cpu().numpy()
        if self.mode == "optical_flow":   # every (t, n) has its own colour: computed where the tracks are
            colors = engine.render_flow_colors(pts, query_frame)
        else:   # only [N] slices of the tracks come to the host
            y_query = (tracks[0, query_frame, :, 1] + pad).long().cpu().numpy()
            y_first = (tracks[0, 0, :, 1] + pad).long().cpu().numpy()
            colors = torch.from_numpy(self._colors(y_query, y_first, segm, T)).to(dev)
        vis = None
        if visibility is not None:
            vis = (visibility[0].reshape(T, N) != 0).to(device=dev, dtype=torch.uint8).contiguous()
        draw_mask = alphas = diff = None
        S = (min(trace, T - 1) if trace > 0 else T - 1) if trace != 0 else 0
        if trace > 0:
            a = np.zeros((T, max(S, 1), 2))
            for t in range(query_frame + 1, T):
                first = max(0, t - trace)
                L = t - first + 1
                for s in range(L - 1):
                    alpha = (s / L) ** 2
                    a[t, s] = (alpha, 1 - alpha)
            alphas = torch.from_numpy(a).to(dev)
        if compensate:
            draw_mask = torch.from_numpy((segm > 0).astype(np.uint8)).to(dev)
            if trace != 0:
                bg = segm <= 0
                tl = (tracks[0] + pad).long()[:, torch.from_numpy(bg).to(tracks.device)].cpu().numpy()   # [T, Nbg, 2]
                d = np.zeros((T, S + 1, 2))
                for t in range(query_frame + 1, T):
                    first = max(0, t - trace) if trace >= 0 else 0
                    d[t, : t - first + 1] = (tl[first: t + 1] - tl[t: t + 1]).mean(1)
                diff = torch.from_numpy(d).to(dev)
        engine.render_tracks(frames, pts, colors, radius=int(self.linewidth * 2), linewidth=int(self.linewidth),
                             trail=trace, query_frame=query_frame, visible=vis, draw_mask=draw_mask, alphas=alphas,
                             diff=diff)
        if self.show_first_frame > 0:
            idx = torch.tensor([0] * self.show_first_frame + list(range(1, T)), device=dev)
            frames = frames.index_select(0, idx)
        return frames.cpu().permute(0, 3, 1, 2)[None]
