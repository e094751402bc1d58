"""YUV test helpers: a torch int64 restatement of cv2's YUV -> RGB conversion (the contract of ct3_prepare_frames_yuv,
include/ct3_b200.h), and synthetic YUV clips packed in each layout."""
import torch

LAYOUTS = ("nv12", "i420", "yuyv")


def frame_hw(layout, data):
    """(H, W) of frames [..., H*3/2, W] (nv12, i420) or [..., H, W, 2] (yuyv)."""
    if layout == "yuyv":
        return data.shape[-3], data.shape[-2]
    return data.shape[-2] // 3 * 2, data.shape[-1]


def planes(layout, data):
    """data uint8 frames [..., <one frame>] -> Y, U, V int64 [..., H, W], each chroma sample repeated over the pixels
    that share it."""
    H, W = frame_hw(layout, data)
    lead = data.shape[:-3] if layout == "yuyv" else data.shape[:-2]
    if layout == "nv12":
        Y = data[..., :H, :]
        uv = data[..., H:, :]
        U, V = uv[..., 0::2], uv[..., 1::2]
    elif layout == "i420":
        flat = data.reshape(*lead, -1)
        q = (H // 2) * (W // 2)
        Y = flat[..., :H * W].reshape(*lead, H, W)
        U = flat[..., H * W:H * W + q].reshape(*lead, H // 2, W // 2)
        V = flat[..., H * W + q:H * W + 2 * q].reshape(*lead, H // 2, W // 2)
    else:
        Y = data[..., 0]
        U, V = data[..., 0::2, 1], data[..., 1::2, 1]
    if layout != "yuyv":
        U, V = (c.repeat_interleave(2, dim=-2) for c in (U, V))
    U, V = (c.repeat_interleave(2, dim=-1) for c in (U, V))
    return Y.long(), U.long(), V.long()


def yuv_to_rgb(layout, data):
    """The RGB cv2.cvtColor(frame, COLOR_YUV2RGB_*) gives, in Q20 integers: uint8 [..., 3, H, W]."""
    Y, U, V = planes(layout, data)
    y = (Y - 16).clamp(min=0) * 1220542
    u, v = U - 128, V - 128
    r = (y + 1673527 * v + (1 << 19)) >> 20
    g = (y - 852492 * v - 409993 * u + (1 << 19)) >> 20
    b = (y + 2116026 * u + (1 << 19)) >> 20
    return torch.stack([r, g, b], dim=-3).clamp(0, 255).to(torch.uint8)


def pack(layout, Y, U, V):
    """Planes uint8 Y [..., H, W] and U, V [..., H/2, W/2] (4:2:0) or [..., H, W/2] (yuyv) -> frames in `layout`."""
    H, W = Y.shape[-2:]
    lead = Y.shape[:-2]
    if layout == "nv12":
        return torch.cat([Y, torch.stack([U, V], dim=-1).reshape(*lead, H // 2, W)], dim=-2)
    if layout == "i420":
        return torch.cat([Y.reshape(*lead, -1), U.reshape(*lead, -1), V.reshape(*lead, -1)], -1).reshape(*lead, -1, W)
    out = torch.empty(*lead, H, W, 2, dtype=torch.uint8)
    out[..., 0] = Y
    out[..., 0::2, 1] = U
    out[..., 1::2, 1] = V
    return out


def yuv_video(layout, B, T, H, W, seed=0):
    """A moving synthetic clip (texture_video's texture) as uint8 YUV frames [B,T,...] in `layout`, on the host."""
    from cotracker_b200.synthetic import texture_video
    clips = [texture_video(T, H, W, seed=seed + b, shift=(1 + (seed + b) % 3, 2))[0].to(torch.uint8) for b in range(B)]
    v = torch.stack(clips)                                   # [B,T,3,H,W]
    Y = v[:, :, 0]
    if layout == "yuyv":
        U, V = v[:, :, 1, :, 0::2], v[:, :, 2, :, 1::2]
    else:
        U, V = v[:, :, 1, 0::2, 0::2], v[:, :, 2, 1::2, 1::2]
    return pack(layout, Y, U.contiguous(), V.contiguous()).contiguous()
