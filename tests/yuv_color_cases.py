"""YUV colour test helpers: an int64 torch restatement of the integer formula of ct3_prepare_frames_yuv_fmt
(include/ct3_b200.h) for every layout, matrix and range; its float64 definition; and a packer for the layouts that
tests/yuv_cases.py does not cover (4:2:2 / 4:4:4 planar and the 16-bit containers).

Arithmetic on torch.uint16 is not supported, so every sample is widened to int64 before any is done."""
import torch

import yuv_cases

# layout -> (container dtype, significant bits n, MSB-aligned, family, chroma x shift, chroma y shift)
FORMATS = {
    "nv12": (torch.uint8, 8, False, "semi", 1, 1),
    "i420": (torch.uint8, 8, False, "planar", 1, 1),
    "yuyv": (torch.uint8, 8, False, "packed", 1, 0),
    "yuv422p": (torch.uint8, 8, False, "planar", 1, 0),
    "yuv444p": (torch.uint8, 8, False, "planar", 0, 0),
    "p010": (torch.uint16, 10, True, "semi", 1, 1),
    "p016": (torch.uint16, 16, True, "semi", 1, 1),
    "yuv420p10": (torch.uint16, 10, False, "planar", 1, 1),
    "yuv422p10": (torch.uint16, 10, False, "planar", 1, 0),
    "yuv444p10": (torch.uint16, 10, False, "planar", 0, 0),
}
NEW_LAYOUTS = tuple(k for k in FORMATS if k not in yuv_cases.LAYOUTS)
# Kr, Kb in units of 1e-4 (the library's integer derivation) and as the floats of the float64 definition
MATRICES = {"bt601": (2990, 1140), "bt709": (2126, 722), "bt2020": (2627, 593)}
KR_KB = {"bt601": (0.299, 0.114), "bt709": (0.2126, 0.0722), "bt2020": (0.2627, 0.0593)}
COLOURS = [(m, f) for m in MATRICES for f in (False, True)]
DERIVED = [c for c in COLOURS if c != ("bt601", False)]
Q = 48                                         # the fraction bits of every derived coefficient
CV2 = (1220542, 1673527, 852492, 409993, 2116026)   # cy, crv, cgv, cgu, cbu of cv2's BT.601 limited range, Q20


def coeffs(matrix, full_range, bits):
    """The integer conversion of (matrix, range) at `bits` significant bits: offsets, the floor of y, the shift and
    the coefficients cy, crv, cgv, cgu, cbu (ct3_b200.h)."""
    s = 1 << (bits - 8)
    if matrix == "bt601" and not full_range:
        return dict(yoff=16 * s, ylo=0, coff=128 * s, shift=20 + bits - 8, c=CV2)
    kr, kb = MATRICES[matrix]
    kg = 10000 - kr - kb
    if full_range:
        yoff, coff, dy, dc = 0, 1 << (bits - 1), (1 << bits) - 1, (1 << bits) - 1
    else:
        yoff, coff, dy, dc = 16 * s, 128 * s, 219 * s, 224 * s

    def q(num, den):                           # num / den * 2^Q rounded half up, exactly
        return (num * (1 << (Q + 1)) + den) // (2 * den)

    c = (q(255, dy), q(510 * (10000 - kr), 10000 * dc), q(510 * kr * (10000 - kr), 10000 * kg * dc),
         q(510 * kb * (10000 - kb), 10000 * kg * dc), q(510 * (10000 - kb), 10000 * dc))
    return dict(yoff=yoff, ylo=-yoff, coff=coff, shift=Q, c=c)


def convert(Y, U, V, matrix="bt601", full_range=False, bits=8):
    """Samples (int64 tensors of one shape [..., H, W]) -> uint8 RGB [..., 3, H, W] by the integer formula."""
    k = coeffs(matrix, full_range, bits)
    cy, crv, cgv, cgu, cbu = k["c"]
    y = (Y - k["yoff"]).clamp(min=k["ylo"]) * cy
    u, v = U - k["coff"], V - k["coff"]
    half = 1 << (k["shift"] - 1)
    r = (y + crv * v + half) >> k["shift"]
    g = (y - cgv * v - cgu * u + half) >> k["shift"]
    b = (y + cbu * u + half) >> k["shift"]
    return torch.stack([r, g, b], dim=-3).clamp(0, 255).to(torch.uint8)


def exact(Y, U, V, matrix, full_range, bits):
    """The float64 definition before rounding: 255 * (R', G', B') [..., 3] of float64 samples Y, U, V."""
    kr, kb = KR_KB[matrix]
    kg = 1.0 - kr - kb
    if full_range:
        n = float((1 << bits) - 1)
        y, cb, cr = Y / n, (U - (1 << (bits - 1))) / n, (V - (1 << (bits - 1))) / n
    else:
        s = float(1 << (bits - 8))
        y, cb, cr = (Y - 16 * s) / (219 * s), (U - 128 * s) / (224 * s), (V - 128 * s) / (224 * s)
    r = y + 2 * (1 - kr) * cr
    g = y - (2 * kr * (1 - kr) / kg) * cr - (2 * kb * (1 - kb) / kg) * cb
    b = y + 2 * (1 - kb) * cb
    return 255 * torch.stack([r, g, b], dim=-1)


def round_exact(x):
    """clamp(floor(x + 0.5), 0, 255) and the distance of x from the nearest rounding tie k + 0.5."""
    t = x + 0.5
    return torch.floor(t).clamp(0, 255), (t - torch.round(t)).abs()


def frame_hw(layout, shape):
    """(H, W) of frames [..., R, W] (planar, semi-planar) or [..., H, W, 2] (yuyv)."""
    if layout == "yuyv":
        return shape[-3], shape[-2]
    xs, ys = FORMATS[layout][4:6]
    per = 2 + 2 * (2 >> ys) // (1 << xs)         # rows per 2 luma rows: 3 (4:2:0), 4 (4:2:2), 6 (4:4:4)
    return shape[-2] * 2 // per, shape[-1]


def samples(layout, data):
    """Container values -> n-bit samples, int64: v >> (16 - n) when MSB-aligned, else v & (2^n - 1)."""
    _, bits, msb, *_ = FORMATS[layout]
    d = data.long()
    return (d >> (16 - bits)) if msb else d & ((1 << bits) - 1)


def planes(layout, data):
    """Frames [..., <one frame>] -> Y, U, V int64 samples [..., H, W], each chroma sample repeated over the pixels
    that share it."""
    family, xs, ys = FORMATS[layout][3:6]
    d = samples(layout, data)
    if family == "semi":
        return yuv_cases.planes("nv12", d)
    if family == "packed":
        return yuv_cases.planes("yuyv", d)
    H, W = frame_hw(layout, data.shape)
    lead = d.shape[:-2]
    flat = d.reshape(*lead, -1)
    ch, cw = H >> ys, W >> xs
    Y = flat[..., :H * W].reshape(*lead, H, W)
    U = flat[..., H * W:H * W + ch * cw].reshape(*lead, ch, cw)
    V = flat[..., H * W + ch * cw:H * W + 2 * ch * cw].reshape(*lead, ch, cw)
    U, V = (c.repeat_interleave(1 << ys, dim=-2).repeat_interleave(1 << xs, dim=-1) for c in (U, V))
    return Y, U, V


def yuv_to_rgb(layout, data, matrix="bt601", full_range=False):
    """The uint8 RGB [..., 3, H, W] the formula gives for frames of `layout`."""
    return convert(*planes(layout, data), matrix, full_range, FORMATS[layout][1])


def pack(layout, Y, U, V):
    """Integer container values Y [..., H, W] and U, V [..., H >> ys, W >> xs] (any integer dtype) -> frames of
    `layout` in its container dtype."""
    dtype, _, _, family, xs, ys = FORMATS[layout]
    Y, U, V = Y.long(), U.long(), V.long()
    if family == "semi":
        out = yuv_cases.pack("nv12", Y, U, V)
    elif family == "packed":
        out = yuv_cases.pack("yuyv", Y.to(torch.uint8), U.to(torch.uint8), V.to(torch.uint8))
    else:
        W = Y.shape[-1]
        lead = Y.shape[:-2]
        out = torch.cat([Y.reshape(*lead, -1), U.reshape(*lead, -1), V.reshape(*lead, -1)], -1).reshape(*lead, -1, W)
    return out.to(dtype).contiguous()


def containers(layout, S, junk=None):
    """n-bit samples S (int64) -> container values: S << (16 - n) for MSB-aligned layouts, S for the others.  `junk`
    (int64 of S's shape) fills the bits the format ignores: the low 16 - n bits (MSB-aligned) or the bits above n."""
    _, bits, msb, *_ = FORMATS[layout]
    if bits == 8 or bits == 16:
        return S
    if msb:
        return (S << (16 - bits)) | (0 if junk is None else junk & ((1 << (16 - bits)) - 1))
    return S | (0 if junk is None else (junk & ((1 << (16 - bits)) - 1)) << bits)


def random_frames(layout, lead, H, W, seed, junk=True):
    """Random frames [*lead, <one frame>] of `layout`, every sample value equally likely, with random ignored bits
    (junk=True) or zero ones."""
    g = torch.Generator().manual_seed(seed)
    _, bits, _, _, xs, ys = FORMATS[layout]
    cshape = (H, W >> 1) if layout == "yuyv" else (H >> ys, W >> xs)

    def plane(shape):
        S = torch.randint(0, 1 << bits, tuple(lead) + shape, generator=g)
        J = torch.randint(0, 1 << 16, tuple(lead) + shape, generator=g)      # drawn either way: same samples
        return containers(layout, S, J if junk else None)

    return pack(layout, plane((H, W)), plane(cshape), plane(cshape))


def as_frames(layout, rgb_like_video):
    """A uint8 RGB clip [..., 3, H, W] (e.g. texture_video) -> frames of `layout` whose Y, U, V samples are its R, G, B
    channels scaled to n bits (subsampled chroma takes the top-left sample of its block): a moving, textured clip."""
    _, bits, _, _, xs, ys = FORMATS[layout]
    v = rgb_like_video.long() << (bits - 8)
    v = v | (v >> 8) if bits > 8 else v                      # fill the low bits so that they are not all zero
    Y = v[..., 0, :, :]
    if layout == "yuyv":
        U, V = v[..., 1, :, 0::2], v[..., 2, :, 1::2]
    else:
        U, V = v[..., 1, ::1 << ys, ::1 << xs], v[..., 2, ::1 << ys, ::1 << xs]
    return pack(layout, *(containers(layout, c) for c in (Y, U, V)))


def coeff_error_bound(bits):
    """The largest |error| of the Q-bit coefficients against the exact ones, over samples of `bits` bits (255 X
    units): half a unit in the last place of each of at most three coefficients times its largest operand."""
    return 0.5 * 2.0 ** -Q * ((1 << bits) + 2 * (1 << (bits - 1)))

