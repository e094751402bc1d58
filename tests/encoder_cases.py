"""CNN encoder test helpers (CPU-importable): decoders for the split operands, float64 restatements of every link of
ct3_encoder (as ct3_encoder_trace returns them), their per-element bounds, a restatement of the conv3x3_tc tile choice
and the case generator.

Operands.  A split operand [rows, 2C] holds hi = bf16_rn(v) in columns 0..C-1 and lo = bf16_rn(v - hi) in C..2C-1
(split2 in csrc/common.cuh; v - hi is exact in fp32), so `split_f32` restates it bit for bit from the fp32 value v.
Every weight is rounded to 16 significant bits before packing (`round16`): its bf16 hi + lo is then the weight
exactly, and the float64 references multiply what the kernel multiplies without reading the packed layout.  Each link
is restated from the kernel's own input to that link (the previous link of the trace), so its error is the kernel's
own, and its bound below is that error per element.  u = 2^-24, the fp32 unit roundoff.

Bounds (err = |got - want|, want in float64):
  conv3x3_tc, stride-2 GEMMs  y = sum x w + b over the split operand x = hi + lo and w = w_hi + w_lo.  The kernel runs
      three products (hi hi, hi lo, lo hi) and drops lo lo: at most L = sum |x_lo| |w_lo| (<= 2^-16 S).  With
      S = sum |x| |w|, each of the n = 3 K / 16 wgmma steps (K = taps * Cp: 9 * 64 .. 9 * 448, or Cp for the 1x1/2)
      adds into the fp32 accumulator with one rounding of at most 2u of the magnitudes involved (2u: the tensor
      core's adder need not round to nearest), so <= (n + 1) 2u S; the bias add and store <= 2u (S + |b|).
      bound = L + (n + 1) 2u S + 2u (S + |b|).
  stem (7x7/2, fp32 SIMT)  147 fmaf in one chain from 0, then + b: bound = (147 + 1) u S + 2u (S + |b|).
  gathers  pure copies with zero fill: bit for bit.
  InstanceNorm stats  fp64 sums of the fp32 values (each thread HW / 256 rows, then 8 lanes, then 32 splits: depth
      nd = HW / 256 + 48), var = E[y^2] - mean^2 in fp64, then mean and rstd = 1 / sqrt(var + eps) rounded to fp32:
      mean: u |mean| + nd 2^-53 E|y|;   rstd: rstd (u + 2^-53 + (nd + 4) 2^-53 E[y^2] / (var + eps)).
      (The last term is the fp64 cancellation; with |mean| / std = 1e4 it is still ~1e-6 relative, where fp32 sums
      would be off by more than the variance itself.)  The ratio sits near 1 by construction: the fp32 rounding is
      all the error there is, and half an ulp reaches u |x| for values just above a power of two.
  norm_act (with the kernel's own stats m, r)  a = relu((y - m) r): one fp32 subtract and one multiply, <= 2u
      |y - m| r; mode 1 adds x (fp32, one more rounding); mode 2 adds (x_d - m_d) r_d (two roundings, possibly one
      fused multiply-add).  bound = 4u (|y - m| r + |x| + |x_d - m_d| r_d) with the terms the mode has.  The split
      outputs are compared bit for bit with split_f32 of the kernel's own fp32 output; where the link has no fp32
      output (mode 0 into a split, instnorm_relu_split) the fp32 value relu((y - m) r) is restated exactly (a
      subtract and a multiply cannot fuse) and its split compared bit for bit.
  resize + concat  where the stage map is H4 x W4 the kernel copies: bit for bit.  Elsewhere the source index is
      (float)(hs - 1) / (float)(H4 - 1) * y in fp32, as the kernel and ATen compute it; at that index the fp32 blend
      (2 x 2 taps, weights 1 - l and l, about 6 roundings) is within 6u sum |v_ij| of the float64 blend, and hi + lo of
      the split is within half an ulp of lo (bf16) of the fp32 blend.  That half ulp is attained by construction (lo
      is the nearest bf16 of the remainder) and dominates, so this ratio sits near 1, like the stats'.  Against the exact-coordinate F.interpolate in float64 a coordinate term is added: the index
      error |dy| (|dx|) times D, the largest difference of vertically (horizontally) adjacent texels of the channel.
  conv3 (1x1 256 -> 128 GEMM)  as the GEMMs, K = 256.
  pyramid  level 0: x / sqrt(max(sum x^2, 1e-12)) of the kernel's conv3 rows: 4 products per lane, a 5-level warp
      sum, sqrtf and a division, all rounded: 16u |want|.  Levels 1..3: the 2 x 2 mean of the kernel's level l - 1,
      three adds then an exact * 0.25: u sum |v|.
  whole encoder  against O.encoder + O.normalized_pyramid in float64: the existing cuDNN tolerance, 2e-5.
"""
import math
from dataclasses import dataclass

import torch
import torch.nn.functional as F

U = 2.0 ** -24
EPS = 1e-5                                   # InstanceNorm2d's eps (the oracle's float64)
EPS32 = float(torch.tensor(EPS, dtype=torch.float32))   # the kernels' 1e-5f, added in fp64
STAGE_C = (64, 96, 128, 128)     # real channels per stage
STAGE_CP = (64, 128, 128, 128)   # carried channels: stage 1's 96 padded to 128
CAT_C, CAT_CP, MID, LATENT = 416, 448, 256, 128


# ---------------------------------------------------------------------------------------------------------------------
# operands
def round16(w):
    """w rounded to 16 significant bits (fp32): bf16 hi + bf16 lo of it is w exactly"""
    m, e = torch.frexp(w.double())
    return torch.ldexp(torch.round(m * 65536.0) / 65536.0, e).float()


def split_f32(v):
    """fp32 v -> (hi, lo) bf16 as split2 writes them"""
    v = v.float()
    hi = v.to(torch.bfloat16)
    return hi, (v - hi.float()).to(torch.bfloat16)


def planes(t, C):
    """split operand [rows, 2C] bf16 -> (hi, lo) float64 [rows, C]"""
    t = t.reshape(-1, 2 * C)
    return t[:, :C].double(), t[:, C:].double()


def same_bits(a, b):
    """bf16 tensors equal as values (+0 and -0 alike)"""
    return a.shape == b.shape and bool((a.float() == b.float()).all())


def stage_hw(H, W):
    hw = [((H - 1) // 2 + 1, (W - 1) // 2 + 1)]
    for _ in range(3):
        hw.append(((hw[-1][0] - 1) // 2 + 1, (hw[-1][1] - 1) // 2 + 1))
    return hw


def nchw(x_nhwc):
    return x_nhwc.permute(0, 3, 1, 2)


def nhwc(x_nchw):
    return x_nchw.permute(0, 2, 3, 1).contiguous()


# ---------------------------------------------------------------------------------------------------------------------
# weights
def weight_names():
    n = ["conv1.weight", "conv1.bias"]
    for s in range(1, 5):
        for u in range(2):
            for c in (1, 2):
                n += [f"layer{s}.{u}.conv{c}.weight", f"layer{s}.{u}.conv{c}.bias"]
        if s > 1:
            n += [f"layer{s}.0.downsample.0.weight", f"layer{s}.0.downsample.0.bias"]
    return n + ["conv2.weight", "conv2.bias", "conv3.weight", "conv3.bias"]


def conv_shape(name):
    """[Cout, Cin, k, k] of a weight"""
    if name.startswith("conv1"):
        return (64, 3, 7, 7)
    if name.startswith("conv2"):
        return (MID, CAT_C, 3, 3)
    if name.startswith("conv3"):
        return (LATENT, MID, 1, 1)
    s = int(name[5]) - 1
    cout = STAGE_C[s]
    if ".downsample." in name:
        return (cout, STAGE_C[s - 1], 1, 1)
    cin = STAGE_C[s - 1] if (s > 0 and name[7] == "0" and ".conv1." in name) else (64 if s == 0 else cout)
    return (cout, cin, 3, 3)


# Engineered output channels (layer, channel), made through the weights:
#   ZERO   zero weights, bias 0.3: a constant map, variance 0, eps decides rstd and relu(IN) is exactly 0
#   DOMINATED  weights * 1e-4, bias 1: |mean| / std ~ 1e4, where one-pass fp32 statistics lose the variance
#   NEGATIVE   bias -8 (~8 std): every value before IN is negative
ZERO = (("conv1", 2), ("layer1.0.conv1", 5), ("layer2.0.conv1", 7), ("layer3.1.conv2", 9), ("conv2", 3))
DOMINATED = (("conv1", 4), ("layer1.1.conv2", 9), ("layer3.0.downsample.0", 11), ("layer2.0.conv2", 17), ("conv2", 7))
NEGATIVE = (("conv1", 6), ("layer1.0.conv2", 13), ("layer2.1.conv1", 15), ("layer4.0.conv1", 21), ("conv2", 11))


def encoder_weights(seed, engineered=False):
    """seeded fnet weights {name: fp32 [Cout, Cin, k, k] / [Cout]} rounded to 16 significant bits, He-scaled so
    activations keep unit scale through the stages"""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name in weight_names():
        if name.endswith(".bias"):
            continue
        shape = conv_shape(name)
        fan = shape[1] * shape[2] * shape[3]
        w = torch.randn(shape, generator=g, dtype=torch.float64) * math.sqrt(2.0 / fan)
        b = torch.randn(shape[0], generator=g, dtype=torch.float64) * 0.1
        layer = name[:-len(".weight")]
        if engineered:
            for (l, c) in ZERO:
                if l == layer:
                    w[c] = 0
                    b[c] = 0.3
            for (l, c) in DOMINATED:
                if l == layer:
                    w[c] *= 1e-4
                    b[c] = 1.0
            for (l, c) in NEGATIVE:
                if l == layer:
                    b[c] = -8.0
        sd[name] = round16(w)
        sd[layer + ".bias"] = round16(b)
    return sd


# ---------------------------------------------------------------------------------------------------------------------
# restatements (float64; NHWC in and out, like the trace)
def conv_ref(x, w, b, stride, pad, cout_pad=None):
    """x [T,h,w,Cx] (Cx >= Cin; extra channels are padding), w [Cout,Cin,k,k] -> (y, S) [T,ho,wo,cout_pad]"""
    cin = w.shape[1]
    xs = nchw(x[..., :cin].double())
    w64 = w.double()
    y = F.conv2d(xs, w64, b.double(), stride=stride, padding=pad)
    S = F.conv2d(xs.abs(), w64.abs(), None, stride=stride, padding=pad)
    y, S = nhwc(y), nhwc(S)
    if cout_pad is not None and cout_pad > y.shape[-1]:
        y, S = F.pad(y, (0, cout_pad - y.shape[-1])), F.pad(S, (0, cout_pad - S.shape[-1]))
    return y, S


def w_lo(w):
    """the lo plane of a packed weight (w - bf16(w)) in float64"""
    w = w.float()
    return (w - w.to(torch.bfloat16).float()).double()


def conv_split_ref(hi, lo, w, b, stride, pad, cout_pad=None):
    """a convolution of the split operand hi + lo ([T,h,w,Cp] float64 each) -> (want, bound) for the tensor-core
    kernels: L + (n + 1) 2u S + 2u (S + |b|), n = 3 K / 16, K = k * k * Cp"""
    cp = hi.shape[-1]
    want, S = conv_ref(hi + lo, w, b, stride, pad, cout_pad)
    L, _ = conv_ref(lo.abs(), w_lo(w).abs(), torch.zeros_like(b), stride, pad, cout_pad)
    n = 3 * w.shape[2] * w.shape[3] * cp // 16
    bb = F.pad(b.double().abs(), (0, want.shape[-1] - b.shape[0]))
    return want, L + (n + 1) * 2 * U * S + 2 * U * (S + bb)


def stem_ref(frames, w, b):
    """conv1 7x7/2 pad 3 of frames [T,3,H,W] -> (want, bound) [T,h0,w0,64]"""
    want, S = conv_ref(nhwc(frames.double()), w, b, 2, 3)
    return want, (147 + 1) * U * S + 2 * U * (S + b.double().abs())


def gather_ref(x_split, T, h, w, C, taps):
    """stride-2 gather of a split operand [T*h*w, 2C] -> [T*ho*wo, 2*taps*C] bf16 (zero outside the map), bit for bit"""
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    x = x_split.reshape(T, h, w, 2, C)
    xp = torch.zeros(T, h + 2, w + 2, 2, C, dtype=x.dtype, device=x.device)
    xp[:, 1:h + 1, 1:w + 1] = x
    offs = [(ky, kx) for ky in range(3) for kx in range(3)] if taps == 9 else [(1, 1)]
    cols = [xp[:, ky:ky + 2 * ho - 1:2, kx:kx + 2 * wo - 1:2] for ky, kx in offs]   # each [T,ho,wo,2,C]
    return torch.stack(cols, dim=4).reshape(T * ho * wo, 2 * taps * C)


def gemm_weight(w, cin_p, cout_pad):
    """conv weight [Cout,Cin,k,k] -> GEMM rows [cout_pad, k*k*cin_p] (tap-major K, zero padded), float64"""
    cout, cin, kh, kw = w.shape
    m = F.pad(w.double().permute(0, 2, 3, 1), (0, cin_p - cin))
    return F.pad(m.reshape(cout, kh * kw * cin_p), (0, 0, 0, cout_pad - cout))


def gemm_ref(rows_split, w, b, cin_p, cout_pad):
    """y = rows w^T + b of a split operand [R, 2K] (K = k*k*cin_p) -> (want, bound) [R, cout_pad]"""
    K = w.shape[2] * w.shape[3] * cin_p
    hi, lo = planes(rows_split, K)
    wm = gemm_weight(w, cin_p, cout_pad)
    wl = gemm_weight(w_lo(w), cin_p, cout_pad)
    bb = F.pad(b.double(), (0, cout_pad - b.shape[0]))
    want = (hi + lo) @ wm.T + bb
    S = (hi + lo).abs() @ wm.abs().T
    L = lo.abs() @ wl.abs().T
    n = 3 * K // 16
    return want, L + (n + 1) * 2 * U * S + 2 * U * (S + bb.abs())


def stats_ref(y):
    """y [T,h,w,C] fp32 (the kernel's input) -> (mean, rstd, bound_mean, bound_rstd) float64 [T,C]"""
    T, C = y.shape[0], y.shape[-1]
    v = y.double().reshape(T, -1, C)
    HW = v.shape[1]
    mean = v.mean(1)
    var = ((v - mean[:, None]) ** 2).mean(1)
    rstd = 1.0 / torch.sqrt(var + EPS32)
    nd = HW / 256 + 48
    e = 2.0 ** -53
    bm = U * mean.abs() + nd * e * v.abs().mean(1)
    br = rstd * (U + e + (nd + 4) * e * (v * v).mean(1) / (var + EPS32))
    return mean, rstd, bm, br


def norm_act_ref(mode, y, stats, x=None, stats_d=None):
    """norm_act with the kernel's own stats [T,C,2] -> (want, bound) [T,h,w,C] float64"""
    T, C = y.shape[0], y.shape[-1]
    st = stats.double().reshape(T, 1, 1, C, 2)
    d = (y.double() - st[..., 0]) * st[..., 1]
    a = d.clamp_min(0)
    mag = d.abs()
    if mode == 1:
        a = (x.double() + a).clamp_min(0)
        mag = mag + x.double().abs()
    elif mode == 2:
        sd = stats_d.double().reshape(T, 1, 1, C, 2)
        xd = (x.double() - sd[..., 0]) * sd[..., 1]
        a = (xd + a).clamp_min(0)
        mag = mag + xd.abs()
    return a, 4 * U * mag


def norm0_f32(y, stats):
    """relu((y - m) r) in fp32 exactly as norm_act mode 0 and instnorm_relu_split compute it"""
    T, C = y.shape[0], y.shape[-1]
    st = stats.float().reshape(T, 1, 1, C, 2)
    return torch.clamp_min((y.float() - st[..., 0]) * st[..., 1], 0.0)


def split_rows(v):
    """fp32 [..., C] -> split operand [rows, 2C] bf16"""
    C = v.shape[-1]
    hi, lo = split_f32(v.reshape(-1, C))
    return torch.cat([hi, lo], dim=1)


def source_index(hs, H, exact=False):
    """the align_corners source coordinate of output rows 0..H-1 from a map of hs rows: fp32 as the kernel and ATen
    compute it, or exact (float64)"""
    y = torch.arange(H, dtype=torch.float64)
    if H <= 1:
        return y * 0
    if exact:
        return y * (hs - 1) / (H - 1)
    s = torch.tensor(float(hs - 1), dtype=torch.float32) / torch.tensor(float(H - 1), dtype=torch.float32)
    return (s * y.float()).double()


def blend(src, fy, fx):
    """bilinear blend of src [T,hs,ws,C] float64 at source rows fy [H] and columns fx [W] -> [T,H,W,C], plus the
    weighted sum of |taps| (the blend error scale)"""
    hs, ws = src.shape[1], src.shape[2]
    y0 = fy.floor().long().clamp(0, hs - 1)
    x0 = fx.floor().long().clamp(0, ws - 1)
    y1, x1 = (y0 + 1).clamp(max=hs - 1), (x0 + 1).clamp(max=ws - 1)
    ly, lx = (fy - y0.double()).to(src.device), (fx - x0.double()).to(src.device)
    y0, y1, x0, x1 = (t.to(src.device) for t in (y0, y1, x0, x1))
    ly, lx = ly[None, :, None, None], lx[None, None, :, None]
    v00, v01 = src[:, y0][:, :, x0], src[:, y0][:, :, x1]
    v10, v11 = src[:, y1][:, :, x0], src[:, y1][:, :, x1]
    out = (1 - ly) * ((1 - lx) * v00 + lx * v01) + ly * ((1 - lx) * v10 + lx * v11)
    return out, v00.abs() + v01.abs() + v10.abs() + v11.abs()


def half_ulp_bf16(lo):
    """half an ulp of each bf16 value (0 for 0): hi + lo of a split lies within it of the fp32 value split"""
    _, e = torch.frexp(lo.double())
    return torch.where(lo.double() == 0, torch.zeros_like(e, dtype=torch.float64), torch.ldexp(torch.ones_like(lo.double()), e - 9))


def resize_ref(srcs, H4, W4, exact=False, split=True):
    """the resize + concat operand's values from the four fp32 stage outputs [T,hs,ws,Cp] -> (want, bound, copied)
    float64 [T,H4,W4,448]; copied [448] marks channels of directly copied stages.  exact=False: at the fp32 source
    index (the blend bound); exact=True: F.interpolate's float64 coordinates, bound with the coordinate term.
    split=False leaves out the split's 2^-17 |v| for a caller that bounds it from the kernel's lo plane."""
    outs, bounds, copied = [], [], []
    for s, src in enumerate(srcs):
        c = STAGE_C[s]
        x = src[..., :c].double()
        hs, ws = x.shape[1], x.shape[2]
        if hs == H4 and ws == W4:
            outs.append(x)
            bounds.append(torch.zeros_like(x))
            copied += [True] * c
            continue
        fy, fx = source_index(hs, H4), source_index(ws, W4)
        v, mag = blend(x, fy, fx)
        bnd = 6 * U * mag + (2.0 ** -17 * v.abs() if split else 0)
        if exact:
            ey, ex = source_index(hs, H4, True), source_index(ws, W4, True)
            v = nhwc(F.interpolate(nchw(x), (H4, W4), mode="bilinear", align_corners=True))
            Dy = (x[:, 1:] - x[:, :-1]).abs().amax(dim=(1, 2)) if hs > 1 else x.new_zeros(x.shape[0], c)
            Dx = (x[:, :, 1:] - x[:, :, :-1]).abs().amax(dim=(1, 2)) if ws > 1 else x.new_zeros(x.shape[0], c)
            dy = (fy - ey).abs().to(x.device)[None, :, None, None]
            dx = (fx - ex).abs().to(x.device)[None, None, :, None]
            bnd = bnd + dy * Dy[:, None, None] + dx * Dx[:, None, None]
        outs.append(v)
        bounds.append(bnd)
        copied += [False] * c
    want = F.pad(torch.cat(outs, dim=-1), (0, CAT_CP - CAT_C))
    bound = F.pad(torch.cat(bounds, dim=-1), (0, CAT_CP - CAT_C))
    return want, bound, torch.tensor(copied + [True] * (CAT_CP - CAT_C))


def l2norm_ref(x):
    """level 0 of the pyramid from conv3's rows [..., 128] -> (want, bound)"""
    x = x.double()
    want = x / torch.sqrt((x * x).sum(-1, keepdim=True).clamp_min(1e-12))
    return want, 16 * U * want.abs()


def pool_ref(prev):
    """level l from the kernel's level l - 1 [T,h,w,128] -> (want, bound) [T,h/2,w/2,128]"""
    T, h, w, C = prev.shape
    p = prev.double()[:, :h // 2 * 2, :w // 2 * 2].reshape(T, h // 2, 2, w // 2, 2, C)
    return p.mean(dim=(2, 4)), U * p.abs().sum(dim=(2, 4))


# ---------------------------------------------------------------------------------------------------------------------
# the encoder's schedule: which link feeds which (the trace's names, engine.encoder_trace_links)
def units(H, W):
    """[(stage, unit, stride, h, w, h_in, w_in)] in launch order"""
    hw = stage_hw(H, W)
    out = []
    for s in range(4):
        for u in range(2):
            stride = 2 if (s > 0 and u == 0) else 1
            hin, win = hw[s - 1] if stride == 2 else hw[s]
            out.append((s, u, stride, hw[s][0], hw[s][1], hin, win))
    return out


def unit_input(s, u):
    """the trace link a unit reads: the previous unit's output (fp32 and split)"""
    if s == 0 and u == 0:
        return "stem.out"
    if u == 1:
        return f"layer{s + 1}.0.out"
    return f"layer{s}.1.out"


def chain64(sd, frames):
    """the float64 encoder chained from the link restatements alone (no kernel values): the pyramid levels
    [T,h,w,128], for comparison with O.encoder + O.normalized_pyramid"""
    def inorm(y):
        v = y.reshape(y.shape[0], -1, y.shape[-1])
        m = v.mean(1)
        r = 1.0 / torch.sqrt(((v - m[:, None]) ** 2).mean(1) + EPS)
        return torch.stack([m, r], -1)

    H, W = frames.shape[-2:]
    y, _ = stem_ref(frames, sd["conv1.weight"], sd["conv1.bias"])
    x, _ = norm_act_ref(0, y, inorm(y))
    outs = []
    for s, u, stride, h, w, _, _ in units(H, W):
        p = f"layer{s + 1}.{u}"
        cp = STAGE_CP[s]
        zero = torch.zeros_like(x)
        if stride == 2:
            yy, _ = conv_split_ref(x, zero, sd[p + ".conv1.weight"], sd[p + ".conv1.bias"], 2, 1, cp)
            yd, _ = conv_split_ref(x, zero, sd[p + ".downsample.0.weight"], sd[p + ".downsample.0.bias"], 2, 0, cp)
        else:
            yy, _ = conv_split_ref(x, zero, sd[p + ".conv1.weight"], sd[p + ".conv1.bias"], 1, 1, cp)
        a, _ = norm_act_ref(0, yy, inorm(yy))
        y2, _ = conv_split_ref(a, torch.zeros_like(a), sd[p + ".conv2.weight"], sd[p + ".conv2.bias"], 1, 1, cp)
        if stride == 2:
            x, _ = norm_act_ref(2, y2, inorm(y2), yd, inorm(yd))
        else:
            x, _ = norm_act_ref(1, y2, inorm(y2), x)
        if u == 1:
            outs.append(x)
    cat, _, _ = resize_ref(outs, H // 4, W // 4, exact=True)
    y, _ = conv_split_ref(cat, torch.zeros_like(cat), sd["conv2.weight"], sd["conv2.bias"], 1, 1)
    a, _ = norm_act_ref(0, y, inorm(y))
    f, _ = conv_split_ref(a, torch.zeros_like(a), sd["conv3.weight"], sd["conv3.bias"], 1, 0)
    lv = [l2norm_ref(f)[0]]
    for _ in range(3):
        lv.append(pool_ref(lv[-1])[0])
    return lv


# ---------------------------------------------------------------------------------------------------------------------
# dispatch restatement and cases
def pick_tile(H, W):
    """conv3x3_tc's tile (tw, th), tw * th = 128, wasting the fewest MMA rows on an H x W map (csrc/enc_front.cu)"""
    best, tile = -1, None
    w = 128
    while w >= 8:
        h = 128 // w
        cover = ((W + w - 1) // w) * w * ((H + h - 1) // h) * h
        if best < 0 or cover < best:
            best, tile = cover, (w, h)
        w //= 2
    return tile


def conv_launches(H, W):
    """every conv3x3_tc launch of an H x W frame -> [(h, w, C, Cout, BN, tw)]"""
    hw = stage_hw(H, W)
    out = []
    for s in range(4):
        cp = STAGE_CP[s]
        for _ in range(3 if s > 0 else 4):
            out.append((hw[s][0], hw[s][1], cp, cp, 128 if cp % 128 == 0 else 64, pick_tile(*hw[s])[0]))
    out.append((H // 4, W // 4, CAT_CP, MID, 128, pick_tile(H // 4, W // 4)[0]))
    return out


def resize_branches(H, W):
    """per stage: 'copy' where the stage map is H/4 x W/4, else 'interpolate'"""
    return ["copy" if hw == (H // 4, W // 4) else "interpolate" for hw in stage_hw(H, W)]


@dataclass(frozen=True)
class Case:
    name: str
    T: int
    H: int
    W: int
    engineered: bool = True
    seed: int = 1


# every link of every case is checked per element; the whole-encoder comparison runs on the plain ones
CASES = [
    Case("production", 1, 384, 512),
    Case("copy_stage", 1, 100, 132),          # stage 1 is 25 x 33 = H4 x W4: the resize copies it
    Case("all_interpolated", 1, 98, 130),     # 49x65, 25x33, 13x17, 7x9 -> 24 x 32
    Case("tall", 1, 520, 32),                 # 130 x 8 and 65 x 4 maps: tw = 8
    Case("wide", 1, 32, 520),
    Case("minimum", 1, 32, 32),               # 16x16, 8x8, 4x4, 2x2 -> 8 x 8
    Case("min_rows", 2, 32, 72),              # 2 x N stage-3 maps
    Case("min_cols", 1, 72, 32),              # N x 2
]
WHOLE_CASES = [Case("production_plain", 1, 384, 512, engineered=False, seed=2),
               Case("all_interpolated_plain", 2, 98, 130, engineered=False, seed=3)]
CHUNK_CASES = [(17, 64, 96), (33, 48, 64)]
