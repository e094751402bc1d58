"""Correlation-stage test helpers (CPU-importable): a float64 gather sampler for the support features and the
correlation volume, the operands each correlation kernel multiplies ("what the kernel reads"), per-element error
bounds, an fp32 restatement of the shift pattern of the correlate-then-interpolate kernels, and the case generator.

Reference.  A sample of level l at offset (a, b) of track coordinate c (fp32, level-0 feature units) sits at
x = c_x 2^-l + (a - 3), y = c_y 2^-l + (b - 3), evaluated exactly in float64 and clamped to [0, size - 1] (grid_sample,
align_corners=True, padding_mode="border"); its taps are floor(x) and min(floor(x) + 1, size - 1) with weights
(1 - fr, fr).  support64 gives the sampled vectors [49, N, 128] (p = a*7 + b), volume64 the volume [T, N, 2401] with
element (a*7 + b)*49 + k: the sampled vector dotted with support vector k.  Both run on any device, in track chunks.

Operands.  What each kernel multiplies, rebuilt in torch (`operands`), as (texel plane, support plane) pairs whose
float64 volumes add up to what the kernel computes before its own rounding:
  corr_tc3  one fp16 texel plane (the scratch copy ct3_corr_sample leaves behind) times the fp16 split support
            hi + lo (split2_h) with prec.corr = 2, times hi only with prec.corr = 1;
  corr_tc2  bf16 texel planes Fh, Fl and bf16 split support Sh, Sl, three products: Fh (Sh + Sl) + Fl Sh (the dropped
            Fl Sl term is in the formula, not in the bound);
  corr_tc, simt  the fp32 pyramid and the fp32 support.

Bounds (err = |got - want| per element, want in float64 on the operands above; u = 2^-24; S = the float64 volume of
|F| . |S| over the taps actually read, with the same tap weights; LAM = 4 is the margin of random-walk sums):
  accumulation  acc(S, n) = LAM sqrt(n) 2^-23 S: n fp32 additions, each off by at most one ulp of a partial sum <= S,
                adding like a random walk.  corr_tc3: n = 8 k16 blocks per product (128 channels); corr_tc2 and corr_tc:
                3 products x 8 + the add of the two accumulator halves; simt: 128 sequential FMAs.
  blend / sampling  6 u S: each of the x and y two-tap blends (or the four-tap bilinear sample of corr_tc / simt) is
                an FMA and a product, <= 2u of the weighted sum of |taps|; 1 - fr is exact but for x < 1/2 (<= u of
                itself); the second order terms are covered by the margin 6 over 5.
  split operands  corr_tc / simt have no decoded planes: corr_tc splits the fp32 sample and the support into bf16
                hi + lo (2^-18 each) and drops lo . lo (2^-18): 3 2^-18 S.
  coordinates   x is evaluated in fp32 (c 2^-l is exact, the add rounds): the exact float64 difference of the
                reference at the fp32 positions and at the exact ones, i.e. |dx| times the difference of the two tap
                correlations per axis (a rounding across a texel centre included).
  output        split bf16 volume: + 2^-17 |want| (hi + lo of an fp32 value).  fp16 volume: the fp32 result lies in
                [want - e, want + e], so its fp16 rounding lies in [rn16(want - e), rn16(want + e)] (rounding is
                monotone, subnormals included); the ratio is the distance to want over the distance to that end.
  prepare_pyramid  level 0: sum of 128 squares (4 FMAs per lane + 5 shuffle adds: 9u), sqrt and divide, correctly
                rounded: 8u |want|.  Level l: the 2x2 mean of level l - 1 (3 adds, exact * 0.25) propagates the
                bounds below it as their mean and adds 4u mean|want|.
  sample_support  the bilinear sample in fp32 on the kernel's own pyramid: 6u S + the coordinate term, with
                S = the sample of |F|; the accumulate path adds u |start + want| for its one add.
"""
import math

import numpy as np
import torch

from test_gpu_tokens import loop_branch

LEVELS, P, C, VOL, VOL_PAD = 4, 49, 128, 2401, 2432
U = 2.0 ** -24
LAM = 4.0
f32 = np.float32


# ---------------------------------------------------------------------------------------------------------------------
# fp32 restatement of the shift pattern (csrc/corr_tc3.cu: box_origin8, tap_weights)
def box_origin8(c, size):
    """c float32 array (level units), size >= 8 -> (origin, d) int64 arrays: the 8-texel box holding every tap of
    the 7 samples around c and the shift of the tap pattern relative to the interior one."""
    cc = np.minimum(np.maximum(c, f32(-16)), f32(size + 16)).astype(f32)
    base = np.floor(cc).astype(np.int64) - 3
    origin = np.clip(base, 0, size - 8)
    return origin, np.clip(base - origin, -7, 7)


def tap_weights(c, a, size, origin, d):
    """Sample a (0..6) of c as the kernel sees it -> (branch, u, w, s0, s1, i0, i1, fr).  branch 1: the border-clamped
    taps (s0, s1) of grid_sample are the box entries (i0, i1) = (clamp07(a + d), clamp07(a + d + 1)), weights
    (1 - fr, fr); 2: c + offset rounded up to an integer in fp32, the sample is entry i1 alone, weights (0, 1);
    0: neither (the kernel traps)."""
    x = np.minimum(np.maximum((c + f32(a - 3)).astype(f32), f32(0)), f32(size - 1)).astype(f32)
    xf = np.floor(x)
    x0 = xf.astype(np.int64)
    fr = (x - xf).astype(f32)
    s0 = np.clip(x0 - origin, 0, 7)
    s1 = np.where(fr > 0, np.clip(np.minimum(x0 + 1, size - 1) - origin, 0, 7), s0)
    i0, i1 = np.clip(a + d, 0, 7), np.clip(a + d + 1, 0, 7)
    direct = (s0 == i0) & ((fr == 0) | (s1 == i1))
    rounded = (~direct) & (fr == 0) & (s0 == i1)
    branch = np.where(direct, 1, np.where(rounded, 2, 0))
    u = np.where(direct, f32(1) - fr, f32(0)).astype(f32)
    w = np.where(direct, fr, np.where(rounded, f32(1), f32(0))).astype(f32)
    return branch, u, w, s0, s1, i0, i1, fr


def level_sizes(H4, W4):
    return [(H4 >> l, W4 >> l) for l in range(LEVELS)]


def shift_coverage(coords, H4, W4):
    """coords [T, N, 2] float32 -> set of (level, axis, d) and of (level, axis, tap_weights branch) reached at the
    levels where the correlate-then-interpolate kernels run (every level >= 8x8)."""
    c = np.asarray(coords, dtype=f32)
    shifts, branches = set(), set()
    if min(min(hw) for hw in level_sizes(H4, W4)) < 8:
        return shifts, branches
    for l, (H, W) in enumerate(level_sizes(H4, W4)):
        for axis, size in ((0, W), (1, H)):
            cl = (c[..., axis] * f32(2.0 ** -l)).astype(f32).reshape(-1)
            origin, d = box_origin8(cl, size)
            shifts |= {(l, axis, int(v)) for v in np.unique(d)}
            for a in range(7):
                br = tap_weights(cl, a, size, origin, d)[0]
                branches |= {(l, axis, int(v)) for v in np.unique(br)}
    return shifts, branches


# ---------------------------------------------------------------------------------------------------------------------
# branch map: which kernel / volume format / products a call runs (loop_branch of test_gpu_tokens.py)
OPTION_SETS = [{"corr": corr, "prec.corr": pc, "prec.fc1": pf} for corr in (0, 1, 2) for pc in (1, 2, 3)
               for pf in (1, 2, 3)]


def corr_branch(opts, T, H4, W4):
    b = loop_branch(T, H4, W4, opts.get("corr", 0), opts.get("prec.corr", 2), opts.get("prec.fc1", 3))
    return b["kernel"], b["volume"], b["corr_products"]


# every reachable (kernel, volume format, corr products)
REACHABLE = {("corr_tc3", "split", 2), ("corr_tc3", "fp16", 2), ("corr_tc3", "split", 1), ("corr_tc3", "fp16", 1),
             ("corr_tc2", "split", 3), ("corr_tc2", "fp16", 3), ("corr_tc", "split", 3), ("simt", "split", 3)}


def branch_options(T, H4, W4):
    """One option set per distinct branch reachable at this map size, in a fixed order."""
    out = {}
    for o in OPTION_SETS:
        out.setdefault(corr_branch(o, T, H4, W4), o)
    return [(k, out[k]) for k in sorted(out)]


# ---------------------------------------------------------------------------------------------------------------------
# float64 reference
def _taps(pos, size):
    p = pos.clamp(0, size - 1)
    i0 = p.floor()
    fr = p - i0
    i0 = i0.long()
    return i0, (i0 + 1).clamp(max=size - 1), fr


def positions(coords, l, fp32=False):
    """coords [..., 2] float32 (level-0 units) -> (x, y) [..., 7] float64 sample positions of level l, unclamped:
    exactly c 2^-l + (a - 3), or (fp32=True) rounded to fp32 as the kernels evaluate it."""
    off = torch.arange(-3, 4, device=coords.device)
    if fp32:
        c = coords.float() * (2.0 ** -l)
        return (c[..., 0:1] + off.float()).double(), (c[..., 1:2] + off.float()).double()
    c = coords.double() * (2.0 ** -l)
    return c[..., 0:1] + off.double(), c[..., 1:2] + off.double()


def sample64(fmap, frames, x, y):
    """Bilinear border-clamped samples.  fmap [F, H, W, C] float64 channels-last; frames: long, broadcastable to
    x.shape[:-1]; x, y [..., 7] positions -> [..., 49, C], p = a*7 + b (a: x offset, b: y offset)."""
    _, H, W, _ = fmap.shape
    x0, x1, fx = _taps(x, W)
    y0, y1, fy = _taps(y, H)
    X0, X1, FX = x0[..., :, None], x1[..., :, None], fx[..., :, None, None]
    Y0, Y1, FY = y0[..., None, :], y1[..., None, :], fy[..., None, :, None]
    f = frames[..., None, None]
    out = ((1 - FY) * (1 - FX)) * fmap[f, Y0, X0] + ((1 - FY) * FX) * fmap[f, Y0, X1] \
        + (FY * (1 - FX)) * fmap[f, Y1, X0] + (FY * FX) * fmap[f, Y1, X1]
    return out.reshape(*out.shape[:-3], P, fmap.shape[-1])


def support64(fmap, qframes, qcoords, l, fp32=False):
    """fmap [T, H, W, C] float64; qframes [N] long (clamped to [0, T-1] as the kernel does); qcoords [N, 2] float32
    -> [49, N, C]."""
    x, y = positions(qcoords, l, fp32)
    f = qframes.clamp(0, fmap.shape[0] - 1)
    return sample64(fmap, f, x, y).transpose(0, 1)


def _chunk(T):
    return max(1, 2048 // T)


def volume64(fmap, support, coords, l, tracks=None, fp32=False):
    """fmap [T, H, W, C] float64 (frame t of the clip); support [49, N, C] float64; coords [T, N, 2] float32
    -> [T, n, 2401] float64 over `tracks` (default all N)."""
    T, N = coords.shape[:2]
    idx = torch.arange(N) if tracks is None else torch.as_tensor(tracks)
    frames = torch.arange(T, device=fmap.device)[:, None]
    out = []
    for i in range(0, len(idx), _chunk(T)):
        sel = idx[i:i + _chunk(T)].to(coords.device)
        x, y = positions(coords[:, sel], l, fp32)
        f = sample64(fmap, frames, x, y)                                  # [T, n, 49, C]
        s = support[:, sel.to(support.device)].transpose(0, 1)           # [n, 49(k), C]
        out.append(torch.einsum("tnpc,nkc->tnpk", f, s).reshape(T, len(sel), VOL))
    return torch.cat(out, dim=1)


# ---------------------------------------------------------------------------------------------------------------------
# what each kernel reads
def split16(x, dtype):
    """fp32 x -> (hi, lo) of the 16-bit split (split2 / split2_h): hi = rn(x), lo = rn(x - hi), as float64."""
    hi = x.to(dtype)
    lo = (x - hi.float()).to(dtype)
    return hi.double(), lo.double()


def scratch_planes(scratch, kernel, T, H4, W4):
    """The pyramid copy ct3_corr_sample leaves in its scratch -> per level [T, H, W, C] 16-bit planes: [fp16] for
    corr_tc3, [bf16 hi, bf16 lo] for corr_tc2 (level l starts at 16-bit element 2 * off[l], as in the fp32 pyramid)."""
    s16 = scratch.view(torch.int16)
    out, off = [], 0
    for H, W in level_sizes(H4, W4):
        n = T * H * W * C
        if kernel == "corr_tc3":
            out.append([s16[2 * off:2 * off + n].view(torch.float16).view(T, H, W, C)])
        else:
            out.append([s16[2 * off + i * n:2 * off + (i + 1) * n].view(torch.bfloat16).view(T, H, W, C)
                        for i in range(2)])
        off += n
    return out


def operands(kernel, products, planes_l, support_l):
    """-> [(texel plane, support plane)] float64 pairs of one level whose volumes sum to what the kernel multiplies.
    planes_l: the level's decoded scratch planes (patch kernels) or [fp32 level] (corr_tc, simt); support_l [49, N, C]
    fp32 with dead tracks already zeroed."""
    if kernel == "corr_tc3":
        sh, sl = split16(support_l, torch.float16)
        return [(planes_l[0].double(), sh + sl if products == 2 else sh)]
    if kernel == "corr_tc2":
        sh, sl = split16(support_l, torch.bfloat16)
        return [(planes_l[0].double(), sh + sl), (planes_l[1].double(), sh)]
    return [(planes_l[0].double(), support_l.double())]


ACC_N = {"corr_tc3": None, "corr_tc2": 25, "corr_tc": 25, "simt": 128}


def acc(S, n):
    return LAM * math.sqrt(n) * 2.0 ** -23 * S


def volume_want_bound(kernel, products, pairs, coords, l, tracks=None):
    """-> (want, e) [T, n, 2401] float64: the float64 volume of the operand pairs and the bound of the kernel's fp32
    result before the output format (accumulation, blend / sampling, split operands, coordinates)."""
    want = sum(volume64(F, S, coords, l, tracks) for F, S in pairs)
    S = sum(volume64(F.abs(), S.abs(), coords, l, tracks) for F, S in pairs)
    coord = (sum(volume64(F, S, coords, l, tracks, fp32=True) for F, S in pairs) - want).abs()
    n = 8 * products if kernel == "corr_tc3" else ACC_N[kernel]
    e = acc(S, n) + 6 * U * S + coord
    if kernel in ("corr_tc", "simt"):
        e = e + 3 * 2.0 ** -18 * S
    return want, e


def ratio_split(got, want, e):
    """got: decoded hi + lo (float64).  err / (e + 2^-17 |want|), 0 where both are 0."""
    err = (got - want).abs()
    bound = e + 2.0 ** -17 * want.abs()
    return torch.where(err == 0, torch.zeros_like(err), err / bound)


def ratio_fp16(got, want, e):
    """got: the fp16 plane (float64).  <= 1 iff got lies in [rn16(want - e), rn16(want + e)]."""
    lo = (want - e).float().half().double()
    hi = (want + e).float().half().double()
    up = torch.where(hi > want, (got - want) / (hi - want), torch.full_like(got, math.inf))
    dn = torch.where(lo < want, (want - got) / (want - lo), torch.full_like(got, math.inf))
    r = torch.where(got > want, up, torch.where(got < want, dn, torch.zeros_like(got)))
    return r


# ---------------------------------------------------------------------------------------------------------------------
# prepare_pyramid / sample_support references and bounds
def pyramid64(fmaps):
    """fmaps [T, C, H, W] float32 -> per level (want [T, H, W, C] float64, bound)."""
    f = fmaps.double()
    ss = (f * f).sum(dim=1, keepdim=True)
    lvl = f / torch.sqrt(ss.clamp(min=1e-12))
    want = [lvl]
    bound = [8 * U * lvl.abs()]
    for _ in range(LEVELS - 1):
        want.append(torch.nn.functional.avg_pool2d(want[-1], 2, stride=2))
        bound.append(torch.nn.functional.avg_pool2d(bound[-1], 2, stride=2)
                     + 4 * U * torch.nn.functional.avg_pool2d(want[-2].abs(), 2, stride=2))
    return [(w.permute(0, 2, 3, 1), b.permute(0, 2, 3, 1)) for w, b in zip(want, bound)]


def support_want_bound(level, qframes, qcoords, l):
    """level [T, H, W, C] fp32 (the kernel's pyramid) -> (want, e) [49, N, C] float64."""
    F = level.double()
    want = support64(F, qframes, qcoords, l)
    S = support64(F.abs(), qframes, qcoords, l)
    coord = (support64(F, qframes, qcoords, l, fp32=True) - want).abs()
    return want, 6 * U * S + coord


# ---------------------------------------------------------------------------------------------------------------------
# case generator
MAP_SIZES = [(64, 64), (64, 72), (96, 128), (24, 32), (25, 33)]


def _ulps(v, k):
    """float32 array v moved k ulps (k < 0: down)."""
    out = np.asarray(v, dtype=f32).copy()
    for _ in range(abs(k)):
        out = np.nextafter(out, f32(np.sign(k) * np.inf)).astype(f32)
    return out


def make_case(T, H4, W4, seed, classes=("sweep", "centre", "far", "moving")):
    """-> (coords [T, N, 2] float32, track_valid [N] uint8, labels [N] of the track classes):
      sweep   level coordinates s = k + frac (k integer from -7 to 3 and from size - 6 to size + 3, frac random per frame)
              at every level: reaches every shift d in [-7, 7] on both axes where the patch kernels run;
      centre  texel centres at every level (0, 1, size - 1, interior), exactly and 1..3 ulps to either side (the
              fp32 add c + offset then rounds onto or off the integer: both tap_weights branches);
      far     just outside the map, and +-1e6 / +-3e9 (beyond int32: the +-16 pre-clamp), each axis alone and both;
      moving  a fresh position in [-20, size + 20] every frame, so the two frames of a tile have different shifts.
    Every 7th track is dead (track_valid = 0)."""
    rng = np.random.default_rng(seed)
    tracks, labels = [], []

    def add(label, xy):   # xy [T, 2] or [2]
        tracks.append(np.broadcast_to(np.asarray(xy, dtype=f32), (T, 2)).copy())
        labels.append(label)

    sizes = level_sizes(H4, W4)
    if "sweep" in classes:
        for l, (H, W) in enumerate(sizes):
            kx = list(range(-7, 4)) + list(range(W - 6, W + 4))
            ky = list(range(-7, 4)) + list(range(H - 6, H + 4))
            ky = ky[::-1] + ky[: max(0, len(kx) - len(ky))]
            for i, k in enumerate(kx):
                fr = rng.uniform(0, 1, (T, 2)).astype(f32)
                s = np.stack([k + fr[:, 0], ky[i % len(ky)] + fr[:, 1]], axis=-1)
                add("sweep", (s * 2.0 ** l).astype(f32))
    if "centre" in classes:
        for l, (H, W) in enumerate(sizes):
            for sx, sy in ((0, 0), (1, H - 1), (W - 1, 0), (W - 1, H - 1), (W // 2, H // 2 + 1)):
                base = np.array([sx, sy], dtype=f32) * f32(2.0 ** l)
                for k in (0, -1, 1, -2, 2, -3, 3):
                    add("centre", _ulps(base, k))
    if "far" in classes:
        W, H = W4, H4
        for xy in ((-0.75, H / 2), (W - 0.25, -1.5), (W + 3.5, H + 0.5), (-1e6, 5.0), (1e6, -1e6), (3e9, 7.25),
                   (-3e9, 3e9), (10.5, -3e9)):
            add("far", xy)
    if "moving" in classes:
        for _ in range(24):
            add("moving", rng.uniform([-20, -20], [W4 + 20, H4 + 20], (T, 2)).astype(f32))
    coords = torch.from_numpy(np.stack(tracks, axis=1))
    valid = torch.ones(coords.shape[1], dtype=torch.uint8)
    valid[3::7] = 0
    return coords, valid, labels


# (case id, T, map size, classes): the map sizes at the dispatch edges with every class, odd T (a last tile of one
# frame), T = 1, T = 2 (one full tile), T = 60, N = 1
CASES = [(f"edges-{H4}x{W4}", 7, H4, W4, ("sweep", "centre", "far", "moving")) for H4, W4 in MAP_SIZES] + [
    ("t60", 60, 96, 128, ("far", "moving")),
    ("t1", 1, 64, 64, ("sweep", "far", "moving")),
    ("t2", 2, 64, 72, ("moving",)),
    ("n1", 5, 64, 72, ()),
]


def case_inputs(case, seed=0):
    """-> (coords, track_valid, labels, T, H4, W4).  The N = 1 case is one moving track."""
    name, T, H4, W4, classes = case
    if not classes:
        rng = np.random.default_rng(seed + 99)
        coords = torch.from_numpy(rng.uniform([-20, -20], [W4 + 20, H4 + 20], (T, 1, 2)).astype(f32))
        return coords, torch.ones(1, dtype=torch.uint8), ["moving"], T, H4, W4
    coords, valid, labels = make_case(T, H4, W4, seed + sum(map(ord, name)), classes)
    return coords, valid, labels, T, H4, W4


def features(T, H4, W4, seed):
    """Seeded raw feature maps [T, 128, H4, W4] fp32 (prepare_pyramid normalises them)."""
    g = torch.Generator().manual_seed(seed)
    return torch.randn(T, C, H4, W4, generator=g) * 2.5


def unit_support(N, seed):
    """Seeded unit support vectors [4, 49, N, 128] fp32."""
    g = torch.Generator().manual_seed(seed)
    s = torch.randn(LEVELS, P, N, C, generator=g)
    return s / s.norm(dim=-1, keepdim=True)
