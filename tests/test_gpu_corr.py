"""The correlation stage on its own against float64 (tests/corr_cases.py derives the reference and the per-element
bounds): prepare_pyramid, sample_support, and every correlation kernel x precision mode x volume format that
loop_branch can reach, on the case generator's cases, plus the headline shape.

Each correlation case checks, besides the bound: the scratch pyramid copy equals torch's rounding of the fp32 pyramid
bit for bit (the format's rounding, kept out of the bound: the decoded planes feed the reference), dead tracks give
exact zeros, the K padding is zero (volume_planes), and sentinel guard rows past the volume are untouched.  The worst
err/bound per (kernel, format, corr products, level, track class) is printed (`corr-worst`).  On an H100 80GB HBM3 at
a 700 W power limit: split volumes corr_tc3 0.61-0.77, corr_tc2 0.55-0.61, corr_tc 0.26-0.32, simt 0.16-0.24; every
fp16 volume 1.0 and sample_support 1.0 (0.99 accumulating), prepare_pyramid 0.32-0.38; the headline sample 0.64.  The
ratios at 1 are attained by construction, not loose: an fp16 volume element is the end of its rounding interval, and
the kernel's fp32 sample position is exactly the rounding the coordinate term accounts for.  Each of these mutations
fails this file: corr_tc3 on its one-product path while prec.corr = 2 (ratio 60), frame 0's shift and weights for
frame 1 of a tile, tap weights rounded to bf16 (both outside the fp16 rounding interval), and the fp16 pyramid copy
rounded toward zero (the format check).
"""
import time

import pytest
import torch

import corr_cases as K

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
OPTION_DEFAULTS = {"corr": 0, "prec.corr": 2, "prec.fc1": 3}
SENTINEL = 0x7FC1          # a NaN as bf16 and as fp16: no finite input makes a kernel write it
GUARD_ROWS = 16


@pytest.fixture(scope="module")
def eng():
    from cotracker_b200 import engine
    engine.lib()
    return engine


def _set(eng, opts):
    for k, v in opts.items():
        eng.set_option(k, v)


def _restore(eng):
    for k, v in OPTION_DEFAULTS.items():
        eng.set_option(k, v)


RATIOS = {}


def _note(key, r):
    RATIOS[key] = max(RATIOS.get(key, 0.0), r)


# ---------------------------------------------------------------------------------------------------------------------
# prepare_pyramid / sample_support
def _scaled_fmaps(T, H4, W4, seed):
    """Raw features with per-texel scales 1e-6 .. 1e3, one zero texel (the 1e-12 clamp) and one texel whose squared
    norm is below 1e-12."""
    g = torch.Generator().manual_seed(seed)
    f = torch.randn(T, K.C, H4, W4, generator=g)
    scale = 10.0 ** (torch.rand(T, 1, H4, W4, generator=g) * 9 - 6)
    f = f * scale
    f[0, :, 0, 0] = 0.0
    f[-1, :, H4 - 1, W4 - 1] *= 1e-8 / f[-1, :, H4 - 1, W4 - 1].norm()
    return f


@pytest.mark.parametrize("T,H4,W4", [(60, 96, 128), (3, 25, 33), (2, 67, 45)])
def test_prepare_pyramid_float64(eng, T, H4, W4):
    fmaps = _scaled_fmaps(T, H4, W4, seed=T + H4)
    pyr = eng.prepare_pyramid(fmaps.to(DEV))
    levels = eng.pyramid_levels(pyr, T, H4, W4)
    worst = 0.0
    for l, (want, bound) in enumerate(K.pyramid64(fmaps.to(DEV))):
        err = (levels[l].double() - want).abs()
        r = float(torch.where(err == 0, torch.zeros_like(err), err / bound).max())
        worst = max(worst, r)
        assert r <= 1.0, (l, r)
    assert bool((levels[0][0, 0, 0] == 0).all())
    _note(("prepare_pyramid", f"{T}x{H4}x{W4}"), worst)


def test_sample_support_float64(eng):
    """96 x 128, T = 60, hundreds of queries on every coordinate class, query frames spread over the clip; then the
    online accumulate path on a non-trivial buffer and mask."""
    T, H4, W4 = 60, 96, 128
    coords, _, labels, *_ = K.case_inputs(("support", 1, H4, W4, ("sweep", "centre", "far", "moving")), seed=1)
    qc = coords[0].contiguous()
    N = qc.shape[0]
    g = torch.Generator().manual_seed(2)
    qf = torch.randint(0, T, (N,), generator=g)
    qf[:2] = torch.tensor([0, T - 1])
    pyr = eng.prepare_pyramid(K.features(T, H4, W4, seed=3).to(DEV))
    levels = eng.pyramid_levels(pyr, T, H4, W4)
    qf_d, qc_d = qf.to(torch.int32).to(DEV), qc.to(DEV)
    got = eng.sample_support(pyr, T, H4, W4, qf_d, qc_d)
    start = torch.randn(K.LEVELS, K.P, N, K.C, generator=g).to(DEV) * 3
    mask = (torch.rand(N, generator=g) < 0.4).to(torch.uint8)
    acc = eng.sample_support(pyr, T, H4, W4, qf_d, qc_d, support=start.clone(), accumulate_mask=mask.to(DEV))
    sel = mask.bool().to(DEV)
    assert N >= 200 and 0 < int(mask.sum()) < N
    for l in range(K.LEVELS):
        want, e = K.support_want_bound(levels[l], qf.to(DEV), qc_d, l)
        err = (got[l].double() - want).abs()
        r = float(torch.where(err == 0, torch.zeros_like(err), err / e).max())
        _note(("sample_support", l), r)
        assert r <= 1.0, (l, r)
        s = start[l].double()
        err = (acc[l].double() - (s + want))[:, sel].abs()
        e_acc = (e + K.U * (s + want).abs())[:, sel]
        r = float(torch.where(err == 0, torch.zeros_like(err), err / e_acc).max())
        _note(("sample_support_accumulate", l), r)
        assert r <= 1.0, (l, r)
        assert torch.equal(acc[l][:, ~sel], start[l][:, ~sel]), "unmasked rows must be untouched"


# ---------------------------------------------------------------------------------------------------------------------
# correlation kernels
def _run_corr(eng, opts, pyr, H4, W4, support, valid, coords, vol, scratch):
    """corr_sample under `opts` into the caller's buffers -> decoded planes [P, N*T*4, 2401] (decoded while the
    options hold: the format and element order depend on them)."""
    T, N, _ = coords.shape
    _set(eng, opts)
    try:
        eng.corr_sample(pyr, H4, W4, support, valid, coords, scratch=scratch, vol=vol)
        planes = eng.volume_planes(vol[:N * T * K.LEVELS], T, N, H4, W4)
        torch.cuda.synchronize()
    finally:
        _restore(eng)
    return planes


def _written(vol, rows, fmt):
    """-> (written 16-bit view, the rest of the buffer): an fp16 volume fills the front rows * 2432 elements."""
    flat = vol.view(torch.int16).reshape(-1)
    n = rows * (K.VOL_PAD if fmt == "fp16" else 2 * K.VOL_PAD)
    return flat[:n], flat[n:]


def _check_format(scratch, kernel, pyr_levels, T, H4, W4):
    """The scratch pyramid copy is torch's round-to-nearest of the fp32 pyramid, bit for bit."""
    planes = K.scratch_planes(scratch, kernel, T, H4, W4)
    for l, lv in enumerate(pyr_levels):
        if kernel == "corr_tc3":
            assert torch.equal(planes[l][0].view(torch.int16), lv.half().view(torch.int16)), ("fp16 texels", l)
        else:
            hi = lv.bfloat16()
            lo = (lv - hi.float()).bfloat16()
            assert torch.equal(planes[l][0].view(torch.int16), hi.view(torch.int16)), ("bf16 hi texels", l)
            assert torch.equal(planes[l][1].view(torch.int16), lo.view(torch.int16)), ("bf16 lo texels", l)
    return planes


def _check_levels(branch, planes, scratch_planes, pyr_levels, support, valid, coords, labels, tracks, tag):
    """Every level of the decoded volume of `tracks` (planes rows: those tracks only) against its float64 bound."""
    kernel, fmt, products = branch
    T = coords.shape[0]
    n = len(tracks)
    vp = planes.reshape(planes.shape[0], n, T, K.LEVELS, K.VOL)
    sup = support * valid[None, None, :, None].float()
    dead = (valid[tracks] == 0).to(planes.device)
    worst = 0.0
    for l in range(K.LEVELS):
        lv = scratch_planes[l] if scratch_planes is not None else [pyr_levels[l]]
        pairs = K.operands(kernel, products, lv, sup[l])
        want, e = K.volume_want_bound(kernel, products, pairs, coords, l, tracks)
        got = vp[:, :, :, l].double().sum(0).transpose(0, 1)                  # [T, n, 2401]
        r = K.ratio_fp16(got, want, e) if fmt == "fp16" else K.ratio_split(got, want, e)
        assert bool((got[:, dead] == 0).all()), ("dead tracks must give exact zeros", l)
        for cls in sorted(set(labels)):
            m = torch.tensor([labels[int(i)] == cls for i in tracks], device=r.device)
            rc = float(r[:, m].max())
            _note((kernel, fmt, products, l, f"{tag}:{cls}"), rc)
            worst = max(worst, rc)
    return worst


CORR_CASES = [(case, branch, opts) for case in K.CASES
              for branch, opts in K.branch_options(case[1], case[2], case[3])]


def _corr_id(c):
    case, (kernel, fmt, products), _ = c
    return f"{case[0]}-{kernel}-{fmt}-p{products}"


@pytest.mark.parametrize("c", CORR_CASES, ids=[_corr_id(c) for c in CORR_CASES])
def test_corr_kernel_float64(eng, c):
    case, branch, opts = c
    kernel, fmt, products = branch
    coords, valid, labels, T, H4, W4 = K.case_inputs(case)
    N = coords.shape[1]
    rows = N * T * K.LEVELS
    pyr = eng.prepare_pyramid(K.features(T, H4, W4, seed=N + T).to(DEV))
    pyr_levels = eng.pyramid_levels(pyr, T, H4, W4)
    support = K.unit_support(N, seed=T).to(DEV)
    coords_d, valid_d = coords.to(DEV), valid.to(DEV)
    vol = torch.empty(rows + GUARD_ROWS, 2 * K.VOL_PAD, dtype=torch.bfloat16, device=DEV)
    vol.view(torch.int16).fill_(SENTINEL)
    scratch = torch.zeros(pyr.numel() * 4, dtype=torch.uint8, device=DEV)
    planes = _run_corr(eng, opts, pyr, H4, W4, support, valid_d, coords_d, vol, scratch)
    written, rest = _written(vol, rows, fmt)
    assert not bool((written == SENTINEL).any()), "a volume element was not written"
    assert bool((rest == SENTINEL).all()), "the kernel wrote past the volume"
    sp = _check_format(scratch, kernel, pyr_levels, T, H4, W4) if kernel in ("corr_tc3", "corr_tc2") else None
    worst = _check_levels(branch, planes, sp, pyr_levels, support, valid_d, coords_d, labels, torch.arange(N),
                          case[0])
    print("corr-ratio", _corr_id(c), f"{worst:.3g}")
    assert worst <= 1.0, (branch, worst)


def test_corr_headline_shape(eng):
    """N = 6400, T = 16, 96 x 128 under the default options: a 3.98 GB split volume (past 2^31 bytes) and many units
    per CTA from the dynamic unit counter.  Every row written (NaN sentinel), two runs bit-identical, and 576 tracks --
    the first and last 64 and a stride over the rest -- within the float64 bound."""
    T, N, H4, W4 = 16, 6400, 96, 128
    torch.cuda.reset_peak_memory_stats(DEV)
    t0 = time.time()
    rows = N * T * K.LEVELS
    branch = K.corr_branch({}, T, H4, W4)
    assert branch == ("corr_tc3", "split", 2)
    g = torch.Generator().manual_seed(16)
    coords = torch.rand(T, N, 2, generator=g) * torch.tensor([W4 + 16.0, H4 + 16.0]) - 8.0
    coords[:, ::97] = torch.rand(T, len(range(0, N, 97)), 2, generator=g) * 400 - 200     # far outside, moving
    valid = torch.ones(N, dtype=torch.uint8)
    valid[5::101] = 0
    labels = ["headline"] * N
    pyr = eng.prepare_pyramid(K.features(T, H4, W4, seed=17).to(DEV))
    pyr_levels = eng.pyramid_levels(pyr, T, H4, W4)
    support = K.unit_support(N, seed=18).to(DEV)
    coords_d, valid_d = coords.to(DEV), valid.to(DEV)
    scratch = torch.zeros(pyr.numel() * 4, dtype=torch.uint8, device=DEV)
    vols = []
    for _ in range(2):
        vol = torch.empty(rows, 2 * K.VOL_PAD, dtype=torch.bfloat16, device=DEV)
        assert vol.numel() * 2 > 2 ** 31
        vol.view(torch.int16).fill_(SENTINEL)
        eng.corr_sample(pyr, H4, W4, support, valid_d, coords_d, scratch=scratch, vol=vol)
        vols.append(vol)
    torch.cuda.synchronize()
    step = 1 << 14
    for r0 in range(0, rows, step):
        a, b = vols[0][r0:r0 + step].view(torch.int16), vols[1][r0:r0 + step].view(torch.int16)
        assert not bool((a == SENTINEL).any()), ("row not written", r0)
        assert torch.equal(a, b), ("runs differ", r0)
    tracks = sorted(set(range(64)) | set(range(N - 64, N)) | set(range(64, N - 64, 14)))
    assert len(tracks) >= 512
    sel = torch.tensor(tracks, device=DEV)
    sub = vols[0].view(N, T * K.LEVELS, 2 * K.VOL_PAD)[sel].reshape(-1, 2 * K.VOL_PAD)
    del vols, vol, a, b
    planes = eng.volume_planes(sub, T, len(tracks), H4, W4)
    sp = _check_format(scratch, branch[0], pyr_levels, T, H4, W4)
    worst = _check_levels(branch, planes, sp, pyr_levels, support, valid_d, coords_d, labels, sel, "headline")
    peak = torch.cuda.max_memory_allocated(DEV) / 2 ** 30
    print("corr-headline", f"worst {worst:.3g}", f"peak {peak:.2f} GiB", f"{time.time() - t0:.1f} s")
    assert worst <= 1.0, worst
    assert peak < 12.0, peak


def test_print_worst_ratios():
    """Runs last in the file: the worst err/bound per (kernel, format, corr products, level, case:class) and stage."""
    for key, r in sorted(RATIOS.items(), key=str):
        print("corr-worst", key, f"{r:.3g}")
