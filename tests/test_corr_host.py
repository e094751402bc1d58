"""CPU: the float64 correlation reference of corr_cases.py pinned to the oracle (run in float64) and to the reference's
own outputs, the arithmetic of its bounds, and the coverage claims of its case list."""
import contextlib

import numpy as np
import torch

import corr_cases as K
from cases import O, reference_golden, stage_inputs


@contextlib.contextmanager
def _float64_default():
    """The oracle builds its offsets and grid scale factors in the default dtype: float64 makes it exact to ~1e-15."""
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        yield
    finally:
        torch.set_default_dtype(old)


def _cl(level):
    """[T, C, H, W] -> channels-last [T, H, W, C]."""
    return level.permute(0, 2, 3, 1).contiguous()


def test_reference_matches_float64_oracle():
    """Border-heavy and far-outside cases (every class of the case generator) at a map where the patch kernels run
    and one where they do not: volume64 / support64 against O.correlation_volume / O.support_features in float64."""
    for T, H4, W4 in ((2, 64, 72), (3, 25, 33)):
        coords, *_ = K.case_inputs(("oracle", T, H4, W4, ("sweep", "centre", "far", "moving")), seed=5)
        keep = torch.arange(coords.shape[1])[:: 3]                     # a third of the tracks keeps the CPU time low
        coords = coords[:, keep].contiguous()
        N = coords.shape[1]
        pyr = O.normalized_pyramid(K.features(T, H4, W4, seed=7).double())
        sup = K.unit_support(N, seed=8).double()
        qf = torch.arange(N) % T
        worst = 0.0
        with _float64_default(), torch.no_grad():
            for l in range(K.LEVELS):
                want = O.correlation_volume(pyr[l], sup[l], coords.double() / 2 ** l)
                got = K.volume64(_cl(pyr[l]), sup[l], coords, l)
                worst = max(worst, float((got - want).abs().max()))
                want_s = O.support_features(pyr[l], qf, coords[0].double() / 2 ** l)
                got_s = K.support64(_cl(pyr[l]), qf, coords[0], l)
                worst = max(worst, float((got_s - want_s).abs().max()))
        assert worst < 1e-12, (T, H4, W4, worst)


def test_reference_matches_reference_outputs():
    """cases.stage_inputs() through volume64 / support64 against the reference's own fp32 outputs
    (tests/golden/reference_stages.npz): raw randn features and support, so |corr| reaches tens; fp32 noise of the
    reference is a few ulps of the products it sums."""
    x = stage_inputs()
    fm, sup, coords = x["corr_fm"][0], x["corr_sup"][0], x["corr_coords"]
    got = K.volume64(_cl(fm.double()), sup.double(), coords, 0)
    S = K.volume64(_cl(fm.double()).abs(), sup.double().abs(), coords, 0)
    _, want = reference_golden("reference_stages", "corr_volume")
    err = (got.reshape(-1) - want.double()).abs()
    assert float((err / (2.0 ** -18 * S.reshape(-1) + 1e-30)).max()) < 1.0, float(err.max())
    assert float(err.max()) < 1e-4
    idx, want_s = reference_golden("reference_stages", "support")
    got_s = K.support64(_cl(x["sup_fm"][0].double()), x["sup_qf"][0], x["sup_qc"][0], 0).reshape(-1)[idx]
    # grid_sample's normalise / denormalise of the fp32 positions moves them by ~1e-7 texels: ~1e-6 in |f| ~ 4
    assert float((got_s - want_s.double()).abs().max()) < 1e-5


def test_bounds_admit_a_weight_ulp_and_reject_a_dropped_lo_plane():
    """At a patch-kernel map with border-heavy coordinates, on the corr_tc3 prec.corr = 2 operands: a volume whose
    x tap weights are all off by one fp32 ulp (2^-24) stays inside the bound in both output formats; the volume
    without the lo support plane (the prec.corr = 1 product) falls far outside it."""
    T, H4, W4 = 2, 64, 64
    coords, valid, *_ = K.case_inputs(("bounds", T, H4, W4, ("sweep", "moving")), seed=3)
    N = coords.shape[1]
    pyr = O.normalized_pyramid(K.features(T, H4, W4, seed=4))
    sup = K.unit_support(N, seed=6) * valid[None, None, :, None].float()
    worst_in, worst_out = 0.0, 0.0
    for l in (0, 3):
        planes = [_cl(pyr[l]).half()]
        pairs = K.operands("corr_tc3", 2, planes, sup[l])
        want, e = K.volume_want_bound("corr_tc3", 2, pairs, coords, l)
        # one ulp on every x weight: the same sample positions moved by 2^-24 (away from the map's last texel)
        x, y = K.positions(coords, l)
        x = torch.where(x < W4 / 2 ** l - 2, x + 2.0 ** -24, x)
        frames = torch.arange(T)[:, None]
        F, S = pairs[0]
        f = K.sample64(F, frames, x, y)
        got = torch.einsum("tnpc,nkc->tnpk", f, S.transpose(0, 1)).reshape(T, N, K.VOL)
        assert float((got - want).abs().max()) > 0
        worst_in = max(worst_in, float(K.ratio_split(got, want, e).max()),
                       float(K.ratio_fp16(got.float().half().double(), want, e).max()))
        dropped = K.volume64(F, K.operands("corr_tc3", 1, planes, sup[l])[0][1], coords, l)
        worst_out = max(worst_out, float(K.ratio_split(dropped, want, e).max()))
    assert worst_in <= 1.0, worst_in
    assert worst_out > 10.0, worst_out


def test_case_list_reaches_every_shift_branch_and_kernel():
    """Every shift d in [-7, 7] on both axes at every level of every map where the patch kernels run, both accepting
    tap_weights branches and never the rejecting one, frame pairs with different shifts, far coordinates beyond int32,
    dead tracks, the T and N edges, and every reachable (kernel, volume format, corr products)."""
    every_shift = {(l, ax, d) for l in range(K.LEVELS) for ax in (0, 1) for d in range(-7, 8)}
    seen_branches, seen_kernels, Ts, Ns, sizes = set(), set(), set(), set(), set()
    for case in K.CASES:
        coords, valid, labels, T, H4, W4 = K.case_inputs(case)
        Ts.add(T)
        Ns.add(coords.shape[1])
        sizes.add((H4, W4))
        shifts, branches = K.shift_coverage(coords, H4, W4)
        assert 0 not in {b for *_, b in branches}, case[0]
        seen_branches |= {b for *_, b in branches}
        if case[0].startswith("edges-") and min(H4, W4) >> 3 >= 8:
            assert shifts == every_shift, (case[0], every_shift - shifts)
        seen_kernels |= {k for k, _ in K.branch_options(T, H4, W4)}
        if "far" in case[4]:
            assert float(coords.abs().max()) >= 3e9 and bool((valid == 0).any())
        if "moving" in case[4] and T >= 2 and min(H4, W4) >> 3 >= 8:
            d0 = K.box_origin8(coords[0::2][: T // 2, :, 0].numpy(), W4)[1]
            d1 = K.box_origin8(coords[1::2][: T // 2, :, 0].numpy(), W4)[1]
            assert bool((d0 != d1).any()), case[0]
    assert seen_branches == {1, 2}
    assert seen_kernels == K.REACHABLE, seen_kernels ^ K.REACHABLE
    assert {K.corr_branch(o, 16, H4, W4) for o in K.OPTION_SETS for H4, W4 in K.MAP_SIZES} == K.REACHABLE
    assert {1, 2, 60} <= Ts and any(t % 2 for t in Ts) and 1 in Ns
    assert sizes >= {(64, 64), (64, 72), (96, 128), (24, 32), (25, 33)}


def test_fp16_ratio_is_the_rounding_interval():
    """ratio_fp16 <= 1 exactly for the fp16 neighbours of [want - e, want + e], subnormals included."""
    want = torch.tensor([0.1, 1e-6, -3e-8, 0.0], dtype=torch.float64)
    e = torch.tensor([1e-7, 1e-9, 1e-9, 0.0], dtype=torch.float64)
    lo, hi = (want - e).float().half(), (want + e).float().half()
    for inside in (lo, hi, want.float().half()):
        assert float(K.ratio_fp16(inside.double(), want, e).max()) <= 1.0
    below = torch.from_numpy(np.nextafter(lo.numpy(), np.float16(-np.inf)))
    above = torch.from_numpy(np.nextafter(hi.numpy(), np.float16(np.inf)))
    assert bool((K.ratio_fp16(below.double(), want, e) > 1).all())
    assert bool((K.ratio_fp16(above.double(), want, e) > 1).all())
