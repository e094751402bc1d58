"""CPU tests of the encoder's float64 link restatements (tests/encoder_cases.py) and of ct3_encoder_trace's argument
checks: the restatements chained reproduce the oracle encoder, their bounds admit a one-ulp error and reject the
kernel errors they exist to catch, the case list reaches every branch, and bad arguments fail before any launch."""
import ctypes

import torch

import encoder_cases as E
from cotracker_b200 import engine
from oracle import ct3_oracle as O

EINVAL, ENOSPC = -1, -3


def _frames(T, H, W, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(T, 3, H, W, generator=g, dtype=torch.float64) * 2 - 1


def test_weight_names_match_the_library():
    assert E.weight_names() == engine.encoder_weight_names()
    sd = E.encoder_weights(0)
    for k, v in sd.items():
        assert v.dtype == torch.float32
        assert torch.equal(E.round16(v), v)                      # hi + lo of the packed weight is the weight
        hi, lo = E.split_f32(v)
        assert torch.equal(hi.double() + lo.double(), v.double()), k


def test_chained_restatements_match_the_oracle():
    for (T, H, W), eng in (((1, 32, 32), True), ((2, 50, 66), False)):
        sd = {k: v.double() for k, v in E.encoder_weights(4, engineered=eng).items()}
        x = _frames(T, H, W, seed=T)
        got = E.chain64(sd, x)
        want = O.normalized_pyramid(O.encoder(sd, x, prefix=""))
        for l in range(4):
            err = float((E.nchw(got[l]) - want[l]).abs().max())
            assert err < 1e-12, (H, W, l, err)


def test_split_restatement_is_bitwise():
    g = torch.Generator().manual_seed(3)
    v = (torch.randn(4096, generator=g) * torch.exp(torch.randn(4096, generator=g) * 8)).float()
    hi, lo = E.split_f32(v)
    # hi is the nearest bf16 and lo the nearest bf16 of the (exact) remainder
    assert torch.equal(hi.float(), v.to(torch.bfloat16).float())
    r = v.double() - hi.double()
    assert torch.equal(r.float().double(), r)
    assert bool(((hi.double() + lo.double() - v.double()).abs() <= 2.0 ** -17 * v.double().abs()).all())


def _conv_case(seed=5, T=1, h=9, w=11, cin=64, cout=64):
    g = torch.Generator().manual_seed(seed)
    x = torch.relu(torch.randn(T, h, w, cin, generator=g)).float()
    hi, lo = E.split_f32(x)
    wt = E.round16(torch.randn(cout, cin, 3, 3, generator=g) * (2.0 / (9 * cin)) ** 0.5)
    b = E.round16(torch.randn(cout, generator=g) * 0.1)
    return hi.double(), lo.double(), wt, b


def test_conv_bound_admits_one_ulp_and_rejects_kernel_errors():
    hi, lo, wt, b = _conv_case()
    want, bound = E.conv_split_ref(hi, lo, wt, b, 1, 1)
    y = want.float()
    one_ulp = torch.nextafter(y, torch.full_like(y, float("inf"))).double()
    assert bool(((one_ulp - want).abs() <= bound).all())
    # a dropped lo plane of the activation: hi * (w_hi + w_lo) only
    drop, _ = E.conv_ref(hi, wt, b, 1, 1)
    assert float(((drop - want).abs() / bound).max()) > 10
    # a border tap shifted by one row (the A box of tap ky requested at y offset ky instead of ky - 1)
    shifted = torch.zeros_like(hi + lo)
    shifted[:, :-1] = (hi + lo)[:, 1:]
    bad, _ = E.conv_ref(shifted, wt, b, 1, 1)
    assert float(((bad - want).abs() / bound).max()) > 1e3
    # the stem: a patch origin off by one column
    f = torch.rand(1, 3, 20, 24, generator=torch.Generator().manual_seed(2)) * 2 - 1
    ws = E.round16(torch.randn(64, 3, 7, 7) * 0.1)
    bs = E.round16(torch.randn(64) * 0.1)
    want, bound = E.stem_ref(f, ws, bs)
    bad, _ = E.stem_ref(torch.roll(f, 1, dims=3), ws, bs)
    assert float(((bad - want).abs() / bound).max()) > 1e3
    y = want.float()
    assert bool(((torch.nextafter(y, torch.zeros_like(y)).double() - want).abs() <= bound).all())


def test_gemm_and_gather_restatements_agree_with_the_convolution():
    hi, lo, _, _ = _conv_case(cin=64)
    g = torch.Generator().manual_seed(9)
    w2 = E.round16(torch.randn(96, 64, 3, 3, generator=g) * 0.05)
    b2 = E.round16(torch.randn(96, generator=g))
    x_split = torch.cat([(hi).to(torch.bfloat16), lo.to(torch.bfloat16)], -1).reshape(-1, 128)
    rows = E.gather_ref(x_split, 1, 9, 11, 64, 9)
    want, bound = E.gemm_ref(rows, w2, b2, 64, 128)
    ref, _ = E.conv_ref(hi + lo, w2, b2, 2, 1, 128)
    assert float((want - ref.reshape(want.shape)).abs().max()) < 1e-12
    assert bool((want[:, 96:] == 0).all()) and bool((bound[:, 96:] == 0).all())   # padded channels: exactly 0
    rows_d = E.gather_ref(x_split, 1, 9, 11, 64, 1)
    wd = E.round16(torch.randn(96, 64, 1, 1, generator=g) * 0.1)
    want_d, _ = E.gemm_ref(rows_d, wd, b2, 64, 128)
    ref_d, _ = E.conv_ref(hi + lo, wd, b2, 2, 0, 128)
    assert float((want_d - ref_d.reshape(want_d.shape)).abs().max()) < 1e-12


def test_stats_bound_rejects_fp32_variance():
    g = torch.Generator().manual_seed(6)
    T, h, w, C = 1, 48, 64, 4
    y = torch.randn(T, h, w, C, generator=g, dtype=torch.float64)
    y[..., 1] = 1.0 + 1e-4 * y[..., 1]                           # |mean| / std = 1e4
    y[..., 2] = 0.3                                              # constant: var 0
    y = y.float()
    mean, rstd, bm, br = E.stats_ref(y)
    # fp64 sums rounded to fp32 stay inside
    v = y.double().reshape(T, -1, C)
    m64 = v.sum(1) / v.shape[1]
    var64 = ((v * v).sum(1) / v.shape[1] - m64 * m64).clamp_min(0)
    assert bool(((m64.float().double() - mean).abs() <= bm).all())
    assert bool(((1 / torch.sqrt(var64 + E.EPS32)).float().double() - rstd).abs().le(br).all())
    assert float(rstd[0, 2]) == 1 / E.EPS32 ** 0.5
    # one-pass fp32 sums lose the dominated channel's variance
    v32 = y.reshape(T, -1, C)
    s, ss = torch.zeros(T, C), torch.zeros(T, C)
    for i in range(v32.shape[1]):
        s += v32[:, i]
        ss += v32[:, i] * v32[:, i]
    m32 = s / v32.shape[1]
    var32 = (ss / v32.shape[1] - m32 * m32).clamp_min(0)
    r32 = 1 / torch.sqrt(var32 + E.EPS32)
    assert float((r32.double() - rstd).abs()[0, 1] / br[0, 1]) > 100


def test_norm_act_modes_and_resize():
    g = torch.Generator().manual_seed(7)
    y = torch.randn(2, 5, 6, 8, generator=g).float()
    x = torch.relu(torch.randn(2, 5, 6, 8, generator=g)).float()
    st = torch.stack([torch.randn(2, 8, generator=g), torch.rand(2, 8, generator=g) + 0.5], -1).float()
    sd = torch.stack([torch.randn(2, 8, generator=g), torch.rand(2, 8, generator=g) + 0.5], -1).float()
    a32 = E.norm0_f32(y, st)
    a, bnd = E.norm_act_ref(0, y, st)
    assert bool(((a32.double() - a).abs() <= bnd).all())
    # mode 2 normalising the shortcut with stats instead of stats_d falls outside
    want, bnd = E.norm_act_ref(2, y, st, x, sd)
    bad, _ = E.norm_act_ref(2, y, st, x, st)
    assert float(((bad - want).abs() / bnd.clamp_min(1e-30)).max()) > 1e3
    # resize: the fp32-index blend sits inside the exact-coordinate bound; align_corners=False does not
    srcs = [torch.randn(1, h, w, c, generator=g).float() for (h, w), c in zip(E.stage_hw(98, 130), E.STAGE_CP)]
    want, bnd, copied = E.resize_ref(srcs, 24, 32, exact=True)
    got, _, _ = E.resize_ref(srcs, 24, 32)
    assert bool(((got - want).abs() <= bnd).all()) and not bool(copied[:416].any())
    bad = torch.cat([E.nhwc(torch.nn.functional.interpolate(E.nchw(s[..., :c].double()), (24, 32), mode="bilinear",
                                                             align_corners=False))
                     for s, c in zip(srcs, E.STAGE_C)], -1)
    assert float(((bad - want[..., :416]).abs() / bnd[..., :416]).max()) > 1e3


def test_cases_reach_every_branch():
    tws, bns, branches, s3 = set(), set(), set(), set()
    for c in E.CASES:
        for (_, _, _, _, bn, tw) in E.conv_launches(c.H, c.W):
            tws.add(tw)
            bns.add(bn)
        branches |= set(E.resize_branches(c.H, c.W))
        h3, w3 = E.stage_hw(c.H, c.W)[3]
        s3.add((min(h3, 3), min(w3, 3)))
    assert tws == {128, 64, 32, 16, 8}, tws
    assert bns == {64, 128}
    assert branches == {"copy", "interpolate"}
    assert {(2, 2), (2, 3), (3, 2)} <= s3, s3                       # 2x2, 2xN and Nx2 stage-3 maps
    # the production shape: tw = 128 on 192x256 and 96x128, 64 on 48x64, 32 on 24x32
    assert [E.pick_tile(*hw)[0] for hw in E.stage_hw(384, 512)] == [128, 128, 64, 32]
    assert E.resize_branches(100, 132) == ["interpolate", "copy", "interpolate", "interpolate"]
    assert E.resize_branches(98, 130) == ["interpolate"] * 4
    assert any(T > 16 and T % 16 for T, _, _ in E.CHUNK_CASES) and any(T > 32 for T, _, _ in E.CHUNK_CASES)


def test_encoder_trace_links_match_the_layout():
    for (T, H, W) in ((1, 384, 512), (16, 32, 32), (3, 98, 130)):
        offs, nb, total = engine.encoder_trace_layout(T, H, W)
        links = engine.encoder_trace_links(T, H, W)
        assert len(links) == engine.ENCODER_TRACE_LINKS == len(offs)
        end = 0
        for (name, dt, shape), o, n in zip(links, offs, nb):
            assert n == dt.itemsize * torch.Size(shape).numel(), name
            assert o % 256 == 0 and o >= end, name
            end = o + n
        assert total >= end


def _p(addr):
    return ctypes.c_void_p(addr)


def test_encoder_trace_rejects_bad_arguments_without_gpu():
    lib = engine.lib()
    n = ctypes.c_size_t(0)
    assert lib.ct3_encoder_trace_layout(1, 32, 32, None, None, ctypes.byref(n)) == 0
    need = n.value
    assert lib.ct3_encoder_trace_layout(1, 32, 32, None, None, None) == EINVAL
    for T, H, W in ((0, 64, 64), (17, 64, 64), (1, 31, 64), (1, 64, 31), (1, 15, 64), (1, 64, -1)):
        assert lib.ct3_encoder_trace_layout(T, H, W, None, None, ctypes.byref(n)) == EINVAL, (T, H, W)
    assert lib.ct3_encoder_workspace_bytes(1, 32, 32, ctypes.byref(n)) == 0
    ws_need = n.value
    base = dict(packed=_p(1 << 20), frames=_p(1 << 21), T=1, H=32, W=32, pyr=_p(1 << 22), trace=_p(1 << 24),
                tbytes=need, ws=_p(1 << 26), wbytes=ws_need)

    def call(**kw):
        a = dict(base, **kw)
        return lib.ct3_encoder_trace(a["packed"], a["frames"], a["T"], a["H"], a["W"], a["pyr"], a["trace"],
                                     a["tbytes"], a["ws"], a["wbytes"], None)

    for kw, code, msg in [
        (dict(packed=None), EINVAL, b"null argument"),
        (dict(frames=None), EINVAL, b"null argument"),
        (dict(pyr=None), EINVAL, b"null argument"),
        (dict(trace=None), EINVAL, b"null argument"),
        (dict(ws=None), EINVAL, b"null argument"),
        (dict(T=0), EINVAL, b"T >= 1"),
        (dict(T=17), EINVAL, b"T <= 16"),
        (dict(H=31), EINVAL, b"4 pyramid levels"),
        (dict(W=16), EINVAL, b"4 pyramid levels"),
        (dict(H=15), EINVAL, b"H, W >= 16"),
        (dict(trace=_p((1 << 24) + 16)), EINVAL, b"256-byte aligned"),
        (dict(ws=_p((1 << 26) + 64)), EINVAL, b"256-byte aligned"),
        (dict(tbytes=need - 1), ENOSPC, b"trace buffer too small"),
        (dict(wbytes=ws_need - 1), ENOSPC, b"workspace too small"),
    ]:
        assert call(**kw) == code, kw
        assert msg in lib.ct3_last_error(), (kw, lib.ct3_last_error())


def test_encoder_rejects_every_size_below_32_without_gpu():
    """the header's minimum, 32 x 32: every H or W in 16..31 fails in ct3_encoder and its workspace query"""
    lib = engine.lib()
    n = ctypes.c_size_t(0)
    for v in range(16, 32):
        for H, W in ((v, 64), (64, v), (v, v)):
            assert lib.ct3_encoder_workspace_bytes(1, H, W, ctypes.byref(n)) == EINVAL, (H, W)
            assert lib.ct3_encoder(_p(1 << 20), _p(1 << 21), 1, H, W, _p(1 << 22), _p(1 << 24), 1 << 40,
                                   None) == EINVAL, (H, W)
            assert b"4 pyramid levels" in lib.ct3_last_error()
    assert lib.ct3_encoder_workspace_bytes(1, 32, 32, ctypes.byref(n)) == 0
