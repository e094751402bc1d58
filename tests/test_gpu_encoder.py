"""The CNN encoder link by link against float64 (bounds derived in tests/encoder_cases.py): ct3_encoder_trace runs
ct3_encoder's own code and hands back every link's output -- the stem, each InstanceNorm's statistics, each norm_act
output (fp32 and split), each conv3x3_tc output, the stride-2 gathers and GEMMs, the resize + concat operand, conv2,
instnorm_relu_split, conv3 before the L2 norm and the pyramid -- and each link is checked per element against its
float64 restatement on the kernel's own input to it.

Cases: the production shape, odd sizes (one with a directly copied stage, one with every stage interpolated), tall and
wide skinny frames (every conv3x3_tc tile width), the 32 x 32 minimum with its 2 x 2 stage-3 maps and skinny variants,
and engineered channels (zero weights, |mean| / std ~ 1e4, all negative).  Besides: stage 1's padded channels and the
concat's channels 416..447 are exactly zero, chunked clips equal their frames encoded alone bit for bit, ct3_encoder
equals the trace's pyramid bit for bit, and the whole encoder meets the float64 oracle."""
import math

import pytest
import torch

import encoder_cases as E
from cotracker_b200 import engine
from oracle import ct3_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RATIOS = {}          # (link kind, case) -> worst err / bound
_PACKED = {}


def _weights(case):
    key = (case.seed, case.engineered)
    if key not in _PACKED:
        sd = E.encoder_weights(case.seed, case.engineered)
        _PACKED[key] = (sd, engine.encoder_pack(sd, DEV), {k: v.to(DEV) for k, v in sd.items()})
    return _PACKED[key]


def _frames(T, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(T, 3, H, W, generator=g) * 2 - 1).to(DEV)


class Checker:
    def __init__(self, case):
        self.case, self.fails = case, []

    def bound(self, kind, name, got, want, bound):
        err = (got.double().reshape(want.shape) - want).abs()
        ok = bool((err <= bound).all())
        r = float((err / bound).nan_to_num(nan=0.0).max())          # 0 / 0: exact where exactness is the bound
        key = (kind, self.case.name)
        RATIOS[key] = max(RATIOS.get(key, 0.0), r)
        if not ok:
            self.fails.append(f"{name}: err/bound {r:.3g}, max err {float(err.max()):.3g}")

    def bits(self, name, got, want):
        if not E.same_bits(got.reshape(want.shape), want):
            n = int((got.reshape(want.shape).float() != want.float()).sum())
            self.fails.append(f"{name}: {n} elements differ bitwise")

    def zero(self, name, t):
        if bool((t.float() != 0).any()):
            self.fails.append(f"{name}: padding not zero")


def _split_nhwc(t, T, h, w, C):
    hi, lo = E.planes(t, C)
    return hi.reshape(T, h, w, C), lo.reshape(T, h, w, C)


def check_case(case, frames=None):
    sd, packed, sdd = _weights(case)
    T, H, W = case.T, case.H, case.W
    frames = _frames(T, H, W, case.seed + 100) if frames is None else frames
    tr = engine.encoder_trace(packed, frames)
    torch.cuda.synchronize()
    ck = Checker(case)
    hw = E.stage_hw(H, W)

    # stem
    want, bnd = E.stem_ref(frames, sdd["conv1.weight"], sdd["conv1.bias"])
    ck.bound("stem", "stem.conv", tr["stem.conv"], want, bnd)
    _stats(ck, "stem.stats", tr["stem.conv"], tr["stem.stats"])
    _norm(ck, "stem", 0, tr["stem.conv"], tr["stem.stats"], tr["stem.out"], tr["stem.out_split"])

    for s, u, stride, h, w, hin, win in E.units(H, W):
        p, cp = f"layer{s + 1}.{u}", E.STAGE_CP[s]
        src = E.unit_input(s, u)
        cin = E.STAGE_CP[s - 1] if stride == 2 else cp
        if stride == 2:
            gat = E.gather_ref(tr[src + "_split"], T, hin, win, cin, 9)
            ck.bits(p + ".gather", tr[p + ".gather"], gat)
            ck.bits(p + ".gather_d", tr[p + ".gather_d"], E.gather_ref(tr[src + "_split"], T, hin, win, cin, 1))
            want, bnd = E.gemm_ref(tr[p + ".gather"], sdd[p + ".conv1.weight"], sdd[p + ".conv1.bias"], cin, cp)
            ck.bound("gemm 3x3/2", p + ".conv1", tr[p + ".conv1"], want, bnd)
        else:
            hi, lo = _split_nhwc(tr[src + "_split"], T, h, w, cp)
            want, bnd = E.conv_split_ref(hi, lo, sdd[p + ".conv1.weight"], sdd[p + ".conv1.bias"], 1, 1, cp)
            ck.bound("conv3x3_tc", p + ".conv1", tr[p + ".conv1"], want, bnd)
        _stats(ck, p + ".conv1.stats", tr[p + ".conv1"], tr[p + ".conv1.stats"])
        _norm(ck, p + ".norm1", 0, tr[p + ".conv1"], tr[p + ".conv1.stats"], None, tr[p + ".norm1_split"])
        hi, lo = _split_nhwc(tr[p + ".norm1_split"], T, h, w, cp)
        want, bnd = E.conv_split_ref(hi, lo, sdd[p + ".conv2.weight"], sdd[p + ".conv2.bias"], 1, 1, cp)
        ck.bound("conv3x3_tc", p + ".conv2", tr[p + ".conv2"], want, bnd)
        _stats(ck, p + ".conv2.stats", tr[p + ".conv2"], tr[p + ".conv2.stats"])
        if stride == 2:
            want, bnd = E.gemm_ref(tr[p + ".gather_d"], sdd[p + ".downsample.0.weight"],
                                   sdd[p + ".downsample.0.bias"], cin, cp)
            ck.bound("gemm 1x1/2", p + ".downsample", tr[p + ".downsample"], want, bnd)
            _stats(ck, p + ".downsample.stats", tr[p + ".downsample"], tr[p + ".downsample.stats"])
            _norm(ck, p + ".out", 2, tr[p + ".conv2"], tr[p + ".conv2.stats"], tr[p + ".out"], tr[p + ".out_split"],
                  tr[p + ".downsample"], tr[p + ".downsample.stats"])
        else:
            _norm(ck, p + ".out", 1, tr[p + ".conv2"], tr[p + ".conv2.stats"], tr[p + ".out"], tr[p + ".out_split"],
                  tr[src])
        if s == 1:   # stage 1 carries 96 channels padded to 128: every link that holds them keeps them exactly zero
            for k in (".conv1", ".conv2", ".out") + ((".downsample",) if stride == 2 else ()):
                ck.zero(p + k, tr[p + k][..., 96:])
            for k in (".norm1_split", ".out_split"):
                ck.zero(p + k, tr[p + k].reshape(-1, 2, 128)[..., 96:])
        if s == 2 and stride == 2:
            ck.zero(p + ".gather", tr[p + ".gather"].reshape(-1, 2, 9, 128)[..., 96:])

    # resize + concat
    H4, W4 = H // 4, W // 4
    srcs = [tr[f"layer{s + 1}.1.out"] for s in range(4)]
    got_hi, got_lo = E.planes(tr["cat_split"], E.CAT_CP)
    want, bnd, copied = E.resize_ref(srcs, H4, W4, split=False)
    cat_val = (got_hi + got_lo).reshape(T, H4, W4, E.CAT_CP)
    split_err = E.half_ulp_bf16(got_lo).reshape(cat_val.shape)
    copied = copied.to(DEV)
    ck.bound("resize", "cat_split", cat_val[..., ~copied], want[..., ~copied], (bnd + split_err)[..., ~copied])
    exact, ebnd, _ = E.resize_ref(srcs, H4, W4, exact=True, split=False)
    ck.bound("resize vs interpolate", "cat_split", cat_val[..., ~copied], exact[..., ~copied],
             (ebnd + split_err)[..., ~copied])
    idx = copied[:E.CAT_C].nonzero().flatten()
    if len(idx):   # a stage the size of H4 x W4 is copied: its split is the fp32 source's, bit for bit
        got = torch.cat([tr["cat_split"][:, idx], tr["cat_split"][:, E.CAT_CP + idx]], 1)
        ck.bits("cat_split (copied stage)", got, E.split_rows(want[..., idx].float()))
    ck.zero("cat_split 416..447", tr["cat_split"].reshape(-1, 2, E.CAT_CP)[..., E.CAT_C:])

    # conv2 -> IN -> relu -> conv3 -> pyramid
    hi, lo = _split_nhwc(tr["cat_split"], T, H4, W4, E.CAT_CP)
    want, bnd = E.conv_split_ref(hi, lo, sdd["conv2.weight"], sdd["conv2.bias"], 1, 1)
    ck.bound("conv3x3_tc", "conv2", tr["conv2"], want, bnd)
    _stats(ck, "conv2.stats", tr["conv2"], tr["conv2.stats"])
    _norm(ck, "conv2.out", 0, tr["conv2"], tr["conv2.stats"], None, tr["conv2.out_split"])
    want, bnd = E.gemm_ref(tr["conv2.out_split"], sdd["conv3.weight"], sdd["conv3.bias"], E.MID, E.LATENT)
    ck.bound("conv3 gemm", "conv3", tr["conv3"], want, bnd)
    levels = engine.pyramid_levels(tr["pyramid"], T, H4, W4)
    want, bnd = E.l2norm_ref(tr["conv3"])
    ck.bound("l2norm", "pyramid level 0", levels[0], want, bnd)
    for l in range(1, 4):
        want, bnd = E.pool_ref(levels[l - 1])
        ck.bound("pool", f"pyramid level {l}", levels[l], want, bnd)

    if case.engineered:
        _engineered(ck, tr, T)
    # ct3_encoder runs the same launches: its pyramid is the trace's, bit for bit
    ws = torch.empty(engine.encoder_workspace_bytes(T, H, W), dtype=torch.uint8, device=DEV)
    pyr = engine.encoder(packed, frames, ws)
    if not torch.equal(pyr, tr["pyramid"]):
        ck.fails.append("ct3_encoder differs from ct3_encoder_trace's pyramid")
    return ck.fails


def _stats(ck, name, y, stats):
    mean, rstd, bm, br = E.stats_ref(y)
    st = stats.double()
    ck.bound("instnorm stats", name + " mean", st[..., 0], mean, bm)
    ck.bound("instnorm stats", name + " rstd", st[..., 1], rstd, br)


def _norm(ck, name, mode, y, stats, out, out_split, x=None, stats_d=None):
    want, bnd = E.norm_act_ref(mode, y, stats, x, stats_d)
    if out is not None:
        ck.bound(f"norm_act {mode}", name, out, want, bnd)
        ck.bits(name + "_split", out_split, E.split_rows(out))
    else:
        a32 = E.norm0_f32(y, stats)
        ck.bound(f"norm_act {mode}", name + " (fp32 restated)", a32, want, bnd)
        ck.bits(name + "_split", out_split, E.split_rows(a32))


def _engineered(ck, tr, T):
    """the engineered channels do what they are made for, and the links above met their bounds on them"""
    layer_out = {"conv1": ("stem.conv", "stem.stats", "stem.out_split", 64)}
    for l in ("layer1.0.conv1", "layer1.0.conv2", "layer1.1.conv2", "layer2.0.conv1", "layer2.0.conv2",
              "layer2.1.conv1", "layer3.0.downsample.0", "layer3.1.conv2", "layer4.0.conv1"):
        s, u, c = l.split(".")[0], l.split(".")[1], l.split(".")[2]
        cp = E.STAGE_CP[int(s[5]) - 1]
        stem = f"{s}.{u}.{'downsample' if c == 'downsample' else c}"
        split = f"{s}.{u}.norm1_split" if c == "conv1" else None
        layer_out[l] = (stem, stem + ".stats", split, cp)
    layer_out["conv2"] = ("conv2", "conv2.stats", "conv2.out_split", 256)
    for l, c in E.ZERO:
        y, st, sp, cp = layer_out[l]
        if bool((tr[y][..., c] != tr[y][..., c].flatten()[0]).any()):
            ck.fails.append(f"{l}[{c}]: zero-weight channel is not constant")
        if bool((tr[st][:, c, 1] != float(torch.tensor(1 / math.sqrt(E.EPS32)).float())).any()):
            ck.fails.append(f"{l}[{c}]: rstd is not 1/sqrt(eps)")
        if sp is not None and bool((tr[sp].reshape(-1, 2, cp)[..., c].float() != 0).any()):
            ck.fails.append(f"{l}[{c}]: relu(IN) of a constant map is not exactly 0")
    for l, c in E.DOMINATED:
        y = tr[layer_out[l][0]][..., c].double().reshape(T, -1)
        ratio = float((y.mean(1).abs() / y.std(1)).min())
        RATIOS[("engineered |mean|/std", ck.case.name)] = ratio
        if ratio < 1e3:
            ck.fails.append(f"{l}[{c}]: |mean|/std only {ratio:.3g}")
    for l, c in E.NEGATIVE:
        if bool((tr[layer_out[l][0]][..., c] >= 0).any()):
            ck.fails.append(f"{l}[{c}]: not all negative before IN")


@pytest.mark.parametrize("case", E.CASES, ids=[c.name for c in E.CASES])
def test_every_link_meets_its_bound(case):
    fails = check_case(case)
    assert not fails, "\n".join(fails)


@pytest.mark.parametrize("case", E.WHOLE_CASES, ids=[c.name for c in E.WHOLE_CASES])
def test_whole_encoder_matches_float64_oracle(case):
    fails = check_case(case)
    assert not fails, "\n".join(fails)
    sd, packed, sdd = _weights(case)
    frames = _frames(case.T, case.H, case.W, case.seed + 100)
    ws = torch.empty(engine.encoder_workspace_bytes(case.T, case.H, case.W), dtype=torch.uint8, device=DEV)
    pyr = engine.encoder(packed, frames, ws)
    sd64 = {k: v.double() for k, v in sdd.items()}
    want = O.normalized_pyramid(O.encoder(sd64, frames.double(), prefix=""))
    levels = engine.pyramid_levels(pyr, case.T, case.H // 4, case.W // 4)
    errs = [float((levels[l].permute(0, 3, 1, 2).double() - want[l]).abs().max()) for l in range(4)]
    print(f"\nwhole encoder {case.name}: worst |err| per level " + " ".join(f"{e:.3e}" for e in errs))
    RATIOS[("whole encoder / 2e-5", case.name)] = max(errs) / 2e-5
    assert max(errs) < 2e-5, errs


@pytest.mark.parametrize("T,H,W", E.CHUNK_CASES)
def test_chunked_frames_equal_frames_encoded_alone(T, H, W):
    _, packed, _ = _weights(E.Case("chunk", T, H, W))
    frames = _frames(T, H, W, 7)
    ws = torch.empty(engine.encoder_workspace_bytes(T, H, W), dtype=torch.uint8, device=DEV)
    levels = engine.pyramid_levels(engine.encoder(packed, frames, ws), T, H // 4, W // 4)
    ws1 = torch.empty(engine.encoder_workspace_bytes(1, H, W), dtype=torch.uint8, device=DEV)
    for t in sorted({0, 15, 16, T - 2, T - 1} | ({31, 32} if T > 32 else set())):
        one = engine.pyramid_levels(engine.encoder(packed, frames[t:t + 1].contiguous(), ws1), 1, H // 4, W // 4)
        for l in range(4):
            assert torch.equal(levels[l][t], one[l][0]), (T, t, l)


def test_zz_print_ratios():
    """the worst err / bound per (link, case), as measured by the tests above"""
    print(f"\npeak device memory {torch.cuda.max_memory_allocated(DEV) / 2 ** 30:.2f} GiB")
    for (kind, case), r in sorted(RATIOS.items()):
        print(f"{kind:28s} {case:24s} {r:.3g}")
