"""The transformer body around the attention cores, stage by stage, against float64: every GEMM epilogue the update loop
and the encoder use (ct3_linear_ex), the fused q|k|v projection + time attention of a time block
(ct3_time_block_attention) and the LayerNorm (ct3_layernorm).

Each float64 reference multiplies exactly the values the kernel reads: x_split and the weight planes are decoded in
float64 (hi + lo, the hi plane alone where only it is read), and weights that go through ct3_pack_weights are rounded
to 16 significant bits first, so that their split into bf16 hi + lo is exact.  What is left is the error the kernel
itself adds, and every bound below is that error, elementwise.  u = 2^-24 is the fp32 unit roundoff.

GEMM (y = act(x w^T + bias + row_bias) [+ residual]), per output element, S = sum_k |x_k| |w_k|:
  dropped product  3 products drop lo*lo: at most L = sum_k |x_lo,k| |w_lo,k| (<= 2^-16 S for bf16, as |lo| <= 2^-8
                   |hi|), computed from the planes; 1 and 2 products multiply exactly what the reference multiplies, and
                   the SIMT kernel multiplies hi + lo: 0.
  accumulation     tensor cores (gemm 0): the products are exact and each of the n = products * Kpad / 16 wgmma steps
                   adds into the fp32 accumulator with one rounding, <= 2u of the magnitudes involved (2u, not u: the
                   tensor core's adder need not round to nearest), so <= (n + 1) 2u S; SIMT (gemm 1): Kpad fmaf in
                   one chain, <= Kpad u S, taken twice.
  epilogue         bias and row bias additions 2u (|acc| + |bias| + |row_bias|); the GELU has slope <= 1.13 (taken
                   as 1.2) and evaluates within 2^-21 |v|; the residual addition and the fp32 store 2^-22 (|r| + |y|);
                   the split of the output: lo holds y - hi (<= 2^-8 |y|) to 8 bits, so hi + lo is within 2^-17 |y|.
  bound = g [L + c_acc S + 2^-22 (|acc| + |bias| + |row_bias|)] + a 2^-21 |v| + 2^-22 (|r| + |y|) + s 2^-17 |y|
  with g = 1.2 and a = 1 with an activation (else 1 and 0), s = 1 for a split output.
  Besides the bound: split outputs are well formed (|lo| <= ulp_bf16(hi) / 2), residual outputs keep the random prefill
  they are added to, and every byte outside the output the layer owns keeps its sentinel.

Time attention (per track n and head h; q, k, v are the fp32 results of the q|k|v GEMM above, with the GEMM bound
dq, dk, dv of each element):
  logit error  ds_ij = (sum_d dq_id |k_jd| + |q_id| dk_jd + dq_id dk_jd + 48 u |q_id k_jd|) / sqrt(48) + 2^-22 |s_ij|
               (48 fp32 fmas; the fp32 scale by log2(e)); D = max_ij ds_ij.
  output       a logit perturbation of at most D moves the softmax weights by at most expm1(2 D) in sum, so
               |do| <= expm1(2 D) vmax + max dv + (T + 16) 2u vmax (exp2, the sum l and the P V fmas) + 2^-17 |o|,
               vmax = max |v| of the track and head.  The separate kernels (fuse 0, T > 128, gemm 1) round q, k, P and V
               to split bf16 on top: + 2 (1 + Labs) 2^-16 vmax, Labs = max_ij sum_d |q_id k_jd| / sqrt(48), as in
               test_gpu_attention.py.
  Besides the bound: every output is finite, and rows after the last one are untouched.

LayerNorm (per element; z the normalised value, A = mean |x| of the row, sigma = sqrt(var + eps)):
  the fp32 mean of 384 values (12 per lane, 5 shuffle levels) is off by <= 16 u A, which moves z by 16 u A / sigma;
  sum of squares, rsqrtf (2 ulp) and the products move z by < 2^-20 |z|; + beta 2u |beta|; split 2^-17 |y|.
  bound = |gamma| 2^-19 (|z| + A / sigma) + 2^-22 |beta| + 2^-17 |y|   (2x margin on the first two terms).
  A / sigma is where a large common offset shows: the fp32 mean loses those bits, and so does any fp32 LayerNorm.

The dispatch map restates which kernel each case reaches (gemm.cu: gemm_launch; api_loop.cu: time_attention); the GPU
tests print the branch and err / bound of every case and assert that the case lists reach every branch on the device
they run on.  A CPU test asserts the same for an H100 SXM (132 SMs) and a PCIe card (114).
"""
import math
import zlib

import pytest
import torch

from body_cases import C, DH, HEADS, acc_bound, ln_ref, planes, qkv64, round16, time_reference

DEV = "cuda:0"
BF16_SENTINEL = 0x7FA5                 # a bf16 NaN: no kernel writes it
F32_SENTINEL = 0x7FC0ABCD              # an fp32 NaN


def pad64(k):
    return (k + 63) // 64 * 64


def assert_well_formed(hi, lo, what):
    """|lo| <= ulp_bf16(hi) / 2 elementwise (hi = m 2^e with m in [0.5, 1): ulp = 2^(e-8)); lo = 0 where hi = 0"""
    h, l = hi.double(), lo.double()
    _, e = torch.frexp(h)
    ok = torch.where(h == 0, l == 0, l.abs() <= torch.ldexp(torch.ones_like(h), e - 9))
    assert bool(ok.all()), f"{what}: {int((~ok).sum())} split elements with |lo| > ulp(hi) / 2"


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def eng():
    from cotracker_b200 import engine
    engine.lib()
    return engine


def with_options(eng, opts, fn):
    for k, v in opts.items():
        eng.set_option(k, v)
    try:
        out = fn()
        torch.cuda.synchronize()
    finally:
        for k in opts:
            eng.set_option(k, {"gemm": 0, "attn": 0, "fuse": 1}[k])
    return out


# =====================================================================================================================
# GEMM epilogues: one configuration per production layer
LAYERS = [
    dict(name="q", K=384, N=384),
    dict(name="kv", K=384, N=768),
    dict(name="qkv", K=384, N=1152),
    dict(name="out_proj", K=384, N=384, residual=True),
    dict(name="fc2", K=1536, N=384, residual=True),
    dict(name="fc1", K=384, N=1536, act=2, split=True),
    dict(name="corr_fc1", K=2401, N=384, act=1, split=True, x_range=1),
    dict(name="corr_fc1_fp16x2", K=2401, N=384, act=1, split=True, x_range=1, products=2, fp16=True),
    dict(name="corr_fc1_fp16x1", K=2401, N=384, act=1, split=True, x_range=1, products=1, fp16=True),
    dict(name="corr_fc2", K=384, N=256, split=True, row_group=4, ld_split=2304, lo_off=1152),
    dict(name="input_transform_mod1", K=1110, N=384, row_mod=1),
    dict(name="input_transform_mod7", K=1110, N=384, row_mod=7),
    dict(name="input_transform_mod60", K=1110, N=384, row_mod=60),
] + [dict(name=f"encoder_K{k}", K=k, N=128) for k in (576, 1152, 64, 128, 256)]


def large_m(N, cta=132):
    """rows giving every persistent CTA at least 4 tiles of 128 x 128, with a ragged last row tile"""
    return 128 * -(-4 * cta // (N // 128)) + 37


GEMM_CASES = [(layer, M, impl) for layer in LAYERS for M in (1, 127, 129, large_m(layer["N"])) for impl in (0, 1)]


def gemm_case_id(c):
    layer, M, impl = c
    return f"{layer['name']}-M{M}-gemm{impl}"


def gemm_layout(layer, M):
    """(ld_y, ld_split, lo_off) of a case: production pitches, with padding columns at M = 127 / 129"""
    N, rg = layer["N"], layer.get("row_group", 1)
    pad = M in (127, 129)
    ld_y = N + (4 if pad else 0)
    if "ld_split" in layer:
        return ld_y, layer["ld_split"], layer["lo_off"]
    return ld_y, 2 * rg * N + (16 if pad else 0), rg * N + (8 if pad else 0)


def gemm_branch(layer, M, impl, n_sms):
    b = {"impl": "simt" if impl else "wgmma", "products": layer.get("products", 3),
         "planes": "fp16" if layer.get("fp16") else "bf16",
         "epilogue": "+".join(k for k in ("residual", "split", "row_bias", "act") if layer.get(k) or
                              (k == "row_bias" and "row_mod" in layer)) or "fp32",
         "row_group": layer.get("row_group", 1), "row_mod": layer.get("row_mod", 0), "M": M}
    if impl == 0:
        tiles = -(-M // 128) * (layer["N"] // 128)
        b["tiles_per_cta"] = -(-tiles // min(tiles, n_sms))
    return b


def gemm_coverage(cases, n_sms):
    """every layer at both engines, at M = 1, at a ragged M, and (wgmma) with >= 4 tiles per persistent CTA"""
    missing = []
    for layer in LAYERS:
        for impl in (0, 1):
            bs = [gemm_branch(lay, M, i, n_sms) for lay, M, i in cases if lay is layer and i == impl]
            if not any(b["M"] == 1 for b in bs):
                missing.append(f"{layer['name']} gemm {impl} at M = 1")
            if not any(b["M"] % 128 and b["M"] > 128 for b in bs):
                missing.append(f"{layer['name']} gemm {impl} at a ragged M > 128")
            if impl == 0 and not any(b["tiles_per_cta"] >= 4 for b in bs):
                missing.append(f"{layer['name']} with >= 4 tiles per CTA")
    epis = {gemm_branch(lay, 1, 0, n_sms)["epilogue"] for lay, _, _ in cases}
    missing += [f"epilogue {e}" for e in ("fp32", "residual", "split+act", "split", "row_bias") if e not in epis]
    if not any(lay.get("row_mod", 0) > 1 and M % lay["row_mod"] for lay, M, _ in cases):
        missing.append("row_mod > 1 with M not a multiple of it")
    return missing


def test_gemm_cases_cover_every_branch_on_h100s():
    for n in (132, 114):
        assert gemm_coverage(GEMM_CASES, n) == [], n


@pytest.mark.gpu
def test_gemm_cases_reach_every_branch_on_this_device():
    n = sms()
    print(f"\n{n} SMs")
    for c in GEMM_CASES:
        b = gemm_branch(*c, n)
        print(f"  {gemm_case_id(c)}: " + " ".join(f"{k}={v}" for k, v in b.items()))
    assert gemm_coverage(GEMM_CASES, n) == []


@pytest.mark.gpu
@pytest.mark.parametrize("case", GEMM_CASES, ids=[gemm_case_id(c) for c in GEMM_CASES])
def test_gemm_epilogue_matches_fp64(eng, case):
    layer, M, impl = case
    K, N = layer["K"], layer["N"]
    Kpad, P, fp16, act = pad64(K), layer.get("products", 3), layer.get("fp16", False), layer.get("act", 0)
    rg, row_mod, residual, split = layer.get("row_group", 1), layer.get("row_mod", 0), layer.get("residual", False), \
        layer.get("split", False)
    ld_y, ld_split, lo_off = gemm_layout(layer, M)
    g = torch.Generator(device=DEV).manual_seed(zlib.crc32(gemm_case_id(case).encode()))
    f64 = dict(device=DEV, dtype=torch.float64, generator=g)

    # operands: x [M, Kpad] (zero padding as in the update loop), w [N, Kpad] of output scale 1 (0.05 under a GELU, whose
    # input is then mostly the bias, spread over where the two GELUs differ most)
    x = torch.zeros(M, Kpad, device=DEV, dtype=torch.float64)
    x[:, :K] = (torch.rand(M, K, **f64) * 2 - 1) if layer.get("x_range") else torch.randn(M, K, **f64)
    w = torch.zeros(N, Kpad, device=DEV, dtype=torch.float64)
    w[:, :K] = torch.randn(N, K, **f64) * ((0.05 if act else 1.0) / math.sqrt(K))
    x_hi, x_lo = planes(x, fp16)
    w_hi, w_lo = planes(w, fp16)
    if P == 3:
        x_split, x_ld, xu = torch.cat([x_hi, x_lo], 1).contiguous(), 0, x_hi.double() + x_lo.double()
    else:                                           # a single activation plane of pitch Kpad
        x_split, x_ld, xu = x_hi.contiguous(), Kpad, x_hi.double()
    w_split = torch.cat([w_hi, w_lo], 1).contiguous()
    wu = w_hi.double() + (w_lo.double() if P >= 2 else 0)
    bias = (torch.randn(N, **f64) * (2.0 if act else 1.0)).float()
    row_bias = torch.randn(max(row_mod, 1), N, **f64).float() if row_mod else None

    # outputs, prefilled with sentinels (and the residual where the layer accumulates)
    y = y_split = r0 = None
    if split:
        rows_out = -(-M // rg)
        y_split = torch.full((rows_out + 3, ld_split), BF16_SENTINEL, dtype=torch.int16, device=DEV)
        y_split = y_split.view(torch.bfloat16)    # the split output is bf16 whatever the operand planes
    else:
        y = torch.full((M + 3, ld_y), F32_SENTINEL, dtype=torch.int32, device=DEV).view(torch.float32)
        if residual:
            r0 = torch.randn(M, N, **f64).float()
            y[:M, :N] = r0
    y_before = None if y is None else y.clone()
    ys_before = None if y_split is None else y_split.clone()

    with_options(eng, {"gemm": impl}, lambda: eng.linear_ex(
        x_split, w_split, bias, M, N, Kpad, x_ld=x_ld, products=P, fp16=fp16, act=act, row_bias=row_bias,
        row_mod=max(row_mod, 1), y=y, ld_y=ld_y, residual=residual, y_split=y_split, ld_split=ld_split, lo_off=lo_off,
        row_group=rg))

    # float64 reference and elementwise bound
    acc = xu @ wu.t()
    S = xu.abs() @ wu.abs().t()
    rb = row_bias.double()[torch.arange(M, device=DEV) % row_mod] if row_mod else torch.zeros_like(acc)
    v = acc + bias.double() + rb
    yv = torch.nn.functional.gelu(v, approximate="tanh" if act == 2 else "none") if act else v
    want = yv + (r0.double() if residual else 0)
    L = x_lo.double().abs() @ w_lo.double().abs().t() if (P == 3 and impl == 0) else 0.0
    gs = 1.2 if act else 1.0
    bd = gs * (L + acc_bound(impl, P, Kpad) * S + 2.0 ** -22 * (acc.abs() + bias.double().abs() + rb.abs()))
    bd = bd + (2.0 ** -21 * v.abs() if act else 0) + 2.0 ** -22 * (want.abs() + (r0.double().abs() if residual else 0))

    if split:
        r = torch.arange(M, device=DEV)
        cols = (r % rg)[:, None] * N + torch.arange(N, device=DEV)[None]
        hi, lo = y_split[(r // rg)[:, None], cols], y_split[(r // rg)[:, None], lo_off + cols]
        assert_well_formed(hi, lo, gemm_case_id(case))
        got = hi.double() + lo.double()
        bd = bd + 2.0 ** -17 * want.abs()
        owned = torch.zeros(y_split.shape, dtype=torch.bool, device=DEV)
        owned[(r // rg)[:, None], cols] = True
        owned[(r // rg)[:, None], lo_off + cols] = True
        after, before = y_split.view(torch.int16), ys_before.view(torch.int16)
    else:
        got = y[:M, :N].double()
        owned = torch.zeros(y.shape, dtype=torch.bool, device=DEV)
        owned[:M, :N] = True
        after, before = y.view(torch.int32), y_before.view(torch.int32)
    assert bool(torch.equal(after[~owned], before[~owned])), "a byte outside the layer's output changed"
    assert bool(torch.isfinite(got).all()), "non-finite output"
    if residual:   # the prefill is in the result: without it the error would be |r0| >> bound
        assert float(r0.double().abs().max()) > 100 * float(bd.max())
    err = (got - want).abs()
    ratio = err / bd
    worst = int(ratio.argmax())
    q = float(ratio.max())
    print(f"\n  {gemm_case_id(case)} [{' '.join(f'{k}={v}' for k, v in gemm_branch(*case, sms()).items())}] "
          f"max err={float(err.max()):.3e} max|y|={float(want.abs().max()):.3e} worst element err={float(err.view(-1)[worst]):.3e} "
          f"bound={float(bd.view(-1)[worst]):.3e} ({q:.3f} of it)")
    assert q <= 1.0, (gemm_case_id(case), q)


# =====================================================================================================================
# fused q|k|v projection + time attention
def ta_branch(T, tracks, fuse, gemm):
    """what ct3_time_block_attention runs (api_loop.cu: time_attention; gemm.cu: gemm_qkv_time_attn_launch)"""
    if fuse == 1 and gemm == 0 and T <= 128:
        R = (128 // T) * T
        rows = T * tracks
        return {"path": "fused", "R": R, "clamped_rows": 128 - R, "chunks": -(-T // 8), "masked_tail": T % 8,
                "ragged": rows % R != 0, "tiles": -(-rows // R) * HEADS}
    return {"path": "unfused", "gemm": "simt" if gemm else "wgmma", "kb": 16 if T <= 16 else 32 if T <= 32 else 64}


REGIMES = ("soft", "sharp30", "sharp80", "dominant", "underflow_first", "underflow_last")
TA_CASES = []   # (T, tracks, depth, regime, fuse, gemm)
for _i, _t in enumerate((1, 2, 3, 7, 8, 9, 16, 43, 60, 64, 65, 100, 127, 128)):
    TA_CASES.append((_t, 3 * (128 // _t) + 1, _i % 3, "soft", 1, 0))        # ragged last tile (T <= 64)
TA_CASES += [(60, 6400 + 64, 0, "soft", 1, 0),                              # headline size
             (129, 37, 1, "soft", 1, 0), (150, 37, 2, "soft", 1, 0),         # T > 128: separate kernels
             (16, 37, 0, "soft", 0, 0), (60, 37, 1, "soft", 0, 0),           # fuse = 0
             (8, 37, 2, "soft", 1, 1), (43, 37, 0, "soft", 1, 1)]            # gemm = 1
for _r in REGIMES[1:]:
    TA_CASES += [(9, 29, 1, _r, 1, 0), (60, 21, 2, _r, 1, 0), (128, 5, 0, _r, 1, 0), (150, 7, 1, _r, 1, 0)]


def ta_case_id(c):
    T, n, depth, regime, fuse, gemm = c
    return f"T{T}-tracks{n}-depth{depth}-{regime}-fuse{fuse}-gemm{gemm}"


def ta_coverage(cases, n_sms):
    bs = [(c, ta_branch(c[0], c[1], c[4], c[5])) for c in cases]
    fused = [b for _, b in bs if b["path"] == "fused"]
    missing = []
    checks = {
        "T = 1": any(b["R"] == 128 and b["chunks"] == 1 and b["masked_tail"] == 1 for b in fused),
        "one track per tile (T = 128)": any(b["R"] == 128 and b["chunks"] == 16 for b in fused),
        "clamped rows past R": any(b["clamped_rows"] > 0 for b in fused),
        "ragged last tile": any(b["ragged"] for b in fused),
        "one 8-key chunk with a masked tail": any(b["chunks"] == 1 and b["masked_tail"] for b in fused),
        "several chunks, masked tail": any(b["chunks"] > 1 and b["masked_tail"] for b in fused),
        "several chunks, no masked tail": any(b["chunks"] > 1 and not b["masked_tail"] for b in fused),
        ">= 4 tiles per persistent CTA": any(b["tiles"] >= 4 * n_sms for b in fused),
        "T > 128": any(b["path"] == "unfused" and c[0] > 128 for c, b in bs),
        "fuse = 0": any(c[4] == 0 for c, _ in bs),
        "gemm = 1": any(b["path"] == "unfused" and b["gemm"] == "simt" for _, b in bs),
    }
    for kb in (16, 64):
        checks[f"separate kernels at KB = {kb}"] = any(b["path"] == "unfused" and b["kb"] == kb for _, b in bs)
    for r in REGIMES:
        checks[f"{r} on the fused kernel over several chunks"] = any(
            c[3] == r and b["path"] == "fused" and b["chunks"] > 1 for c, b in bs)
    missing += [k for k, ok in checks.items() if not ok]
    return missing


def test_time_attention_cases_cover_every_branch_on_h100s():
    for n in (132, 114):
        assert ta_coverage(TA_CASES, n) == [], n


@pytest.mark.gpu
def test_time_attention_cases_reach_every_branch_on_this_device():
    n = sms()
    print(f"\n{n} SMs")
    for c in TA_CASES:
        print(f"  {ta_case_id(c)}: " + " ".join(f"{k}={v}" for k, v in ta_branch(c[0], c[1], c[4], c[5]).items()))
    assert ta_coverage(TA_CASES, n) == []


@pytest.fixture(scope="module")
def base_state():
    from cotracker_b200.synthetic import seeded_state_dict
    return seeded_state_dict(17, offline=True, window_len=60)


def time_inputs(T, n, regime, g):
    """-> the crafted split operand x_split [rows, 768] and float64 weights exact to 16 bits (wq [384, 384], bq,
    wkv [768, 384], bkv) of the regime"""
    f64 = dict(device=DEV, dtype=torch.float64, generator=g)
    rows = n * T
    x = torch.randn(rows, C, **f64)
    wq, wkv = torch.randn(C, C, **f64) / math.sqrt(C), torch.randn(2 * C, C, **f64) / math.sqrt(C)
    bq, bkv = torch.randn(C, **f64) * 0.1, torch.randn(2 * C, **f64) * 0.1
    if regime in ("dominant", "underflow_first", "underflow_last"):
        # feature column 0 of x carries a per-key value a_j; to_k maps it onto a unit direction u_h in every head, the q
        # bias points every query along u_h and the rest of q and k is small: logit_ij ~ 56 a_j
        u = torch.randn(HEADS, DH, **f64)
        u = (u / u.norm(dim=1, keepdim=True)).reshape(C)
        t = torch.arange(T, device=DEV)
        if regime == "dominant":   # one key per track at logit 30, the rest ~N(0, 4.3)
            a = torch.randn(n, T, **f64) * (4.3 / 56)
            hot = torch.randint(0, T, (n,), device=DEV, generator=g)
            a[torch.arange(n, device=DEV), hot] = 30 / 56
        else:   # the keys of the first or the last 8-key chunk at ~ +56, every other key at ~ -56: exp(-112) = 0 in fp32
            first = 0 if regime == "underflow_first" else ((T - 1) // 8) * 8
            sign = torch.where((t >= first) & (t < first + 8), 1.0, -1.0).double()
            a = sign[None] + 0.02 * torch.randn(n, T, **f64)
        x[:, 0] = a.reshape(rows)
        wq = wq * 0.01
        bq = 56 * math.sqrt(DH) * u
        wkv[:C] *= 0.01
        wkv[:C, 0] = u
        bkv[:C] = 0
    xh, xl = planes(x)
    x = xh.double() + xl.double()
    if regime.startswith("sharp"):   # q weights and bias scaled so that max |logit| is the target
        q, k, *_ = qkv64(x, wq, bq, wkv, bkv)
        m = float(torch.einsum("nihd,njhd->nhij", q.view(n, T, HEADS, DH), k.view(n, T, HEADS, DH)).abs().max())
        s = float(regime[5:]) / (m / math.sqrt(DH))
        wq, bq = wq * s, bq * s
    wq, bq, wkv, bkv = (round16(w).float().double() for w in (wq, bq, wkv, bkv))
    return torch.cat([xh, xl], 1).contiguous(), wq, bq, wkv, bkv


@pytest.mark.gpu
@pytest.mark.parametrize("case", TA_CASES, ids=[ta_case_id(c) for c in TA_CASES])
def test_time_block_attention_matches_fp64(eng, base_state, case):
    T, n, depth, regime, fuse, gemm = case
    g = torch.Generator(device=DEV).manual_seed(zlib.crc32(ta_case_id(case).encode()))
    x_split, wq, bq, wkv, bkv = time_inputs(T, n, regime, g)
    p = f"updateformer.time_blocks.{depth}.attn."
    sd = dict(base_state)
    sd.update({p + "to_q.weight": wq.float(), p + "to_q.bias": bq.float(), p + "to_kv.weight": wkv.float(),
               p + "to_kv.bias": bkv.float()})
    packed = eng.pack_weights(sd, DEV)
    rows, guard = n * T, 64
    out = torch.full((rows + guard, 2 * C), BF16_SENTINEL, dtype=torch.int16, device=DEV).view(torch.bfloat16)
    with_options(eng, {"fuse": fuse, "gemm": gemm}, lambda: eng.time_block_attention(packed, depth, x_split, T, out=out))
    assert bool((out[rows:].view(torch.int16) == BF16_SENTINEL).all()), "a row after the last one was written"
    got = out[:rows, :C].double() + out[:rows, C:].double()
    assert bool(torch.isfinite(got).all()), "non-finite output"
    b = ta_branch(T, n, fuse, gemm)
    want, bd, lmax = time_reference(x_split, wq, bq, wkv, bkv, T, n, b["path"] == "fused", gemm)
    err = (got - want).abs()
    q = float((err / bd).max())
    print(f"\n  {ta_case_id(case)} [{' '.join(f'{k}={v}' for k, v in b.items())}] max|logit|={lmax:.1f} "
          f"max err={float(err.max()):.3e} min bound={float(bd.min()):.3e} ({q:.3f} of it)")
    assert q <= 1.0, (ta_case_id(case), q)


# =====================================================================================================================
# LayerNorm
ROW_KINDS = ("normal", "var1e-5", "var1e-6", "var1e-7", "constant", "offset")
LN_CASES = [(rows, eps, affine) for rows in (1, 7, 8, 9, 1000, 100003) for eps in (1e-6, 1e-5) for affine in (0, 1)]


def ln_rows(rows, g):
    """[rows, 384] fp32, row i of kind ROW_KINDS[i % 6]: N(0, 1); N(0, 1) scaled to variance 1e-5 / 1e-6 / 1e-7 (eps
    decides the result); a constant; N(0, 1) on a common offset of +-1000"""
    f64 = dict(device=DEV, dtype=torch.float64, generator=g)
    x = torch.randn(rows, C, **f64)
    kind = torch.arange(rows, device=DEV) % len(ROW_KINDS)
    for k, var in ((1, 1e-5), (2, 1e-6), (3, 1e-7)):
        x[kind == k] *= math.sqrt(var)
    x[kind == 4] = 3 * torch.randn(rows, 1, **f64).expand(rows, C)[kind == 4]
    x[kind == 5] += 1000 * torch.sign(torch.randn(rows, 1, **f64)).expand(rows, C)[kind == 5]
    return x.float()


@pytest.mark.gpu
@pytest.mark.parametrize("rows,eps,affine", LN_CASES)
def test_layernorm_matches_fp64(eng, rows, eps, affine):
    g = torch.Generator(device=DEV).manual_seed(rows * 10 + affine + int(eps * 1e6))
    x = ln_rows(rows, g)
    gamma = beta = None
    if affine:   # a trained-like affine: gamma around 1, some negative; beta of the same order
        gamma = (1 + 0.7 * torch.randn(C, device=DEV, dtype=torch.float64, generator=g)).float()
        beta = (0.5 * torch.randn(C, device=DEV, dtype=torch.float64, generator=g)).float()
        assert bool((gamma < 0).any())
    out = eng.layernorm(x, gamma, beta, eps)
    torch.cuda.synchronize()
    hi, lo = out[:, :C], out[:, C:]
    assert_well_formed(hi, lo, "layernorm")
    got = hi.double() + lo.double()
    want, bd = ln_ref(x.double(), eps, gamma.double() if affine else None, beta.double() if affine else None)
    err = (got - want).abs()
    ratio = err / bd
    kind = torch.arange(rows, device=DEV) % len(ROW_KINDS)
    parts = []
    for k, name in enumerate(ROW_KINDS):
        if bool((kind == k).any()):
            parts.append(f"{name} {float(ratio[kind == k].max()):.3f}")
    print(f"\n  layernorm rows={rows} eps={eps:g} affine={affine}: max err={float(err.max()):.3e}; err / bound by row "
          f"kind: {', '.join(parts)}")
    assert float(ratio.max()) <= 1.0
