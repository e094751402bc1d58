"""Every attention kernel on its own (ct3_attention) against softmax(q k^T / sqrt(48)) v computed in float64, over the
dispatch matrix of the transformer body and at sharp logits; and the whole EfficientUpdateFormer at sharp attention
against the float64 oracle.

The branch map (tests/body_cases.py) restates, in Python, how the host picks a kernel (attention_tc.cu: attention_tc_splits and
launch_attention_tc; api_loop.cu: run_attention, space_attention, plan_groups).  A CPU test pins it to values computed by
the C++; the GPU test prints the branch of every case and asserts that the case list reaches every branch on the
device it runs on, so a change to the heuristics cannot silently drop one from coverage.

Tolerances (err = max |got - want| over the written rows, want in float64):
  Labs  = max over (sequence, head, query, key) of sum_d |q_d k_d| / sqrt(48), the scale of a logit's rounding error;
  vmax  = max |v|, the scale of the output.
  attn 0 (split-bf16x3 tensor cores): q, k, P and V are each held as hi + lo bf16 pairs, 2^-18 relative, and the
    lo*lo product is dropped, so a logit is off by at most ~3 * 2^-18 * Labs < 2^-16 * Labs.  A probability
    exp(s - m) / l carries that error twice (numerator and sum), and P V adds 2^-16 * vmax for its own splits and the
    split of the output:   err <= 2 * (1 + Labs) * 2^-16 * vmax.
  attn 1 (fp32 SIMT): the same terms at fp32 rounding.  A 48-term dot product, a Lk-term sum of P V and the split of
    the output (2^-17 relative): rounding errors of independent terms add like a random walk, sqrt(n) * 2^-24, and a
    margin of 4 covers it:   err <= (2^-17 + 4 * 2^-24 * (sqrt(48) * (1 + Labs) + sqrt(Lk))) * vmax.
"""
import math
import zlib

import pytest
import torch

from body_cases import C, DH, HEADS, KV, P_FROM_V, TIME, V_FROM_P, V_SELF, bound, branch, describe, tc_qtw, tc_splits
from cases import O

DEV = "cuda:0"
KIND_NAMES = {TIME: "time", V_FROM_P: "virtual<-point", V_SELF: "virtual self", P_FROM_V: "point<-virtual"}


def coverage(branches):
    """The branches a case list must reach; -> list of the ones it misses."""
    missing = []
    pw = [b for b in branches if b["path"] == "per_warp"]
    for kb in (16, 32, 64):
        if not any(b["kb"] == kb for b in pw):
            missing.append(f"per-warp KB={kb}")
    for T in (1, 2, 129, 150, 200):
        if not any(b["T"] == T for b in pw):
            missing.append(f"time attention at T={T}")
    qtws = {b["qtw"] for b in branches if "qtw" in b}
    missing += [f"qtw={q}" for q in (1, 8) if q not in qtws]
    if not any(b["path"] == "split_k" for b in branches):
        missing.append("ungrouped split-K")
    if not any(b["path"] == "grouped_split_k" and len(set(b["group_splits"])) >= 3 and 1 in b["group_splits"]
               for b in branches):
        missing.append("grouped split-K with >= 3 distinct counts including 1")
    if not any(b["path"] == "grouped_p2v" and b["wgmma_groups"] >= 2 and b["mma_groups"] >= 1 for b in branches):
        missing.append("grouped point<-virtual with >= 2 wgmma groups and mma.sync groups")
    if not any(b["path"] == "wgmma" for b in branches):
        missing.append("ungrouped point<-virtual on wgmma")
    if not any(b["path"] == "simt" for b in branches):
        missing.append("exact-fp32 SIMT")
    return missing


# ---------------------------------------------------------------------------------------------------------------------
# cases: (kind, T, N, group sizes or None, logit regime, attn)
MIXED = (3000, 1, 449, 448, 700, 64, 65, 90)
CASES = []
for _n in (1, 15, 16, 17, 63, 64, 65, 127, 128, 129, 1030, 3000):      # ragged query tiles of point<-virtual
    CASES.append((P_FROM_V, 8, _n, None, "soft", 0))
for _n in (1, 64, 65, 448, 449, 1030, 6400):                           # key counts around chunk and split boundaries
    CASES.append((V_FROM_P, 16, _n, None, "soft", 0))
CASES += [(V_SELF, 8, 5, None, "soft", 0), (V_SELF, 66, 3, None, "soft", 0), (V_SELF, 16, 40, None, "soft", 1)]
for _t in (1, 2, 16, 17, 32, 33, 64, 65, 128, 129, 150, 200):          # time attention: KB 16 / 32 / 64, 1..4 chunks
    CASES.append((TIME, _t, 37, None, "soft", 0))
CASES += [(TIME, 150, 37, None, "soft", 1), (TIME, 17, 37, None, "soft", 1)]
for _t in (16, 48):                                                    # full size
    for _attn in (0, 1):
        CASES.append((P_FROM_V, _t, 6400, None, "soft", _attn))
        CASES.append((V_FROM_P, _t, 6400, None, "soft", _attn))
for _regime in ("sharp30", "sharp80", "dominant", "underflow_last", "underflow_first"):
    CASES += [(TIME, 17, 37, None, _regime, 0), (TIME, 65, 37, None, _regime, 0), (TIME, 150, 37, None, _regime, 0),
              (TIME, 200, 20, None, _regime, 0), (TIME, 150, 37, None, _regime, 1),
              (V_FROM_P, 16, 449, None, _regime, 0), (V_FROM_P, 16, 1030, None, _regime, 0),
              (V_FROM_P, 16, 6400, None, _regime, 0), (V_FROM_P, 48, 6400, None, _regime, 0),
              (V_FROM_P, 16, 6400, None, _regime, 1), (V_FROM_P, 8, sum(MIXED), MIXED, _regime, 0),
              (P_FROM_V, 16, 17, None, _regime, 0), (P_FROM_V, 16, 1030, None, _regime, 0),
              (P_FROM_V, 16, 6400, None, _regime, 1)]
    if not _regime.startswith("underflow"):   # 64 keys are one chunk: nothing to underflow across
        CASES += [(V_SELF, 8, 5, None, _regime, 0), (V_SELF, 66, 3, None, _regime, 0)]
CASES = list(dict.fromkeys(CASES))   # the full-size loop repeats two shapes of the lists above
GROUP_CASES = [(kind, T, attn) for kind in (V_FROM_P, V_SELF, P_FROM_V) for T in (8, 16) for attn in (0, 1)]


def case_id(c):
    kind, T, N, sizes, regime, attn = c
    return f"{KIND_NAMES[kind].replace(' ', '_').replace('<-', '_from_')}-T{T}-N{N}{'-grouped' if sizes else ''}-{regime}-attn{attn}"


# ---------------------------------------------------------------------------------------------------------------------
# the float64 reference
def widths(kind):
    """(q row width, q col, kv row width, k col, v col) of the kind's buffers, as the body lays them out"""
    return (3 * C, 0, 3 * C, C, 2 * C) if kind in (TIME, V_SELF) else (C, 0, 2 * C, 0, C)


def sequences(kind, T, N, sizes):
    """-> per group: (query row index [S, Lq], key row index [S, Lk]) of its sequences (int64, on DEV)"""
    sizes = list(sizes) if sizes is not None else [N]
    G = len(sizes)
    t = torch.arange(T, device=DEV)
    if kind == TIME:   # sequence = track (points and every group's virtual tokens), rows n*T + t
        rows = torch.arange(N + KV * G, device=DEV)[:, None] * T + t[None]
        return [(rows, rows)]
    out, off = [], 0
    for g, n in enumerate(sizes):
        pts = (off + torch.arange(n, device=DEV))[None, :] * T + t[:, None]           # [T, n]
        virt = (N + KV * g + torch.arange(KV, device=DEV))[None, :] * T + t[:, None]   # [T, 64]
        out.append({V_FROM_P: (virt, pts), V_SELF: (virt, virt), P_FROM_V: (pts, virt)}[kind])
        off += n
    return out


def gather(buf, rows, col):
    S, L = rows.shape
    return buf[rows.reshape(-1), col:col + C].double().view(S, L, HEADS, DH)


def scatter(buf, rows, col, x):
    buf[rows.reshape(-1), col:col + C] = x.reshape(-1, C).to(buf.dtype)


def reference(kind, q, kv, T, N, sizes):
    """-> (want [rows, 384] float64 with 0 on rows the kind does not write, per-group list of (query rows, Labs, vmax,
    Lk, max|logit|))"""
    _, qc, _, kc, vc = widths(kind)
    want = torch.zeros(q.shape[0], C, dtype=torch.float64, device=DEV)
    stats = []
    for qr, kr in sequences(kind, T, N, sizes):
        Q, K, V = gather(q, qr, qc), gather(kv, kr, kc), gather(kv, kr, vc)
        logits = torch.einsum("sihd,sjhd->shij", Q, K) / math.sqrt(DH)
        labs = float(torch.einsum("sihd,sjhd->shij", Q.abs(), K.abs()).max()) / math.sqrt(DH)
        out = torch.einsum("shij,sjhd->sihd", torch.softmax(logits, dim=-1), V)
        want[qr.reshape(-1)] = out.reshape(-1, C)
        stats.append((qr, labs, float(V.abs().max()), K.shape[1], float(logits.abs().max())))
        del logits
    return want, stats


# ---------------------------------------------------------------------------------------------------------------------
# inputs: N(0, 1) token rows (logits of std 1, max about 5), then the regime reshapes q and k of every sequence
def apply_regime(regime, Q, K, g):
    """Q [S, Lq, 8, 48], K [S, Lk, 8, 48] float64 -> new (Q, K)"""
    if regime == "soft":
        return Q, K
    if regime.startswith("sharp"):   # q scaled so that max |logit| is the target
        target = float(regime[5:])
        m = float((torch.einsum("sihd,sjhd->shij", Q, K).abs().max())) / math.sqrt(DH)
        return Q * (target / m), K
    S, Lq, Lk = Q.shape[0], Q.shape[1], K.shape[1]
    if regime == "dominant":         # every query row is a multiple of one key: that key's logit is 30, the rest ~N(0, 4.3)
        j = torch.randint(0, Lk, (S, Lq), generator=g, device=DEV)
        Kj = torch.gather(K, 1, j[:, :, None, None].expand(S, Lq, HEADS, DH))
        return Kj * (30 * math.sqrt(DH) / (Kj * Kj).sum(-1, keepdim=True)), K
    # underflow: q ~ 8 u (u a unit vector per sequence and head), k_j ~ c_j sqrt(48)/8 u, so logit_j ~ c_j.  The keys of
    # one 64-key chunk (the last or the first) have c ~ +56, every other key c ~ -56: their probabilities are
    # exp(-112) = 0 in fp32 while the hot chunk (and the split that holds it) carries the whole softmax.
    u = torch.randn(S, 1, HEADS, DH, generator=g, device=DEV, dtype=torch.float64)
    u = u / u.norm(dim=-1, keepdim=True)
    Qn = 8 * u + 0.01 * torch.randn(Q.shape, generator=g, device=DEV, dtype=torch.float64)
    hot = torch.zeros(Lk, dtype=torch.bool, device=DEV)
    first = ((Lk - 1) // 64) * 64 if regime == "underflow_last" else 0
    hot[first:first + 64] = True
    c = torch.where(hot, 56.0, -56.0)[None, :, None] + torch.randn(S, Lk, HEADS, generator=g, device=DEV,
                                                                   dtype=torch.float64)
    Kn = c[..., None] * (math.sqrt(DH) / 8) * u + 0.05 * torch.randn(K.shape, generator=g, device=DEV, dtype=torch.float64)
    return Qn, Kn


def make_inputs(kind, T, N, sizes, regime, seed):
    G = len(sizes) if sizes is not None else 1
    rows = (N + KV * G) * T
    wq, qc, wkv, kc, _ = widths(kind)
    g = torch.Generator(device=DEV).manual_seed(seed)
    q = torch.randn(rows, wq, generator=g, device=DEV)
    kv = q if kind in (TIME, V_SELF) else torch.randn(rows, wkv, generator=g, device=DEV)   # one q|k|v buffer, as the body
    if regime != "soft":
        for qr, kr in sequences(kind, T, N, sizes):
            Qn, Kn = apply_regime(regime, gather(q, qr, qc), gather(kv, kr, kc), g)
            scatter(q, qr, qc, Qn)
            scatter(kv, kr, kc, Kn)
    return q, kv


# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def eng():
    from cotracker_b200 import engine
    engine.lib()
    return engine


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def run(eng, kind, q, kv, T, N, sizes, attn):
    eng.set_option("attn", attn)
    try:
        got = eng.attention(kind, q, kv, T, N, group_sizes=sizes)
        torch.cuda.synchronize()
    finally:
        eng.set_option("attn", 0)
    return got


def check(eng, case, q, kv):
    """-> (output, per group (err, bound, group)); prints each group's branch, error and bound"""
    kind, T, N, sizes, regime, attn = case
    got = run(eng, kind, q, kv, T, N, sizes, attn)
    want, stats = reference(kind, q, kv, T, N, sizes)
    written = torch.zeros(q.shape[0], dtype=torch.bool, device=DEV)
    for qr, *_ in stats:
        written[qr.reshape(-1)] = True
    assert bool(torch.isfinite(got).all()), "non-finite output"
    assert bool((got[~written] == 0).all()), "a row outside the kind's queries was written"
    b = branch(kind, T, N, sizes, attn, sms())
    errs = []
    for gi, (qr, labs, vmax, lk, lmax) in enumerate(stats):
        rows = qr.reshape(-1)
        err = float((got[rows].double() - want[rows]).abs().max())
        bd = bound(attn, labs, vmax, lk)
        print(f"  {case_id(case)} group {gi} [{describe(b)}] max|logit|={lmax:.1f} Labs={labs:.1f} "
              f"err={err:.3e} bound={bd:.3e} ({err / bd:.3f} of it)")
        errs.append((err, bd, gi))
    return got, errs


def test_branch_map_matches_the_cpp():
    """The restatement against attention_tc_splits as the compiled library computes it (attention_tc.cu), and the
    qtw / KB / wgmma rules at their thresholds."""
    want = {(16, 64, 6400, 132): 4, (48, 64, 6400, 132): 1, (16, 64, 1030, 132): 4, (8, 64, 3000, 132): 8,
            (8, 64, 449, 132): 4, (8, 64, 448, 132): 1, (8, 64, 700, 132): 4, (16, 64, 3000, 132): 4,
            (1, 64, 100000, 132): 32, (32, 64, 6400, 132): 2, (33, 64, 6400, 132): 1, (16, 64, 6400, 114): 7,
            (8, 64, 3000, 78): 4, (4, 64, 1000, 16): 1, (16, 64, 512, 132): 4, (16, 64, 513, 132): 3}
    assert {k: tc_splits(*k) for k in want} == want
    # qtw: T sequences x 8 heads x ceil(q_tiles / (8 qtw)) CTAs must stay >= 4 per SM
    assert [tc_qtw(16, n, 64, 132) for n in (300, 512, 513, 1024, 1025, 2048, 2049, 6400)] == [1, 1, 2, 2, 4, 4, 8, 8]
    assert tc_qtw(65, 64, 64, 132) == 1 and tc_qtw(66, 64, 64, 132) == 8
    assert tc_qtw(16, 6400, 65, 132) == 1                          # two key chunks: K/V are restaged, no qtw
    assert [branch(TIME, t, 5, None, 0, 132)["kb"] for t in (1, 16, 17, 32, 33, 200)] == [16, 16, 32, 32, 64, 64]
    assert branch(P_FROM_V, 16, 65, None, 0, 132) == {"path": "wgmma"}
    assert branch(P_FROM_V, 16, 64, None, 0, 132)["path"] == "shared"
    assert branch(V_FROM_P, 8, sum(MIXED), MIXED, 0, 132)["group_splits"] == [8, 1, 4, 1, 4, 1, 1, 1]
    assert branch(P_FROM_V, 8, sum(MIXED), MIXED, 0, 132) == {"path": "grouped_p2v", "wgmma_groups": 6,
                                                              "mma_groups": 2, "qtw": 1}
    assert branch(V_FROM_P, 16, 100, None, 1, 132) == {"path": "simt"}
    # the case list covers every branch on an H100 SXM (132 SMs) and on a PCIe card (114)
    for n in (132, 114):
        bs = [branch(k, T, N, s, a, n) for k, T, N, s, _, a in CASES]
        bs += [branch(k, T, sum(MIXED), MIXED, a, n) for k, T, a in GROUP_CASES]
        assert coverage(bs) == [], n


@pytest.mark.gpu
def test_cases_reach_every_branch_on_this_device():
    n = sms()
    bs = [branch(k, T, N, s, a, n) for k, T, N, s, _, a in CASES]
    bs += [branch(k, T, sum(MIXED), MIXED, a, n) for k, T, a in GROUP_CASES]
    print(f"\n{n} SMs")
    for c, b in zip(CASES, bs):
        print(f"  {case_id(c)}: {describe(b)}")
    assert coverage(bs) == []


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_attention_matches_fp64(eng, case):
    print()
    q, kv = make_inputs(*case[:5], seed=zlib.crc32(case_id(case).encode()))
    _, errs = check(eng, case, q, kv)
    for err, bd, gi in errs:
        assert err <= bd, (case_id(case), gi, err, bd)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,T,attn", GROUP_CASES, ids=[f"{KIND_NAMES[k]}-T{T}-attn{a}" for k, T, a in GROUP_CASES])
def test_grouped_attention_matches_fp64_and_standalone_calls(eng, kind, T, attn):
    """Groups of mixed sizes in one call: every group against fp64, and (attn 0) bit-identical to an ungrouped call on
    that group's tracks and virtual tokens alone -- the split-K count, chunk ranges and combine order are per group."""
    print()
    N, G = sum(MIXED), len(MIXED)
    case = (kind, T, N, MIXED, "soft", attn)
    q, kv = make_inputs(kind, T, N, MIXED, "soft", seed=T * 10 + kind)
    got, errs = check(eng, case, q, kv)
    for err, bd, gi in errs:
        assert err <= bd, (KIND_NAMES[kind], T, attn, gi, err, bd)
    if attn != 0:
        return
    off = 0
    for g, n in enumerate(MIXED):
        pts, virt = slice(off * T, (off + n) * T), slice((N + KV * g) * T, (N + KV * g + KV) * T)
        qg = torch.cat([q[pts], q[virt]])
        kvg = qg if kv is q else torch.cat([kv[pts], kv[virt]])
        alone = run(eng, kind, qg, kvg, T, n, None, 0)
        mine = torch.cat([got[pts], got[virt]])
        assert torch.equal(mine, alone), (KIND_NAMES[kind], T, g, n)
        off += n


# ---------------------------------------------------------------------------------------------------------------------
# sharp attention through the whole transformer
SHARP = 30.0


def _sharp_state(sd, N, T, x):
    """to_q weight and bias of every attention scaled so that its max |logit| on x reaches about SHARP (measured on the
    float64 oracle; LayerNorm before every attention keeps the later blocks' inputs at the same scale)."""
    seen = {}
    orig = O.attention

    def record(sd_, prefix, xx, ctx, heads=8):
        B, N1, Cc = xx.shape
        q = O.linear(sd_, prefix + ".to_q", xx).reshape(B, N1, heads, -1).permute(0, 2, 1, 3)
        k = O.linear(sd_, prefix + ".to_kv", ctx).chunk(2, dim=-1)[0].reshape(B, ctx.shape[1], heads, -1).permute(0, 2, 1, 3)
        seen[prefix] = max(seen.get(prefix, 0.0), float((q @ k.transpose(-2, -1)).abs().max()) * 48 ** -0.5)
        return orig(sd_, prefix, xx, ctx, heads)

    O.attention = record
    try:
        with torch.no_grad():
            sd = {k: v.double() for k, v in sd.items()}
            for _ in range(2):
                seen.clear()
                O.updateformer(sd, x.double()[None])
                for p, m in seen.items():
                    s = SHARP / m
                    sd[p + ".to_q.weight"] = sd[p + ".to_q.weight"] * s
                    sd[p + ".to_q.bias"] = sd[p + ".to_q.bias"] * s
            seen.clear()
            want = O.updateformer(sd, x.double()[None])[0]
    finally:
        O.attention = orig
    return sd, want, seen


@pytest.fixture(scope="module")
def sharp_cases():
    from cotracker_b200.synthetic import seeded_state_dict
    out = {}
    for N, T in ((130, 40), (40, 150)):
        sd = seeded_state_dict(3, offline=True, window_len=60, head_gain=100.0, vis_gain=100.0)
        x = torch.randn(N, T, 1110, generator=torch.Generator().manual_seed(N + T))
        out[(N, T)] = (x,) + _sharp_state(sd, N, T, x)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("fuse", [0, 1])
@pytest.mark.parametrize("attn", [0, 1])
@pytest.mark.parametrize("N,T", [(130, 40), (40, 150)])
def test_updateformer_at_sharp_attention_matches_fp64(eng, sharp_cases, N, T, fuse, attn):
    """EfficientUpdateFormer with every attention at max |logit| ~ 30 against the oracle in float64.  T = 40 runs the
    fused projection + time attention kernel (fuse 1), T = 150 the separate kernels.  The attention error grows like
    (1 + max|logit|) (module docstring); the soft-logit tolerance of test_updateformer_attention_shapes, 2e-4 x max|delta|
    at max|logit| ~ 5, is scaled by that factor, (1 + 30) / (1 + 5)."""
    x, sd, want, seen = sharp_cases[(N, T)]
    assert min(seen.values()) > 0.8 * SHARP and max(seen.values()) < 1.25 * SHARP, seen
    packed = eng.pack_weights({k: v.float() for k, v in sd.items()}, DEV)
    eng.set_option("fuse", fuse)
    eng.set_option("attn", attn)
    try:
        got = eng.updateformer(packed, x.to(DEV)).cpu().double()
    finally:
        eng.set_option("fuse", 1)
        eng.set_option("attn", 0)
    scale = max(float(want.abs().max()), 1.0)
    err = float((got - want).abs().max())
    bd = 2e-4 * (1 + SHARP) / (1 + 5) * scale
    print(f"\n  updateformer N={N} T={T} fuse={fuse} attn={attn}: max|logit| {min(seen.values()):.1f}..{max(seen.values()):.1f} "
          f"err={err:.3e} bound={bd:.3e} ({err / bd:.3f} of it)")
    assert err <= bd, (N, T, fuse, attn, err, bd)
