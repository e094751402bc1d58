"""The stretch of the update loop from the correlation volume to the point tokens (ct3_loop_tokens, which runs
update_loop's own code), link by link against float64 arithmetic on the kernel's own input to each link, and end to end
against the float64 CPU oracle, for every correlation kernel, volume format, corr_mlp.fc1 weight flavour and product
count, on both GEMM engines.

The branch map below restates in Python which path a call takes (api_loop.cu: effective_prec, Prec; corr.cu:
corr_uses_patch_kernel, launch_corr_sample; corr_tc2.cu: corr_patch_supported): with the default "corr" = 0 and every
pyramid level at least 8x8, corr_tc3.cu runs prec.corr 1 and 2 and corr_tc2.cu prec.corr 3; "corr" 1 and 2 and smaller
pyramids run the SIMT and corr_tc.cu kernels at full precision.  test_host_logic.py pins it to the
compiled ct3_precision_info / ct3_volume_is_support_major; the GPU test prints every case's branch and asserts that the
case list reaches every reachable combination.

Bounds (err = |got - want| per element, want in float64; u = 2^-24; S = sum_k |x_k w_k| + |b| in float64 over the
operands as the GEMM sees them, i.e. the planes it multiplies: x_hi (+ x_lo with 3 products) times w_hi (+ w_lo with 2
or 3), bf16 planes or fp16 ones):
  accumulation  acc(S, n) = LAM * sqrt(n) * 2^-23 * S: n fp32 additions of k16 tensor-core blocks (products * Kpad / 16,
                plus the bias), each off by at most one ulp of a partial sum <= S; independent roundings add like a random
                walk, LAM = 4 is the margin.  The same per-product formula is evaluated exactly in float64, so a wrong
                plane or product count is not inside the bound.
  propagation   rw(W, e) = LAM * sqrt(sum_k W_k^2 e_k^2): independent input errors e through a layer W (random walk).
  corr_mlp      X's correlation columns against fc2(gelu_erf(fc1(v))) with v the volume as the GEMM reads it:
                e1 = acc(S1, n1);  e_h = 1.13 e1 (max |gelu'|) + 2^-21 |a| (fp32 erff) + 2^-17 |h| (split of h);
                e_X = rw(W2, e_h) + 2^-8 |h| . |w2_lo| (the dropped lo*lo product) + acc(S2, n2) + 2^-17 |X| (split of X).
  small columns vis, conf: |err| <= 2^-17 |v| (the split alone).  posenc: u = (c_t - c_t+-1) / (128 | 96) carries two
                fp32 roundings, so an argument x 2^k is off by 2 * |u 2^k| * 2^-23 (margin 2 over 2 * 2^-24); the pi/2
                shift adds 2 * ((|x 2^k| + 2) 2^-24 + 4.4e-8) (the add and fp32(pi/2)); sinf adds 2^-22; the split 2^-17.
                Pad columns 1110..1151 are exactly 0.
  input_transform  tokens against W_in . (X_got + time_emb[t]) + b: acc(S3, 3 * 1152/16 + 2) for the split GEMM,
                40 u S_te for the fp32 row-bias dot product (a worst case: 35 fma per lane and 5 shuffle adds), and
                2^-23 (|W_in X| + |b| + |W_in te|) for the two epilogue adds.
  end to end    tokens against O.correlation_embeddings -> O.transformer_input -> input_transform in float64: the
                volume tolerance of test_corr_sample (EV below, per kernel and format) propagated with rw through fc1,
                plus the rounding of the packed fc1 weights (2^-11 S1 for one fp16 plane, 2^-16 + 2^-17 for bf16 splits,
                2^-21 for fp16 splits), then the link bounds above, with X's error propagated through W_in.
The worst err/bound per (branch, link) is printed (`tokens-worst`).  On an H100 80GB HBM3 at a 700 W power limit:
small columns 0.73-1.0 (the vis / conf split bound is attained), corr_mlp 0.065-0.21, input_transform 0.0075-0.39,
end to end 0.0006-0.021.  Two bounds sit below 1/100 on some branches, for stated reasons: the end-to-end one because EV
is the worst element of test_corr_sample over whole volumes and bounds every element here; input_transform on the
branches whose only cases are N = 1 or a time-embedding case, where the worst-case 40 u S_te of the row-bias dot
product dominates the bound (the mutation with every frame given frame 0's bias fails it by orders of magnitude).
"""
import math
import zlib

import pytest
import torch
import torch.nn.functional as F

from cases import O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
LEVELS, P, VOL, VOL_PAD, HID, XDIM, XPAD = 4, 49, 2401, 2432, 384, 1110, 1152
LAM = 4.0
U = 2.0 ** -24
OPTION_DEFAULTS = {"gemm": 0, "corr": 0, "attn": 0, "prec.corr": 2, "prec.fc1": 3, "fuse": 1}


# ---------------------------------------------------------------------------------------------------------------------
# branch map
def loop_branch(T, H4, W4, corr=0, prec_corr=2, prec_fc1=3, gemm=0):
    """What ct3_loop_tokens / one update_loop iteration runs for these options and this pyramid shape."""
    # the workspace holds the split pyramid iff every level is >= 8x8 texels (corr_patch_supported)
    patch = corr == 0 and (H4 >> 3) >= 8 and (W4 >> 3) >= 8
    pc, pf = (prec_corr, prec_fc1) if patch else (3, 3)
    if patch:
        kernel = "corr_tc3" if pc != 3 else "corr_tc2"
    else:
        kernel = "simt" if corr == 1 else "corr_tc"
    support_major = kernel == "corr_tc3"
    vol16 = pf < 3
    suffix = ("t" if support_major else "") + ("h" if vol16 else "")
    return {"kernel": kernel, "volume": "fp16" if vol16 else "split", "weights": "corr_fc1" + ("_" + suffix if suffix else ""),
            "products": pf, "corr_products": pc, "support_major": support_major, "gemm": "simt" if gemm else "wgmma"}


def branch_key(b):
    return (b["kernel"], b["weights"], b["products"], b["gemm"])


# every reachable (kernel, fc1 weights, fc1 products) combination
REACHABLE = {("corr_tc3", "corr_fc1_t", 3), ("corr_tc3", "corr_fc1_th", 2), ("corr_tc3", "corr_fc1_th", 1),
             ("corr_tc2", "corr_fc1", 3), ("corr_tc2", "corr_fc1_h", 2), ("corr_tc2", "corr_fc1_h", 1),
             ("corr_tc", "corr_fc1", 3), ("simt", "corr_fc1", 3)}

# (options, T, N, H4, W4, regime).  N*T and 4*N*T land on ragged 128-row tiles (37 x 7 = 259, 1036), plus N = 1.
CASES = [
    ({}, 16, 37, 96, 128, "base"),
    ({}, 7, 37, 64, 72, "motion"),
    ({}, 60, 5, 64, 72, "base"),
    ({}, 7, 37, 64, 72, "gelu"),
    ({"gemm": 1}, 7, 37, 64, 72, "state"),
    ({"prec.fc1": 2}, 7, 37, 96, 128, "base"),
    ({"prec.fc1": 2}, 48, 11, 64, 72, "time"),
    ({"prec.fc1": 2, "gemm": 1}, 2, 37, 64, 72, "dead"),
    ({"prec.corr": 1, "prec.fc1": 1}, 2, 37, 64, 72, "motion"),
    ({"prec.corr": 1, "prec.fc1": 1, "gemm": 1}, 1, 1, 64, 72, "base"),
    ({"prec.corr": 3}, 48, 11, 64, 72, "base"),
    ({"prec.corr": 3}, 16, 8, 96, 128, "gelu"),
    ({"prec.corr": 3, "gemm": 1}, 7, 37, 64, 72, "time"),
    ({"prec.corr": 3, "prec.fc1": 2}, 7, 37, 64, 72, "state"),
    ({"prec.corr": 3, "prec.fc1": 2, "gemm": 1}, 1, 37, 64, 72, "base"),
    ({"prec.corr": 3, "prec.fc1": 1}, 1, 1, 64, 72, "base"),
    ({"prec.corr": 3, "prec.fc1": 1, "gemm": 1}, 7, 37, 64, 72, "dead"),
    ({}, 7, 37, 24, 32, "base"),
    ({}, 60, 5, 24, 32, "base"),
    ({"corr": 2}, 16, 37, 64, 72, "motion"),
    ({"gemm": 1}, 7, 37, 24, 32, "gelu"),
    ({"corr": 1}, 7, 37, 24, 32, "dead"),
    ({"corr": 1, "gemm": 1}, 16, 37, 64, 72, "state"),
    ({}, 2, 37, 64, 72, "time"),
]


def _branch_of(opts, T, H4, W4):
    return loop_branch(T, H4, W4, opts.get("corr", 0), opts.get("prec.corr", 2), opts.get("prec.fc1", 3),
                       opts.get("gemm", 0))


def _case_id(c):
    opts, T, N, H4, W4, regime = c
    o = ",".join(f"{k}={v}" for k, v in opts.items()) or "default"
    return f"{o}-T{T}-N{N}-{H4}x{W4}-{regime}"


# ---------------------------------------------------------------------------------------------------------------------
# inputs
@pytest.fixture(scope="module")
def eng():
    from cotracker_b200 import engine
    engine.lib()
    return engine


@pytest.fixture(scope="module")
def sd():
    from cotracker_b200.synthetic import seeded_state_dict
    return seeded_state_dict(17, offline=True, window_len=60)


def _inputs(sd, T, N, H4, W4, regime, seed):
    """Seeded fmaps, unit-norm support and a state, shaped by the regime."""
    g = torch.Generator().manual_seed(seed)
    if regime == "gelu":   # smooth maps and support read from them: coherent volumes, large pre-activations
        small = torch.randn(T, 128, H4 // 8 + 2, W4 // 8 + 2, generator=g)
        fmaps = F.interpolate(small, (H4, W4), mode="bilinear", align_corners=True)
    else:
        fmaps = torch.randn(T, 128, H4, W4, generator=g) * 2.5
    base = torch.rand(N, 2, generator=g) * torch.tensor([W4 - 1.0, H4 - 1.0])
    if regime == "gelu":
        pyr = O.normalized_pyramid(fmaps)
        qf = torch.randint(0, T, (N,), generator=g)
        support = torch.stack([O.support_features(pyr[l], qf, base / 2 ** l) for l in range(LEVELS)])
    else:
        support = torch.randn(LEVELS, P, N, 128, generator=g)
        support = support / support.norm(dim=-1, keepdim=True)
    if regime == "motion":   # tens of feature units per frame, past the border on both sides
        steps = (torch.rand(T, N, 2, generator=g) * 2 - 1) * torch.tensor([70.0, 50.0])
        coords = base[None] + torch.cumsum(steps, dim=0) - steps[:1]
    else:
        coords = base[None] + torch.randn(T, N, 2, generator=g) * 1.5
    if N >= 2:
        coords[:, 0] = torch.tensor([-7.3, -2.0])
        coords[:, -1] = torch.tensor([W4 + 5.5, H4 + 9.25])
    vis = torch.randn(T, N, generator=g) * 3
    conf = torch.randn(T, N, generator=g) * 3
    if regime == "state":    # +-50 logits, distinct per (t, n) and between vis and conf
        vis = (torch.randperm(T * N, generator=g).float() / (T * N) * 100 - 50).reshape(T, N) + 0.125
        conf = (torch.randperm(T * N, generator=g).float() / (T * N) * 100 - 50).reshape(T, N) - 0.375
    valid = torch.ones(N, dtype=torch.uint8)
    if regime == "dead":
        valid[::2] = 0
    elif N > 2:
        valid[1] = 0
    if regime == "time":     # per-frame values of large magnitude: a wrong row_mod moves every frame but the first
        te = torch.randn(T, XDIM, generator=g) * 4 + 20 * torch.arange(T, dtype=torch.float32)[:, None] - 7
    else:
        te = O.time_embedding(sd, T)[0].contiguous()
    return fmaps, support, coords.contiguous(), vis, conf, valid, te


# ---------------------------------------------------------------------------------------------------------------------
# float64 references and bounds
def _split16(w, fp16):
    """The packing's split of fp32 w into 16-bit hi / lo planes, as float64."""
    hi = w.to(torch.float16 if fp16 else torch.bfloat16)
    lo = (w - hi.float()).to(hi.dtype)
    return hi.double(), lo.double()


def _products(xh, xl, wh, wl, n):
    """float64 of what n tensor-core products compute: x_hi w_hi (+ x_hi w_lo) (+ x_lo w_hi)."""
    out = xh @ wh.T
    if n >= 2:
        out = out + xh @ wl.T
    if n >= 3:
        out = out + xl @ wh.T
    return out


def _acc(S, n):
    return LAM * math.sqrt(n) * 2.0 ** -23 * S


def _rw(W, e):
    return LAM * torch.sqrt((e * e) @ (W * W).T)


def _gelu(a, approx):
    return F.gelu(a, approximate=approx)


def _corr_mlp(sd, planes, b, approx="none", e_in=None):
    """planes: [1 | 2, R, 2401] float64 volume as the GEMM reads it (reference order) -> (X corr [R/4, 1024], bound,
    pre-activations).  e_in: a per-element volume error to propagate (end to end), with the exact fp32 weights."""
    fp16, n = b["volume"] == "fp16", b["products"]
    w1 = sd["corr_mlp.fc1.weight"].to(DEV)
    b1 = sd["corr_mlp.fc1.bias"].to(DEV).double()
    xh = planes[0]
    xl = planes[1] if len(planes) > 1 else torch.zeros_like(xh)
    if e_in is None:
        wh, wl = _split16(w1, fp16)
        a = _products(xh, xl, wh, wl, n) + b1
        weff = wh + (wl if n >= 2 else 0)
        S1 = (xh + (xl if n >= 3 else 0)).abs() @ weff.abs().T + b1.abs()
        e1 = _acc(S1, n * VOL_PAD // 16 + 1)
    else:
        W1 = w1.double()
        a = (xh + xl) @ W1.T + b1
        S1 = (xh + xl).abs() @ W1.abs().T + b1.abs()
        wround = 2.0 ** -11 if n == 1 else (2.0 ** -21 if fp16 else 2.0 ** -16 + 2.0 ** -17)
        e1 = _rw(W1, e_in.expand_as(xh)) + wround * S1 + _acc(S1, n * VOL_PAD // 16 + 1)
    h = _gelu(a, approx)
    e_h = 1.13 * e1 + 2.0 ** -21 * a.abs() + 2.0 ** -17 * h.abs()
    w2 = sd["corr_mlp.fc2.weight"].to(DEV)
    b2 = sd["corr_mlp.fc2.bias"].to(DEV).double()
    w2h, w2l = _split16(w2, False)
    W2 = w2h + w2l
    X = h @ W2.T + b2
    S2 = h.abs() @ W2.abs().T + b2.abs()
    e_X = _rw(W2, e_h) + 2.0 ** -8 * (h.abs() @ w2l.abs().T) + _acc(S2, 3 * HID // 16 + 1) + 2.0 ** -17 * X.abs()
    if e_in is not None:
        e_X = e_X + 2.0 ** -17 * S2
    R4 = X.shape[0] // LEVELS
    return X.reshape(R4, LEVELS * 256), e_X.reshape(R4, LEVELS * 256), a


def _small(coords, vis, conf):
    """-> (want, bound) of the reference columns [vis, conf, posenc(84)] for rows n*T + t, float64 on DEV."""
    c = coords.cpu().double()
    T, N, _ = c.shape
    z = torch.zeros_like(c[:1])
    fwd = torch.cat([c[:-1] - c[1:], z], dim=0)
    bwd = torch.cat([z, c[1:] - c[:-1]], dim=0)
    u = torch.cat([fwd, bwd], dim=-1) / torch.tensor([128.0, 96.0, 128.0, 96.0], dtype=torch.float64)
    pe = O.posenc(u)
    xb = (u.abs()[..., None, :] * (2.0 ** torch.arange(10, dtype=torch.float64))[:, None]).reshape(T, N, 40)
    arg = 2 * xb * 2.0 ** -23
    b_pe = torch.cat([2 * u.abs() * 2.0 ** -23, arg + 2.0 ** -22,
                      arg + 2 * ((xb + 2) * U + 4.4e-8) + 2.0 ** -22], dim=-1) + 2.0 ** -17 * pe.abs()
    vc = torch.stack([vis.cpu().double(), conf.cpu().double()], dim=-1)
    want = torch.cat([vc, pe], dim=-1).transpose(0, 1).reshape(N * T, 86)
    bound = torch.cat([2.0 ** -17 * vc.abs(), b_pe], dim=-1).transpose(0, 1).reshape(N * T, 86)
    return want.to(DEV), bound.to(DEV), xb.max().item() if xb.numel() else 0.0


def _tokens(sd, xh, xl, te, T, e_in=None):
    """tokens of X planes [R, 1110] (reference order, rows n*T + t) + time_emb[t] -> (want, bound)."""
    win = sd["updateformer.input_transform.weight"].to(DEV)
    b = sd["updateformer.input_transform.bias"].to(DEV).double()
    wh, wl = _split16(win, False)
    W = win.double()
    ti = torch.arange(xh.shape[0], device=DEV) % T
    ted = te.to(DEV).double()
    rb = (ted @ W.T)[ti]
    S_te = (ted.abs() @ W.abs().T)[ti]
    if e_in is None:
        Pm = _products(xh, xl, wh, wl, 3)
        S3 = (xh + xl).abs() @ (wh + wl).abs().T + b.abs()
        extra = 0
    else:
        Pm = (xh + xl) @ W.T
        S3 = (xh + xl).abs() @ W.abs().T + b.abs()
        extra = _rw(W, e_in) + (2.0 ** -16 + 2.0 ** -17) * S3
    want = Pm + rb + b
    bound = _acc(S3, 3 * XPAD // 16 + 2) + 40 * U * S_te + 2.0 ** -23 * (Pm.abs() + b.abs() + rb.abs()) + extra
    return want, bound


# volume tolerances of test_corr_sample / test_corr_sample_precision_modes (max abs error, |corr| <= 1)
def _ev(b):
    if b["volume"] == "fp16":
        return 4e-4
    return 1.5e-4 if b["kernel"] in ("corr_tc3", "corr_tc2") else 5e-5


RATIOS = {}


def _ratio(b, link, err, bound):
    # exact zeros (posenc of a still track, pad) have a zero bound
    r = float(torch.where(err == 0, 0.0, err / bound).max()) if err.numel() else 0.0
    key = (branch_key(b), link)
    RATIOS[key] = max(RATIOS.get(key, 0.0), r)
    return r


def _set(eng, opts):
    for k, v in opts.items():
        eng.set_option(k, v)


def _restore(eng):
    for k, v in OPTION_DEFAULTS.items():
        eng.set_option(k, v)


def _run(eng, sd, opts, T, N, H4, W4, regime, seed, tracks=None, e2e_tracks=None):
    """One case: loop_tokens and corr_sample under `opts`, then every link (on `tracks`, default all) and the end-to-end
    check (on `e2e_tracks`).  Returns the branch and the worst err/bound per link."""
    b = _branch_of(opts, T, H4, W4)
    fmaps, support, coords, vis, conf, valid, te = _inputs(sd, T, N, H4, W4, regime, seed)
    if regime == "gelu":
        sd = dict(sd, **{"corr_mlp.fc1.weight": sd["corr_mlp.fc1.weight"] * 10})
    packed = eng.pack_weights(sd, DEV)
    pyr = eng.prepare_pyramid(fmaps.to(DEV))
    dv = [t.to(DEV) for t in (support, valid, coords, vis, conf, te)]
    _set(eng, opts)
    try:
        vol_raw, xs_raw, tok = eng.loop_tokens(packed, pyr, H4, W4, dv[0], dv[1], dv[2], dv[3], dv[4], dv[5], raw=True)
        planes = eng.volume_planes(vol_raw, T, N, H4, W4)
        vol_cs = eng.corr_sample(pyr, H4, W4, dv[0], dv[1], dv[2])
        torch.cuda.synchronize()
    finally:
        _restore(eng)
    # the state is read only
    assert torch.equal(dv[2].cpu(), coords) and torch.equal(dv[3].cpu(), vis) and torch.equal(dv[4].cpu(), conf)
    # volume: bit-identical to the correlation stage under the same options
    assert torch.equal(planes.sum(0).reshape(N, T, LEVELS, VOL), vol_cs), "loop volume != ct3_corr_sample"
    assert planes.shape[0] == (1 if b["volume"] == "fp16" else 2)
    del vol_cs
    idx = torch.arange(N) if tracks is None else torch.as_tensor(tracks)
    rows = (idx[:, None] * T + torch.arange(T)[None]).reshape(-1).to(DEV)                    # X / token rows n*T + t
    vrows = (rows[:, None] * LEVELS + torch.arange(LEVELS, device=DEV)[None]).reshape(-1)   # volume rows
    vp = planes[:, vrows].double()
    del planes
    xs = xs_raw[rows]
    assert bool((xs.reshape(-1, 2, XPAD)[:, :, XDIM:] == 0).all()), "X pad columns must be exactly 0"
    xp = eng.x_planes(xs).double()
    xg = xp.sum(0)
    out = {}

    # corr_mlp: X's correlation columns against fc2(gelu_erf(fc1(v)))
    want, bound, a = _corr_mlp(sd, vp, b)
    got = xg[:, 2:2 + LEVELS * 256]
    err = (got - want).abs()
    out["corr_mlp"] = _ratio(b, "corr_mlp", err, bound)
    if regime == "gelu":
        want_t, _, _ = _corr_mlp(sd, vp, b, "tanh")
        gap = float((want - want_t).abs().max())
        assert float(a.abs().max()) > 2.0 and gap > 4 * float(err.max()), (float(a.abs().max()), gap)
        d_erf, d_tanh = float(err.mean()), float((got - want_t).abs().mean())
        assert d_erf < 0.2 * d_tanh, ("corr_mlp GELU is not erf", d_erf, d_tanh)
    dead = ~valid[idx].bool()
    if bool(dead.any()):   # no support: zero volume rows, every row of X fc2(gelu(b1)) + b2, bit-identical
        dr = dead.repeat_interleave(T).to(DEV)
        assert bool((vp.reshape(vp.shape[0], -1, LEVELS, VOL)[:, dr] == 0).all())
        dx = got[dr].reshape(-1, LEVELS, 256)
        assert bool((dx == dx[:1, :1]).all()), "dead-track rows differ"

    # small columns
    want_s, bound_s, max_arg = _small(coords[:, idx], vis[:, idx], conf[:, idx])
    got_s = torch.cat([xg[:, :2], xg[:, 2 + LEVELS * 256:]], dim=1)
    out["small"] = _ratio(b, "small", (got_s - want_s).abs(), bound_s)
    if regime == "motion":
        assert max_arg > 100, max_arg

    # input_transform on X as written + time_emb[t]
    want_t, bound_t = _tokens(sd, xp[0], xp[1], te, T)
    got_t = tok[rows].double()
    out["input_transform"] = _ratio(b, "input_transform", (got_t - want_t).abs(), bound_t)

    # end to end against the float64 oracle
    e_idx = idx if e2e_tracks is None else torch.as_tensor(e2e_tracks)
    sd64 = {k: sd[k].double() for k in ("corr_mlp.fc1.weight", "corr_mlp.fc1.bias", "corr_mlp.fc2.weight",
                                         "corr_mlp.fc2.bias")}
    sd64["time_emb"] = torch.zeros(1, T, XDIM, dtype=torch.float64)   # X without it; _tokens adds time_emb[t]
    pyr64 = O.normalized_pyramid(fmaps.double())
    sup = support[:, :, e_idx].double() * valid[e_idx].double()[None, None, :, None]
    c64 = coords[:, e_idx].double()
    with torch.no_grad():
        vols = torch.stack([O.correlation_volume(pyr64[l], sup[l], c64 / 2 ** l) for l in range(LEVELS)], dim=2)
        x64 = O.transformer_input(sd64, torch.zeros(T, len(e_idx), 1024, dtype=torch.float64), c64,
                                  vis[:, e_idx].double(), conf[:, e_idx].double())[0]
    v64 = vols.permute(1, 0, 2, 3).reshape(1, -1, VOL).to(DEV)            # rows (n*T + t)*4 + l
    ev = torch.full((1, VOL), _ev(b), dtype=torch.float64, device=DEV)
    xc, exc, _ = _corr_mlp(sd, v64, b, e_in=ev)
    x64 = x64.reshape(-1, XDIM).to(DEV)
    x64[:, 2:2 + LEVELS * 256] = xc
    _, bs, _ = _small(coords[:, e_idx], vis[:, e_idx], conf[:, e_idx])
    ex = torch.cat([bs[:, :2], exc, bs[:, 2:]], dim=1)
    want_e, bound_e = _tokens(sd, x64, torch.zeros_like(x64), te, T, e_in=ex)
    er = (e_idx[:, None] * T + torch.arange(T)[None]).reshape(-1).to(DEV)
    out["end_to_end"] = _ratio(b, "end_to_end", (tok[er].double() - want_e).abs(), bound_e)
    return b, out


@pytest.mark.parametrize("case", CASES, ids=[_case_id(c) for c in CASES])
def test_loop_tokens_links(eng, sd, case):
    opts, T, N, H4, W4, regime = case
    b, out = _run(eng, sd, opts, T, N, H4, W4, regime, seed=zlib.crc32(_case_id(case).encode()))
    print("tokens-branch", _case_id(case), b)
    print("tokens-ratio", _case_id(case), {k: f"{v:.3g}" for k, v in out.items()})
    for link, r in out.items():
        assert r <= 1.0, (link, r, b)


@pytest.mark.parametrize("fc1", [3, 2])
def test_loop_tokens_full_size_sampled(eng, sd, fc1):
    """N = 6400, T = 16, 96 x 128 (the headline problem): the stage is independent per track, so a seeded sample of
    128 tracks, the first and the last included (first and last GEMM tiles), is checked link by link and 16 of them
    end to end."""
    N, T, H4, W4 = 6400, 16, 96, 128
    g = torch.Generator().manual_seed(fc1)
    tracks = sorted({0, N - 1} | set(torch.randperm(N, generator=g)[:126].tolist()))
    b, out = _run(eng, sd, {"prec.fc1": fc1}, T, N, H4, W4, "base", seed=100 + fc1, tracks=tracks,
                  e2e_tracks=tracks[::8] + [N - 1])
    print("tokens-branch full-size", b)
    print("tokens-ratio full-size", fc1, {k: f"{v:.3g}" for k, v in out.items()})
    for link, r in out.items():
        assert r <= 1.0, (link, r, b)


def test_case_list_reaches_every_branch():
    seen = [branch_key(_branch_of(o, T, H4, W4)) for o, T, _, H4, W4, _ in CASES]
    for c in CASES:
        print("tokens-branch-map", _case_id(c), branch_key(_branch_of(c[0], c[1], c[3], c[4])))
    combos = {k[:3] for k in seen}
    assert combos == REACHABLE, combos ^ REACHABLE
    for gemm in ("wgmma", "simt"):
        assert {k[:3] for k in seen if k[3] == gemm} == REACHABLE, gemm
    assert {T for _, T, *_ in CASES} >= {1, 2, 7, 16, 48, 60}
    assert {(H4, W4) for _, _, _, H4, W4, _ in CASES} >= {(24, 32), (64, 72), (96, 128)}


def test_print_worst_ratios():
    """Runs last in the file: the worst err/bound per (branch, link) over every case above."""
    for (key, link), r in sorted(RATIOS.items()):
        print("tokens-worst", key, link, f"{r:.3g}")
