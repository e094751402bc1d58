"""Float64 restatements of the transformer body and the heads (api_loop.cu: transformer_body, transform_and_heads), link
by link, with the per-element bound of each link, and the attention branch map.

Shared by test_gpu_body.py (GEMM epilogues, fused time attention, LayerNorm on synthetic operands), test_gpu_attention.py
(every attention kernel) and test_gpu_body_trace.py (every link of ct3_body_trace on the kernel's own input to it).
u = 2^-24 is the fp32 unit roundoff.  The bounds themselves are derived in the docstrings of test_gpu_body.py (GEMM,
time attention, LayerNorm) and test_gpu_attention.py (attention cores); this module states the links that are new here:

  virtual init     every virtual row i*T + t is virual_tracks[i], bit for bit: bound 0.
  context LN       the LayerNorm bound with gamma / beta = norm_context's weight / bias and eps 1e-5 (fp32).
  heads            four fp32 dot products of 384 terms, P = sum_k |x_k w_k|: each lane sums its 12 products in one chain
                   (<= 12 u P over its terms), the 5-step warp sum adds <= 5 u P, the bias one rounding
                   u (|acc| + |b|), and state += delta one more, u |state'|:
                   bound = 2 [(12 + 5) u P + u (|acc| + |b|)] + u |state'|   (2x margin on the sum).

Each link is checked against float64 computed on the kernel's own input to that link, which is the tapped output of the
link before it (BodyWalk.get), so errors never compound.  Weights are rounded to 16 significant bits before packing
(round16), so the reference multiplies exactly the planes the GEMM reads.
"""
import math

import torch

C, HEADS, DH, KV, HID, DEPTH = 384, 8, 48, 64, 1536, 3
U = 2.0 ** -24
WARPS, MAX_SPLITS = 4, 32
TIME, V_FROM_P, V_SELF, P_FROM_V = 0, 1, 2, 3


# =====================================================================================================================
# split planes and weights
def round16(w):
    """w rounded to 16 significant bits: exactly bf16 hi + bf16 lo, so that packing it adds no error"""
    m, e = torch.frexp(w.double())
    return torch.ldexp(torch.round(m * 65536.0) / 65536.0, e)


def planes(v, fp16=False):
    """float64 values -> (hi, lo) 16-bit planes (bf16 or fp16)"""
    dt = torch.float16 if fp16 else torch.bfloat16
    hi = v.to(dt)
    return hi, (v - hi.double()).to(dt)


def decode(split):
    """split 16-bit rows [rows, 2*C'] (hi | lo) -> float64 hi + lo [rows, C']"""
    c = split.shape[1] // 2
    return split[:, :c].double() + split[:, c:].double()


def acc_bound(impl, products, Kpad):
    """GEMM accumulation error per unit of S = sum_k |x_k| |w_k| (test_gpu_body.py)"""
    if impl == 1:
        return 2 * Kpad * U
    return (products * Kpad // 16 + 1) * 2 * U


# =====================================================================================================================
# GEMM, LayerNorm, heads
def gemm_ref(x, w, b, impl, act=0, residual=None, split=False):
    """y = act(x w^T + b) [+ residual] in float64 on x (float64, = hi + lo of the split operand) and w (float64, exact
    to 16 bits), b fp32 -> (want, bound), the bound of test_gpu_body.py's GEMM epilogues (3 products)"""
    acc = x @ w.t()
    S = x.abs() @ w.abs().t()
    L = planes(x)[1].double().abs() @ planes(w)[1].double().abs().t() if impl == 0 else 0.0
    v = acc + b
    y = torch.nn.functional.gelu(v, approximate="tanh") if act else v
    want = y + residual if residual is not None else y
    bd = (1.2 if act else 1.0) * (L + acc_bound(impl, 3, w.shape[1]) * S + 2.0 ** -22 * (acc.abs() + b.abs()))
    bd = bd + (2.0 ** -21 * v.abs() if act else 0) + 2.0 ** -22 * (want.abs() + (residual.abs() if residual is not None
                                                                                   else 0))
    if split:
        bd = bd + 2.0 ** -17 * want.abs()
    return want, bd


def ln_ref(x, eps, gamma=None, beta=None):
    """LayerNorm of float64 rows x [rows, 384] with fp32 eps (and the affine) -> (want, bound) (test_gpu_body.py)"""
    mean = x.mean(1, keepdim=True)
    eps32 = float(torch.tensor(eps, dtype=torch.float32))   # the eps the kernel adds
    sigma = (x.var(1, unbiased=False, keepdim=True) + eps32).sqrt()
    z = (x - mean) / sigma
    gm = gamma if gamma is not None else torch.ones(C, device=x.device, dtype=torch.float64)
    bt = beta if beta is not None else torch.zeros(C, device=x.device, dtype=torch.float64)
    want = z * gm + bt
    A = x.abs().mean(1, keepdim=True)
    return want, gm.abs() * 2.0 ** -19 * (z.abs() + A / sigma) + 2.0 ** -22 * bt.abs() + 2.0 ** -17 * want.abs()


def heads_ref(tok, w4, b4, state):
    """state [rows, 4] fp32 (dx, dy, vis, conf per point row) += tok [rows, 384] w4^T + b4 -> (want, bound) (module
    docstring)"""
    acc = tok @ w4.t()
    P = tok.abs() @ w4.abs().t()
    want = state + acc + b4
    return want, 2 * ((12 + 5) * U * P + U * (acc.abs() + b4.abs())) + U * want.abs()


# =====================================================================================================================
# attention
def bound(attn, labs, vmax, lk):
    """attention-core bound (test_gpu_attention.py): Labs = max sum_d |q_d k_d| / sqrt(48), vmax = max |v|"""
    if attn == 1:
        return (2.0 ** -17 + 4 * 2.0 ** -24 * (math.sqrt(DH) * (1 + labs) + math.sqrt(lk))) * vmax
    return 2 * (1 + labs) * 2.0 ** -16 * vmax


def attn_ref(Q, K, V, attn):
    """softmax(Q K^T / sqrt(48)) V per sequence and head of float64 Q [S, Lq, 8, 48], K, V [S, Lk, 8, 48] -> (want,
    bound) [S, Lq, 8, 48], the bound with Labs and vmax of each (sequence, head)"""
    s = torch.einsum("sihd,sjhd->shij", Q, K) / math.sqrt(DH)
    out = torch.einsum("shij,sjhd->sihd", torch.softmax(s, dim=-1), V)
    del s
    labs = torch.einsum("sihd,sjhd->shij", Q.abs(), K.abs()).amax(dim=(2, 3)) / math.sqrt(DH)
    vmax = V.abs().amax(dim=(1, 3))
    return out, bound(attn, labs, vmax, K.shape[1])[:, None, :, None].expand_as(out)


def qkv64(x, wq, bq, wkv, bkv):
    """float64 q, k, v [rows, 384] and their elementwise magnitudes S = |x| |w|^T"""
    q, kv = x @ wq.t() + bq, x @ wkv.t() + bkv
    sq, skv = x.abs() @ wq.abs().t(), x.abs() @ wkv.abs().t()
    return q, kv[:, :C], kv[:, C:], sq, skv[:, :C], skv[:, C:]


def time_reference(x_split, wq, bq, wkv, bkv, T, n, fused, impl, chunk=256):
    """q|k|v projection + per-track attention from the split LayerNorm output (test_gpu_body.py's bound)
    -> (want [rows, 384] float64, bound [rows, 384], max |logit|)"""
    x = x_split[:, :C].double() + x_split[:, C:].double()
    q, k, v, sq, sk, sv = qkv64(x, wq, bq, wkv, bkv)
    if impl == 0:   # the dropped lo*lo products, from the planes (the weights split exactly, see round16)
        xl = x_split[:, C:].double().abs()
        lq, lkv = xl @ planes(wq)[1].double().abs().t(), xl @ planes(wkv)[1].double().abs().t()
    else:
        lq, lkv = torch.zeros_like(q), torch.zeros(q.shape[0], 2 * C, device=q.device, dtype=q.dtype)
    c_acc = acc_bound(impl, 3, C)

    def gemm_err(val, lolo, s, b):
        return lolo + c_acc * s + 2 * U * (val.abs() + b.abs())
    dq, dk, dv = (gemm_err(q, lq, sq, bq), gemm_err(k, lkv[:, :C], sk, bkv[:C]),
                  gemm_err(v, lkv[:, C:], sv, bkv[C:]))
    want = torch.empty_like(q)
    bound_ = torch.empty_like(q)
    lmax = 0.0
    for n0 in range(0, n, chunk):
        r = slice(n0 * T, min(n, n0 + chunk) * T)
        Q, K, V, DQ, DK, DV = (t[r].view(-1, T, HEADS, DH) for t in (q, k, v, dq, dk, dv))
        s = torch.einsum("nihd,njhd->nhij", Q, K) / math.sqrt(DH)
        qk = torch.einsum("nihd,njhd->nhij", Q.abs(), K.abs()) / math.sqrt(DH)
        ds = (torch.einsum("nihd,njhd->nhij", DQ, K.abs()) + torch.einsum("nihd,njhd->nhij", Q.abs(), DK)
              + torch.einsum("nihd,njhd->nhij", DQ, DK)) / math.sqrt(DH) + 48 * U * qk + 2.0 ** -22 * s.abs()
        o = torch.einsum("nhij,njhd->nihd", torch.softmax(s, dim=-1), V)
        D = ds.amax(dim=(2, 3))                                        # [n, h]
        vmax = V.abs().amax(dim=(1, 3))
        b = torch.expm1(2 * D) * vmax + DV.amax(dim=(1, 3)) + (T + 16) * 2 * U * vmax
        if not fused:
            b = b + 2 * (1 + qk.amax(dim=(2, 3))) * 2.0 ** -16 * vmax
        want[r] = o.reshape(-1, C)
        bound_[r] = (b[:, None, :, None] + 2.0 ** -17 * o.abs()).reshape(-1, C)
        lmax = max(lmax, float(s.abs().max()))
    return want, bound_, lmax


# =====================================================================================================================
# branch map: which kernel the host picks (attention_tc.cu: attention_tc_splits, launch_attention_tc; api_loop.cu:
# run_attention, space_attention, plan_groups, time_attention)
def tc_splits(num_seq, Lq, Lk, sms):
    """attention_tc_splits: split-K count of a shared-K/V launch (mma.sync kernel)."""
    q_tiles = (Lq + 15) // 16
    ctas = num_seq * HEADS * ((q_tiles + WARPS - 1) // WARPS)
    chunks = (Lk + 63) // 64
    splits = 1
    if ctas < 2 * sms and chunks >= 8:
        slots, best = 4 * sms, -1
        for sp in range(1, min(MAX_SPLITS, chunks // 2) + 1):
            cost = ((ctas * sp + slots - 1) // slots) * ((chunks + sp - 1) // sp)
            if best < 0 or cost < best:
                best, splits = cost, sp
    return splits


def tc_qtw(num_seq, Lq, Lk, sms):
    """launch_attention_tc without split-K: query tiles per warp when K/V fit one chunk."""
    q_tiles = (Lq + 15) // 16
    qtw = 1
    if (Lk + 63) // 64 == 1:
        while qtw < 8 and num_seq * HEADS * ((q_tiles + WARPS * 2 * qtw - 1) // (WARPS * 2 * qtw)) >= 4 * sms:
            qtw *= 2
    return qtw


def branch(kind, T, N, sizes, attn, sms):
    """What ct3_attention runs for this call: a dict of the branch's features."""
    sizes = list(sizes) if sizes is not None else [N]
    G = len(sizes)
    if attn == 1:
        return {"path": "simt"}
    if kind == TIME:   # run_attention(per_warp): every track, KB by the key count
        return {"path": "per_warp", "kb": 16 if T <= 16 else 32 if T <= 32 else 64, "T": T}
    if G == 1:
        if kind == P_FROM_V and N > KV:
            return {"path": "wgmma"}
        Lq, Lk = {V_FROM_P: (KV, N), V_SELF: (KV, KV), P_FROM_V: (N, KV)}[kind]
        s = tc_splits(T, Lq, Lk, sms)
        if s > 1:
            return {"path": "split_k", "splits": s}
        return {"path": "shared", "qtw": tc_qtw(T, Lq, Lk, sms)}
    if kind == V_FROM_P:   # per-group split-K counts (plan_groups), one launch
        splits = [tc_splits(T, KV, n, sms) for n in sizes]
        if max(splits) > 1:
            return {"path": "grouped_split_k", "group_splits": splits}
        return {"path": "grouped", "qtw": tc_qtw(T * G, KV, max(sizes), sms)}
    if kind == V_SELF:
        return {"path": "grouped", "qtw": tc_qtw(T * G, KV, KV, sms)}
    small = [n for n in sizes if n <= KV]   # point <- virtual: groups of > 64 tracks on wgmma tiles, the rest mma.sync
    out = {"path": "grouped_p2v", "wgmma_groups": G - len(small), "mma_groups": len(small)}
    if small:
        out["qtw"] = tc_qtw(T * len(small), KV, KV, sms)
    return out


def describe(b):
    return " ".join(f"{k}={v}" for k, v in b.items())


def time_fused(T, gemm, attn, fuse):
    """time_attention: the fused q|k|v + attention kernel, else the q|k|v GEMM and the per-warp (or SIMT) kernel"""
    return fuse == 1 and gemm == 0 and attn != 1 and T <= 128


def body_branch(T, N, gemm, attn, fuse, sms):
    """The kernels one G = 1 pass of transformer_body runs: the GEMM engine, the time path and each space attention"""
    return {"gemm": "simt" if gemm else "wgmma",
            "time": {"path": "fused"} if time_fused(T, gemm, attn, fuse) else branch(TIME, T, N, None, attn, sms),
            "v2p": branch(V_FROM_P, T, N, None, attn, sms), "vself": branch(V_SELF, T, N, None, attn, sms),
            "p2v": dict(branch(P_FROM_V, T, N, None, attn, sms), **({"ragged_tile": N % 128 != 0} if N > KV else {}))}


def body_coverage(cases, sms):
    """The branches a case list (T, N, regime, gemm, attn, fuse) must reach on a device of `sms` SMs -> missing ones"""
    bs = [(c, body_branch(c[0], c[1], *c[3:], sms)) for c in cases]
    checks = {
        "fused time attention": any(b["time"]["path"] == "fused" for _, b in bs),
        "SIMT GEMM": any(b["gemm"] == "simt" for _, b in bs),
        "SIMT attention": any(b["time"]["path"] == "simt" for _, b in bs),
        "unfused time attention at T > 128": any(b["time"]["path"] == "per_warp" and c[0] > 128 for c, b in bs),
        "split-K virtual <- point": any(b["v2p"]["path"] == "split_k" for _, b in bs),
        "unsplit virtual <- point over >= 8 key chunks": any(b["v2p"]["path"] == "shared" and c[1] > 7 * 64
                                                              for c, b in bs),
        "point <- virtual on wgmma with a ragged tile": any(b["p2v"].get("ragged_tile") for _, b in bs),
        "point <- virtual on mma.sync": any(b["p2v"]["path"] == "shared" for _, b in bs),
    }
    for kb in (16, 32, 64):
        checks[f"per-warp time attention KB = {kb}"] = any(b["time"].get("kb") == kb for _, b in bs)
    for r in ("default", "norm_context", "sharp"):
        checks[f"regime {r}"] = any(c[2] == r for c in cases)
    return [k for k, ok in checks.items() if not ok]


# cases of test_gpu_body_trace.py: (T, N, regime, gemm, attn, fuse)
BODY_CASES = [
    (16, 6400, "default", 0, 0, 1),       # headline: 80 x 80 grid, online window; split-K virtual <- point
    (16, 2500, "default", 0, 0, 1),       # online grid
    (60, 1225, "default", 0, 0, 1),       # offline window
    (48, 600, "default", 0, 0, 1),        # virtual <- point over 10 key chunks
    (20, 65, "default", 0, 0, 1),         # point <- virtual on wgmma, one ragged 128-track tile
    (20, 64, "default", 0, 0, 1),         # point <- virtual on mma.sync
    (129, 5, "default", 0, 0, 1),         # T > 128: unfused time attention
    (2, 3, "default", 0, 0, 1),           # tiny
    (2, 3, "default", 0, 0, 0),           # per-warp time attention, KB 16
    (40, 130, "default", 0, 0, 0),        # per-warp time attention, KB 64
    (24, 200, "default", 1, 0, 1),        # SIMT GEMM
    (24, 200, "default", 0, 1, 1),        # SIMT attention
    (24, 200, "default", 0, 0, 0),        # per-warp time attention, KB 32
    (16, 600, "norm_context", 0, 0, 1),   # trained-like norm_context below its eps
    (40, 130, "sharp", 0, 0, 1),          # max |logit| about 30
]


def body_case_id(c):
    T, N, regime, gemm, attn, fuse = c
    return f"T{T}-N{N}-{regime}-gemm{gemm}-attn{attn}-fuse{fuse}"


# =====================================================================================================================
# weights and regimes
TOKEN_SCALE = 1e-3


def body_state(sd, regime, seed=8):
    """A float32 state dict for the body: every GEMM weight of the updateformer rounded to 16 significant bits, and
    every Linear bias of the updateformer (heads included) ~ 0.1 N(0, 1), where a fresh module has zeros, so that a
    bias read from the wrong layer, at the wrong column offset or added more than once moves its link; shaped by the
    regime:
      default       as seeded, with those biases;
      norm_context  a trained-like affine norm_context in every cross block (gamma ~ 1 + 0.7 N(0, 1), some negative;
                    beta ~ 0.5 N(0, 1)), and the virtual tracks and every residual write of the time, virtual <- point
                    and virtual self blocks scaled by TOKEN_SCALE, so that the tokens the first norm_contexts see have a
                    variance near 1e-6, below their eps of 1e-5: eps then decides those LayerNorms;
      sharp         every to_q weight and bias x 6: max |logit| about 30."""
    g = torch.Generator().manual_seed(seed)
    sd = dict(sd)
    for k in [k for k in sd if k.startswith("updateformer.") and k.endswith(".bias") and "norm_context" not in k]:
        sd[k] = 0.1 * torch.randn(sd[k].shape, generator=g)
    if regime == "norm_context":
        for k in [k for k in sd if k.endswith("norm_context.weight")]:
            sd[k] = 1 + 0.7 * torch.randn(sd[k].shape, generator=g)
            sd[k[:-len("weight")] + "bias"] = 0.5 * torch.randn(sd[k].shape, generator=g)
        sd["updateformer.virual_tracks"] = sd["updateformer.virual_tracks"] * TOKEN_SCALE
        for k in [k for k in sd if k.startswith(("updateformer.time_blocks.", "updateformer.space_virtual_blocks.",
                                                 "updateformer.space_virtual2point_blocks."))
                  and (".to_out." in k or ".mlp.fc2." in k)]:
            sd[k] = sd[k] * TOKEN_SCALE
    elif regime == "sharp":
        for k in [k for k in sd if k.startswith("updateformer.") and ".to_q." in k]:
            sd[k] = sd[k] * 6.0
    for k in [k for k in sd if k.startswith("updateformer.") and k.endswith(".weight") and sd[k].dim() == 2
              and "_head." not in k]:
        sd[k] = round16(sd[k]).float()
    return sd


def body_tokens(N, T, regime, g):
    """Seeded point tokens fp32 [N*T, 384] of the regime (norm_context: scaled by TOKEN_SCALE)"""
    x = torch.randn(N * T, C, generator=g)
    return x * TOKEN_SCALE if regime == "norm_context" else x


# =====================================================================================================================
# the walk: every link of ct3_body_trace in order, each from the links it reads
def _frames(x, L, T):
    """rows l*T + t of x [L*T, 384] -> [T, L, 8, 48] (sequence = frame)"""
    return x.view(L, T, HEADS, DH).transpose(0, 1)


def _rows(o, L, T):
    return o.transpose(0, 1).reshape(L * T, C)


class BodyWalk:
    """Walks the links of one G = 1 pass in ct3_body_trace's order.  For each link it calls emit(name, want, bound)
    with the float64 reference computed on get(...) of the links it reads; a subclass decides what get returns (the
    trace, or the walk's own references) and what emit does with the reference."""

    def __init__(self, sd, T, N, gemm=0, attn=0, fuse=1):
        dev = self.device
        self.T, self.N, self.impl, self.attn = T, N, gemm, attn
        self.fused = time_fused(T, gemm, attn, fuse)
        self.w = {k: v.to(dev).double() for k, v in sd.items() if k.startswith("updateformer.")}

    def emit(self, name, want, bd):
        raise NotImplementedError

    def get(self, name):
        raise NotImplementedError

    def lin(self, p):
        return self.w[p + ".weight"], self.w[p + ".bias"]

    def gemm(self, name, x, p, **kw):
        w, b = self.lin(p)
        self.emit(name, *gemm_ref(x, w, b, self.impl, **kw))

    def mlp(self, name, p, x):
        """LayerNorm, fc1 + tanh GELU, fc2 + residual of rows x -> the tokens after fc2"""
        self.emit(f"{name}.mlp_ln", *ln_ref(x, 1e-6))
        self.gemm(f"{name}.fc1", self.get(f"{name}.mlp_ln"), p + ".mlp.fc1", act=2, split=True)
        self.gemm(f"{name}.fc2", self.get(f"{name}.fc1"), p + ".mlp.fc2", residual=x)
        return self.get(f"{name}.fc2")

    def space(self, name, q, kv, Lq, Lk, k_col):
        """space attention: per frame, Lq query rows of q over Lk key rows of kv (k at k_col, v at k_col + 384)"""
        T = self.T
        out, bd = attn_ref(_frames(q, Lq, T), _frames(kv[:, k_col:k_col + C], Lk, T),
                           _frames(kv[:, k_col + C:k_col + 2 * C], Lk, T), self.attn)
        self.emit(name, _rows(out, Lq, T), _rows(bd, Lq, T))

    def run(self, tokens, state):
        """tokens float64 [N*T, 384] (the call's input), state float64 [N*T, 4] (coords x, y, vis, conf per point row
        before the heads) -> runs every link, then emits "heads" (the state after the update)"""
        T, N, w, pre = self.T, self.N, self.w, "updateformer."
        Rp = N * T
        virt = w[pre + "virual_tracks"].reshape(KV, C)
        self.emit("virtual_init", virt.repeat_interleave(T, 0), torch.zeros(KV * T, C, dtype=torch.float64,
                                                                             device=self.device))
        pts, vt = tokens, self.get("virtual_init")
        for i in range(DEPTH):
            # time block over every row: sequence = track
            n, p = f"{i}.time", f"{pre}time_blocks.{i}"
            x = torch.cat([pts, vt])
            self.emit(f"{n}.ln", *ln_ref(x, 1e-6))
            h = self.get(f"{n}.ln")
            wq, bq = self.lin(p + ".attn.to_q")
            wkv, bkv = self.lin(p + ".attn.to_kv")
            if self.fused:
                hs = torch.cat(planes(h), 1)
                want, bd, _ = time_reference(hs, wq, bq, wkv, bkv, T, N + KV, True, self.impl)
                self.emit(f"{n}.attn", want, bd)
            else:
                self.emit(f"{n}.qkv", *gemm_ref(h, torch.cat([wq, wkv]), torch.cat([bq, bkv]), self.impl))
                qkv = self.get(f"{n}.qkv").view(N + KV, T, 3, HEADS, DH)
                out, bd = attn_ref(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], self.attn)
                self.emit(f"{n}.attn", out.reshape(-1, C), bd.reshape(-1, C))
            self.gemm(f"{n}.out", self.get(f"{n}.attn"), p + ".attn.to_out", residual=x)
            x = self.mlp(n, p, self.get(f"{n}.out"))
            pts, vt = x[:Rp], x[Rp:]
            # virtual <- point: x = virtual, context = points through norm_context
            n, p = f"{i}.v2p", f"{pre}space_virtual2point_blocks.{i}"
            self.emit(f"{n}.ln", *ln_ref(vt, 1e-6))
            self.gemm(f"{n}.q", self.get(f"{n}.ln"), p + ".cross_attn.to_q")
            self.emit(f"{n}.ctx_ln", *ln_ref(pts, 1e-5, w[p + ".norm_context.weight"], w[p + ".norm_context.bias"]))
            self.gemm(f"{n}.kv", self.get(f"{n}.ctx_ln"), p + ".cross_attn.to_kv")
            self.space(f"{n}.attn", self.get(f"{n}.q"), self.get(f"{n}.kv"), KV, N, 0)
            self.gemm(f"{n}.out", self.get(f"{n}.attn"), p + ".cross_attn.to_out", residual=vt)
            vt = self.mlp(n, p, self.get(f"{n}.out"))
            # virtual self attention
            n, p = f"{i}.vself", f"{pre}space_virtual_blocks.{i}"
            self.emit(f"{n}.ln", *ln_ref(vt, 1e-6))
            wq, bq = self.lin(p + ".attn.to_q")
            wkv, bkv = self.lin(p + ".attn.to_kv")
            self.emit(f"{n}.qkv", *gemm_ref(self.get(f"{n}.ln"), torch.cat([wq, wkv]), torch.cat([bq, bkv]),
                                            self.impl))
            qkv = self.get(f"{n}.qkv")
            self.space(f"{n}.attn", qkv[:, :C], qkv, KV, KV, C)
            self.gemm(f"{n}.out", self.get(f"{n}.attn"), p + ".attn.to_out", residual=vt)
            vt = self.mlp(n, p, self.get(f"{n}.out"))
            # point <- virtual: x = points, context = virtual through norm_context
            n, p = f"{i}.p2v", f"{pre}space_point2virtual_blocks.{i}"
            self.emit(f"{n}.ln", *ln_ref(pts, 1e-6))
            self.gemm(f"{n}.q", self.get(f"{n}.ln"), p + ".cross_attn.to_q")
            self.emit(f"{n}.ctx_ln", *ln_ref(vt, 1e-5, w[p + ".norm_context.weight"], w[p + ".norm_context.bias"]))
            self.gemm(f"{n}.kv", self.get(f"{n}.ctx_ln"), p + ".cross_attn.to_kv")
            self.space(f"{n}.attn", self.get(f"{n}.q"), self.get(f"{n}.kv"), N, KV, 0)
            self.gemm(f"{n}.out", self.get(f"{n}.attn"), p + ".cross_attn.to_out", residual=pts)
            pts = self.mlp(n, p, self.get(f"{n}.out"))
        w4 = torch.cat([w[pre + "flow_head.weight"], w[pre + "vis_conf_head.weight"]])
        b4 = torch.cat([w[pre + "flow_head.bias"], w[pre + "vis_conf_head.bias"]])
        self.emit("heads", *heads_ref(pts, w4, b4, state))


class SelfWalk(BodyWalk):
    """The restatement chained on its own float64 outputs: get returns the reference emitted for that link"""
    device = "cpu"

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.out = {}

    def emit(self, name, want, bd):
        self.out[name] = want

    def get(self, name):
        return self.out[name]


def state_rows(coords, vis, conf):
    """coords [T, N, 2], vis / conf [T, N] -> [N*T, 4] in point-row order n*T + t"""
    return torch.cat([coords, vis[..., None], conf[..., None]], -1).transpose(0, 1).reshape(-1, 4)
