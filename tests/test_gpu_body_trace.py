"""The transformer body and the heads link by link against float64: ct3_body_trace runs the update loop's own
transformer_body and heads on seeded point tokens and copies every link's output; tests/body_cases.py restates each
link in float64 on the kernel's own input to it (the tapped output of the link before) and bounds its error per
element.  The cases reach every branch of the body on the device they run on (body_cases.body_coverage).

Every Linear bias of the updateformer, heads included, is seeded nonzero (body_cases.body_state), so each link also
checks that its GEMM reads the right bias at the right columns, once.

Besides the bounds:
  - every virtual row equals virual_tracks bit for bit after the init;
  - bytes no link owns keep a sentinel: in the trace, the alignment gaps and, with the fused time kernel, the q|k|v
    link; in the workspace (prefilled), the correlation-half scratch and the row bias, which the body must not touch,
    and with the fused time kernel the fp32 q|k|v buffer past the point rows' virtual <- point k|v, so a k|v written
    at a wider pitch or over more rows shows;
  - the workspace's token rows after the call are the last point <- virtual and virtual-self fc2 links, bit for bit;
  - "ct3_loop_tokens on the state, then ct3_body_trace on its tokens", repeated, leaves coords / vis / conf
    bit-identical to ct3_update_loop.  With test_gpu_tokens.py this puts the whole iteration under float64 link bounds.

Measured on an NVIDIA H100 80GB HBM3 at 700 W (132 SMs), one run of this file with pytest -s: 24 tests in 30 s; the
largest case, (N, T) = (6400, 16), peaks at 31.1 GiB of device memory (torch.cuda.max_memory_allocated: the 12.0 GB
trace, the 6.7 GB workspace and the float64 references of one link at a time).  Worst err / bound over all cases, as the
run prints it per (link kind, case): LayerNorms 0.78 and norm_context 0.96 (the fp32 rounding of the statistics is the
whole error, as in test_gpu_body.py), time attention 0.48, space attention 0.15, GEMMs 0.20 or less, heads 0.06.

Mutations, each built alone into the library and run against this file and against the existing GPU tests that run
the whole transformer (test_gpu_stages.py, test_gpu_attention.py's sharp updateformer test, test_gpu_fullsize.py,
test_gpu_e2e.py), on the same card:
  mutation                                                   this file fails at           existing tests
  virtual-self MLP hidden layer of block 1, lo plane zeroed  1.vself.fc1 (62 x its bound)  pass (164 passed)
  erf GELU in place of tanh in time block 1's MLP            1.time.fc1 (4.7 x)            fail (test_update_loop_vs_oracle)
  point <- virtual norm_context at eps 1e-6                  p2v.ctx_ln (4e5 x)            pass (164 passed)
  attention scale rounded to bf16 in point <- virtual        p2v.attn (4.0 x)              fail (test_updateformer_stage)
  heads' bias added on every lane before the warp sum        heads (6e4 x)                 pass (164 passed)
"""
import zlib

import pytest
import torch

from body_cases import (BODY_CASES, C, DEPTH, KV, BodyWalk, body_branch, body_case_id, body_coverage, body_state,
                        body_tokens, decode, state_rows)
from cases import O

DEV = "cuda:0"
SENTINEL = 0xFF     # a NaN in bf16 and fp32


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def eng():
    from cotracker_b200 import engine
    engine.lib()
    return engine


@pytest.fixture(scope="module")
def seeded():
    from cotracker_b200.synthetic import seeded_state_dict
    return seeded_state_dict(17, offline=True, window_len=60, head_gain=100.0, vis_gain=100.0)


def with_options(eng, opts, fn):
    before = {k: eng.get_option(k) for k in opts}
    for k, v in opts.items():
        eng.set_option(k, v)
    try:
        out = fn()
        torch.cuda.synchronize()
    finally:
        for k, v in before.items():
            eng.set_option(k, v)
    return out


def scratch_layout(T, N):
    """{buffer: (byte offset, bytes)} of the workspace of a {T, N, 0, 0, G = 1} pass up to the row bias (api_loop.cu:
    carve; consecutive buffers, each 1024-byte aligned)"""
    Rp, Rv = N * T, KV * T
    R = Rp + Rv
    sizes = (("vol", Rp * 4 * 2 * 2432 * 2), ("h1", Rp * 4 * 2 * 384 * 2), ("xs", Rp * 2 * 1152 * 2),
             ("tokens", R * C * 4), ("ln", R * 2 * C * 2), ("att", R * 2 * C * 2), ("qkv", R * 3 * C * 4),
             ("vqkv", Rv * 3 * C * 4), ("hmid", R * 2 * 1536 * 2), ("row_bias", T * C * 4))
    out, off = {}, 0
    for name, n in sizes:
        out[name] = (off, n)
        off = (off + n + 1023) // 1024 * 1024
    return out


class TraceWalk(BodyWalk):
    """get: the traced link, decoded to float64; emit: the link's worst err / bound, by link kind"""
    device = DEV

    def __init__(self, tr, heads_got, *a, **kw):
        super().__init__(*a, **kw)
        self.tr, self.heads_got = tr, heads_got
        self.worst, self.fails = {}, []

    def get(self, name):
        t = self.tr[name]
        return decode(t) if t.dtype == torch.bfloat16 else t.double()

    def emit(self, name, want, bd):
        kind = name.split(".", 1)[1] if name[0].isdigit() else name
        got = self.heads_got if name == "heads" else self.get(name)
        if name == "virtual_init":
            ok = torch.equal(self.tr[name], want.float())
            q = 0.0 if ok else float("inf")
        else:
            ok = bool(torch.isfinite(got).all())
            q = float(((got - want).abs() / bd).max()) if ok else float("inf")
        if not ok or q > 1.0:
            self.fails.append((name, q))
        self.worst[kind] = max(self.worst.get(kind, 0.0), q)


def run_case(eng, seeded, case):
    T, N, regime, gemm, attn, fuse = case
    sd = body_state(seeded, regime)
    packed = eng.pack_weights(sd, DEV)
    g = torch.Generator().manual_seed(zlib.crc32(body_case_id(case).encode()))
    tokens = body_tokens(N, T, regime, g).to(DEV)
    coords = (torch.rand(T, N, 2, generator=g) * 100).to(DEV)
    vis, conf = (torch.randn(T, N, generator=g) * 3).to(DEV), (torch.randn(T, N, generator=g) * 3).to(DEV)
    state0 = state_rows(coords, vis, conf).double()
    offs, nbytes, total = eng.body_trace_layout(T, N)
    torch.cuda.reset_peak_memory_stats()
    buf = torch.full((total,), SENTINEL, dtype=torch.uint8, device=DEV)
    ws = torch.full((eng.workspace_bytes(T, N),), SENTINEL, dtype=torch.uint8, device=DEV)
    tr = with_options(eng, {"gemm": gemm, "attn": attn, "fuse": fuse},
                      lambda: eng.body_trace(packed, tokens, coords, vis, conf, workspace=ws, trace=buf))
    walk = TraceWalk(tr, state_rows(coords, vis, conf).double(), sd, T, N, gemm, attn, fuse)
    walk.run(tokens.double(), state0)
    # trace bytes no link owns: the alignment gaps, and the time block's q|k|v when the fused kernel keeps it on chip
    untouched = [(o + n, nxt) for o, n, nxt in zip(offs, nbytes, offs[1:] + [total])]
    if walk.fused:
        untouched += [(o, o + n) for (name, _, _), o, n in zip(eng.body_trace_links(T, N), offs, nbytes)
                      if name.endswith("time.qkv")]
    # workspace bytes the body does not own: the scratch of the correlation half of an iteration and the row bias;
    # with the fused time kernel, the fp32 q|k|v buffer past the point rows' virtual <- point k|v [N*T, 768]
    sc = scratch_layout(T, N)
    ws_untouched = [(o, o + n) for k, (o, n) in sc.items() if k in ("vol", "h1", "xs", "row_bias")]
    if walk.fused:
        o, n = sc["qkv"]
        ws_untouched.append((o + N * T * 2 * C * 4, o + n))
    for what, mem, spans in (("trace", buf, untouched), ("workspace", ws, ws_untouched)):
        for a, b in spans:
            if b > a and int(mem[a:b].min()) != SENTINEL:   # SENTINEL is the largest uint8
                walk.fails.append((f"{what} bytes [{a}, {b}) that no link owns were written", float("inf")))
    # the token buffer ends as the last block left it: point rows from point <- virtual, virtual rows from virtual self
    o, n = sc["tokens"]
    tok_end = ws[o:o + n].view(torch.float32).view(-1, C)
    if not (torch.equal(tok_end[:N * T], tr[f"{DEPTH - 1}.p2v.fc2"])
            and torch.equal(tok_end[N * T:], tr[f"{DEPTH - 1}.vself.fc2"])):
        walk.fails.append(("the token rows after the last block are not the last links", float("inf")))
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    b = body_branch(T, N, gemm, attn, fuse, sms())
    print(f"\n  {body_case_id(case)}: {b}  peak {peak:.2f} GiB")
    for kind, q in walk.worst.items():
        print(f"    {kind:14s} {q:.3f}")
    return walk


@pytest.mark.gpu
def test_body_cases_reach_every_branch_on_this_device():
    n = sms()
    print(f"\n{n} SMs")
    for c in BODY_CASES:
        print(f"  {body_case_id(c)}: {body_branch(c[0], c[1], *c[3:], n)}")
    assert body_coverage(BODY_CASES, n) == []


@pytest.mark.gpu
@pytest.mark.parametrize("case", BODY_CASES, ids=[body_case_id(c) for c in BODY_CASES])
def test_body_links_within_their_bounds(eng, seeded, case):
    walk = run_case(eng, seeded, case)
    assert walk.fails == [], walk.fails[:10]


# ---------------------------------------------------------------------------------------------------------------------
# the composition is the loop
def _loop_inputs(sd, T, N, H4, W4, seed):
    g = torch.Generator().manual_seed(seed)
    fmaps = torch.randn(T, 128, H4, W4, generator=g) * 2.5
    support = torch.randn(4, 49, N, 128, generator=g)
    support = support / support.norm(dim=-1, keepdim=True)
    coords = torch.rand(1, N, 2, generator=g) * torch.tensor([W4 - 1.0, H4 - 1.0]) + torch.randn(T, N, 2, generator=g)
    vis, conf = torch.randn(T, N, generator=g) * 3, torch.randn(T, N, generator=g) * 3
    valid = torch.ones(N, dtype=torch.uint8)
    te = O.time_embedding(sd, T)[0].contiguous()
    return fmaps, support, coords.contiguous(), vis, conf, valid, te


@pytest.mark.gpu
@pytest.mark.parametrize("gemm", [0, 1])
@pytest.mark.parametrize("iters", [1, 4])
@pytest.mark.parametrize("N,T", [(5, 8), (600, 16)])
def test_update_loop_is_loop_tokens_then_body_trace(eng, seeded, N, T, iters, gemm):
    H4, W4 = 24, 32
    sd = body_state(seeded, "default")
    packed = eng.pack_weights(sd, DEV)
    fmaps, support, coords, vis, conf, valid, te = (t.to(DEV) for t in _loop_inputs(sd, T, N, H4, W4, N + T))
    pyr = eng.prepare_pyramid(fmaps)
    loop = [t.clone() for t in (coords, vis, conf)]
    body = [t.clone() for t in (coords, vis, conf)]

    def run():
        ws = torch.empty(eng.workspace_bytes(T, N, H4, W4), dtype=torch.uint8, device=DEV)
        eng.update_loop(packed, pyr, H4, W4, support, valid, *loop, te, iters, ws)
        for _ in range(iters):
            *_, tok = eng.loop_tokens(packed, pyr, H4, W4, support, valid, *body, te, raw=True)
            eng.body_trace(packed, tok, *body)
    with_options(eng, {"gemm": gemm}, run)
    for name, a, b in zip(("coords", "vis", "conf"), loop, body):
        assert torch.equal(a, b), (name, float((a - b).abs().max()))
    assert not torch.equal(loop[0], coords)
