"""CPU tests of the transformer-body stage entry points (ct3_linear_ex, ct3_layernorm, ct3_time_block_attention and its
workspace query): every invalid argument returns CT3_EINVAL, or CT3_ENOSPC for a too small workspace, before any
launch.  All device pointers are fake and the stream is the legacy default, so reaching a launch would fail
differently (and a valid argument list is never passed)."""
import ctypes
import math

from cotracker_b200 import engine

EINVAL, ENOSPC = -1, -3
BODY_SYMBOLS = ("ct3_linear_ex", "ct3_layernorm", "ct3_time_block_attention_workspace_bytes", "ct3_time_block_attention")


def _p(addr):
    return ctypes.c_void_p(addr)


def test_body_symbols_exported():
    lib = engine.lib()
    for name in BODY_SYMBOLS:
        assert hasattr(lib, name) and name in engine.EXPORTED_SYMBOLS, name


# a valid problem: M = 10 rows, Nout = 128, Kpad = 64, fp32 output of pitch 128 (every case below breaks one thing)
LINEAR = dict(x=_p(1 << 20), x_ld=0, w=_p(1 << 21), bias=None, M=10, Nout=128, Kpad=64, products=3, fp16=0, act=0,
              row_bias=None, row_mod=1, y=_p(1 << 22), ld_y=128, residual=0, y_split=None, ld_split=0, lo_off=0,
              row_group=1)
SPLIT = dict(y=None, y_split=_p(1 << 23), ld_split=256, lo_off=128)   # a valid split output instead of y


def _linear(**kw):
    a = dict(LINEAR, **kw)
    return engine.lib().ct3_linear_ex(a["x"], a["x_ld"], a["w"], a["bias"], a["M"], a["Nout"], a["Kpad"], a["products"],
                                      a["fp16"], a["act"], a["row_bias"], a["row_mod"], a["y"], a["ld_y"], a["residual"],
                                      a["y_split"], a["ld_split"], a["lo_off"], a["row_group"], None)


def test_linear_ex_rejects_bad_epilogues_without_gpu():
    lib = engine.lib()
    cases = [
        (dict(x=None), b"null argument"),
        (dict(w=None), b"null argument"),
        (dict(y=None), b"no output"),                                    # neither y nor y_split
        (dict(M=0), b"M>0"),
        (dict(Nout=100), b"N % 128"),
        (dict(Kpad=96), b"Kpad % 64"),
        (dict(act=3), b"act in 0..2"),
        (dict(act=-1), b"act in 0..2"),
        (dict(products=0), b"products in 1..3"),
        (dict(products=4), b"products in 1..3"),
        (dict(fp16=2), b"fp16 in 0..1"),
        (dict(x_ld=64), b"x_ld too small"),                              # 3 products read two planes of 64
        (dict(x_ld=132), b"x_ld"),                                       # not a multiple of 8
        (dict(products=2, x_ld=60), b"x_ld too small"),
        (dict(row_mod=0), b"row_mod >= 1"),
        (dict(row_group=0), b"row_group >= 1"),
        (dict(residual=2), b"residual"),
        (dict(SPLIT, residual=1), b"residual"),                          # accumulate into no fp32 output
        (dict(ld_y=127), b"fp32 output pitch"),                          # < Nout
        (dict(ld_y=130), b"fp32 output pitch"),                          # not a multiple of 4
        (dict(SPLIT, ld_split=260), b"multiples of 8"),
        (dict(SPLIT, lo_off=132, ld_split=264), b"multiples of 8"),
        (dict(SPLIT, lo_off=120), b"overlap"),                           # lo plane starts inside the hi plane
        (dict(SPLIT, ld_split=248), b"overlap"),                         # next row's hi plane inside this lo plane
        (dict(SPLIT, row_group=2), b"overlap"),                          # 2 rows of 128 per plane: lo_off >= 256
        (dict(SPLIT, row_group=2, lo_off=256, ld_split=504), b"overlap"),
        (dict(x=_p((1 << 20) + 8)), b"operands must be 16-byte aligned"),
        (dict(w=_p((1 << 21) + 2)), b"operands must be 16-byte aligned"),
        (dict(bias=_p((1 << 24) + 4)), b"16-byte aligned"),
        (dict(row_bias=_p((1 << 24) + 8)), b"16-byte aligned"),
        (dict(y=_p((1 << 22) + 4)), b"16-byte aligned"),
        (dict(SPLIT, y_split=_p((1 << 23) + 8)), b"16-byte aligned"),
    ]
    for kw, msg in cases:
        assert _linear(**kw) == EINVAL, kw
        assert msg in lib.ct3_last_error(), (kw, lib.ct3_last_error(), msg)
    # ct3_linear and ct3_linear_prec are the same call: the same checks, the same messages
    x, w, y = LINEAR["x"], LINEAR["w"], LINEAR["y"]
    assert lib.ct3_linear(x, w, None, 10, 100, 64, 0, y, None) == EINVAL and b"N % 128" in lib.ct3_last_error()
    assert lib.ct3_linear(x, w, None, 10, 128, 64, 0, None, None) == EINVAL and b"no output" in lib.ct3_last_error()
    assert lib.ct3_linear(x, w, _p((1 << 24) + 4), 10, 128, 64, 0, y, None) == EINVAL
    assert lib.ct3_linear_prec(x, w, None, 10, 128, 64, 0, 0, 0, y, None) == EINVAL
    assert lib.ct3_linear_prec(x, w, None, 10, 128, 64, 0, 3, 2, y, None) == EINVAL and b"fp16" in lib.ct3_last_error()
    assert lib.ct3_linear_prec(x, w, None, 0, 128, 64, 0, 3, 0, y, None) == EINVAL


def test_layernorm_rejects_bad_arguments_without_gpu():
    lib = engine.lib()
    base = dict(x=_p(1 << 20), rows=5, gamma=_p(1 << 21), beta=_p(1 << 22), eps=1e-5, out=_p(1 << 23))

    def call(**kw):
        a = dict(base, **kw)
        return lib.ct3_layernorm(a["x"], a["rows"], a["gamma"], a["beta"], a["eps"], a["out"], None)

    cases = [
        (dict(x=None), b"null argument"),
        (dict(out=None), b"null argument"),
        (dict(gamma=None), b"together"),
        (dict(beta=None), b"together"),
        (dict(rows=0), b"rows"),
        (dict(rows=-3), b"rows"),
        (dict(eps=-1e-6), b"eps"),
        (dict(eps=math.inf), b"eps"),
        (dict(eps=math.nan), b"eps"),
        (dict(x=_p((1 << 20) + 4)), b"16-byte"),
        (dict(gamma=_p((1 << 21) + 8)), b"16-byte"),
        (dict(beta=_p((1 << 22) + 4)), b"16-byte"),
        (dict(out=_p((1 << 23) + 8)), b"16-byte"),
    ]
    for kw, msg in cases:
        assert call(**kw) == EINVAL, kw
        assert msg in lib.ct3_last_error(), (kw, lib.ct3_last_error(), msg)


def test_time_block_attention_rejects_bad_arguments_without_gpu():
    lib = engine.lib()
    n = ctypes.c_size_t(0)
    assert lib.ct3_time_block_attention_workspace_bytes(60, 600, ctypes.byref(n)) == 0
    need = n.value
    assert need >= 600 * 1152 * 4                                        # fp32 q|k|v of the unfused route
    assert lib.ct3_time_block_attention_workspace_bytes(60, 600, None) == EINVAL
    for T, rows in ((0, 10), (-1, 10), (4, 0), (4, 10), (7, 50)):
        assert lib.ct3_time_block_attention_workspace_bytes(T, rows, ctypes.byref(n)) == EINVAL, (T, rows)
        assert b"rows % T" in lib.ct3_last_error()
    base = dict(packed=_p(1 << 20), depth=0, x=_p(1 << 21), T=60, rows=600, out=_p(1 << 22), ws=_p(1 << 24),
                bytes=need)

    def call(**kw):
        a = dict(base, **kw)
        return lib.ct3_time_block_attention(a["packed"], a["depth"], a["x"], a["T"], a["rows"], a["out"], a["ws"],
                                            a["bytes"], None)

    cases = [
        (dict(packed=None), b"null argument"),
        (dict(x=None), b"null argument"),
        (dict(out=None), b"null argument"),
        (dict(ws=None), b"null argument"),
        (dict(depth=-1), b"depth"),
        (dict(depth=3), b"depth"),
        (dict(T=0), b"rows % T"),
        (dict(rows=0), b"rows % T"),
        (dict(rows=610), b"rows % T"),
        (dict(packed=_p((1 << 20) + 8)), b"16-byte"),
        (dict(x=_p((1 << 21) + 8)), b"16-byte"),
        (dict(out=_p((1 << 22) + 4)), b"16-byte"),
        (dict(ws=_p((1 << 24) + 16)), b"256-byte"),
    ]
    for kw, msg in cases:
        assert call(**kw) == EINVAL, kw
        assert msg in lib.ct3_last_error(), (kw, lib.ct3_last_error(), msg)
    assert call(bytes=need - 1) == ENOSPC and b"workspace too small" in lib.ct3_last_error()
    assert call(bytes=0) == ENOSPC


# =====================================================================================================================
# ct3_body_trace: the float64 restatement (tests/body_cases.py), its layout and its argument checks
def _oracle_case(N, T, regime, seed):
    """(state dict, x [N, T, 1110], point tokens float64 [N*T, 384], state rows [N*T, 4]) of a small seeded case"""
    import torch

    from body_cases import TOKEN_SCALE, body_state
    from cases import O
    from cotracker_b200.synthetic import seeded_state_dict
    sd = body_state(seeded_state_dict(17, offline=True, window_len=60, head_gain=100.0, vis_gain=100.0), regime)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, T, 1110, generator=g, dtype=torch.float64)
    sd64 = {k: v.double() for k, v in sd.items()}
    if regime == "norm_context":   # point tokens of variance about 1e-6, as body_tokens gives them
        for k in ("weight", "bias"):
            sd64["updateformer.input_transform." + k] = sd64["updateformer.input_transform." + k] * TOKEN_SCALE
    tokens = O.linear(sd64, "updateformer.input_transform", x).reshape(N * T, 384)
    state = torch.randn(N * T, 4, generator=g, dtype=torch.float64) * 10
    return sd, sd64, x, tokens, state


def test_body_restatement_is_the_model():
    """The link restatements chained on their own float64 outputs reproduce oracle.updateformer and the state update,
    with the default seeded weights and with an affine norm_context whose input variance is below its eps."""
    import torch

    from body_cases import SelfWalk, ln_ref
    from cases import O
    for N, T, regime in ((5, 3, "default"), (70, 6, "default"), (70, 6, "norm_context"), (3, 2, "sharp")):
        sd, sd64, x, tokens, state = _oracle_case(N, T, regime, N * 100 + T)
        walk = SelfWalk(sd, T, N, fuse=0)   # the fused route re-splits its input, which only the trace holds exactly
        walk.run(tokens, state)
        ln = O.ln   # the oracle with the eps the kernels add, fp32 (it decides the LayerNorms below eps)
        O.ln = lambda xx, eps, w_=None, b_=None: ln(xx, float(torch.tensor(eps, dtype=torch.float32)), w_, b_)
        try:
            with torch.no_grad():
                delta = O.updateformer(sd64, x[None])[0].reshape(N * T, 4)
        finally:
            O.ln = ln
        want = state + delta
        err = float((walk.out["heads"] - want).abs().max())
        assert err <= 1e-12 * float(want.abs().max()), (N, T, regime, err)
        if regime == "norm_context":
            # the context the first virtual <- point block normalises is below eps: eps 1e-6 there moves it by far more
            # than its bound
            pts = walk.out["0.time.fc2"][:N * T]
            assert float(pts.var(1, unbiased=False).max()) < 1e-5
            w = walk.w["updateformer.space_virtual2point_blocks.0.norm_context.weight"]
            b = walk.w["updateformer.space_virtual2point_blocks.0.norm_context.bias"]
            want_ln, bd = ln_ref(pts, 1e-5, w, b)
            assert float(((ln_ref(pts, 1e-6, w, b)[0] - want_ln).abs() / bd).amax(1).min()) > 10.0


def test_body_trace_links_match_the_layout():
    import torch

    from body_cases import SelfWalk
    for T, N in ((1, 1), (2, 3), (16, 6400), (60, 1225), (129, 5)):
        offs, nb, total = engine.body_trace_layout(T, N)
        links = engine.body_trace_links(T, N)
        assert len(links) == engine.BODY_TRACE_LINKS == len(offs)
        end = 0
        for (name, dtype, shape), o, n in zip(links, offs, nb):
            assert n == math.prod(shape) * dtype.itemsize, name
            assert o >= end and o % 256 == 0, name
            end = o + n
        assert total >= end and total - end < 256
    # the restatement walks exactly these links, in this order
    sd, _, _, tokens, state = _oracle_case(3, 2, "default", 1)

    class Names(SelfWalk):
        def emit(self, name, want, bd):
            self.names = getattr(self, "names", []) + [name]
            super().emit(name, want, bd)
    walk = Names(sd, 2, 3, fuse=0)
    walk.run(tokens, state)
    assert walk.names == [n for n, _, _ in engine.body_trace_links(2, 3)] + ["heads"]
    for name, dtype, shape in engine.body_trace_links(2, 3):
        assert tuple(walk.out[name].shape) == (shape[0], shape[1] // 2 if dtype == torch.bfloat16 else shape[1]), name


def test_body_trace_rejects_bad_arguments_without_gpu():
    lib = engine.lib()
    n = ctypes.c_size_t(0)
    assert lib.ct3_body_trace_layout(16, 100, None, None, ctypes.byref(n)) == 0
    trace_need = n.value
    assert lib.ct3_body_trace_layout(16, 100, None, None, None) == EINVAL
    for T, N in ((0, 5), (5, 0), (-1, 5)):
        assert lib.ct3_body_trace_layout(T, N, None, None, ctypes.byref(n)) == EINVAL
        assert b"T and N must be >= 1" in lib.ct3_last_error()
    ws_need = engine.workspace_bytes(16, 100)
    base = dict(packed=_p(1 << 20), tokens=_p(1 << 21), T=16, N=100, coords=_p(1 << 22), vis=_p(1 << 23),
                conf=_p(1 << 24), trace=_p(1 << 30), trace_bytes=trace_need, ws=_p(1 << 34), ws_bytes=ws_need)

    def call(**kw):
        a = dict(base, **kw)
        return lib.ct3_body_trace(a["packed"], a["tokens"], a["T"], a["N"], a["coords"], a["vis"], a["conf"],
                                  a["trace"], a["trace_bytes"], a["ws"], a["ws_bytes"], None)

    for k in ("packed", "tokens", "coords", "vis", "conf", "trace", "ws"):
        assert call(**{k: None}) == EINVAL and b"null argument" in lib.ct3_last_error(), k
    cases = [
        (dict(T=0), b"T and N must be >= 1"),
        (dict(N=0), b"T and N must be >= 1"),
        (dict(T=1 << 20, N=1 << 20), b"problem too large"),
        (dict(ws=_p((1 << 34) + 16)), b"256-byte"),
        (dict(trace=_p((1 << 30) + 64)), b"256-byte"),
    ]
    for kw, msg in cases:
        assert call(**kw) == EINVAL, kw
        assert msg in lib.ct3_last_error(), (kw, lib.ct3_last_error(), msg)
    assert call(ws_bytes=ws_need - 1) == ENOSPC and b"workspace too small" in lib.ct3_last_error()
    assert call(trace_bytes=trace_need - 1) == ENOSPC and b"trace buffer too small" in lib.ct3_last_error()


def test_body_branch_map_pinned():
    """The body's branch map at an H100 SXM (132 SMs) and a PCIe card (114): the case list of test_gpu_body_trace.py
    reaches every branch on both"""
    from body_cases import BODY_CASES, body_branch, body_coverage
    for sms in (132, 114):
        assert body_coverage(BODY_CASES, sms) == [], sms
    b = body_branch(16, 6400, 0, 0, 1, 132)
    assert b["time"] == {"path": "fused"} and b["v2p"] == {"path": "split_k", "splits": 4}
    assert b["p2v"] == {"path": "wgmma", "ragged_tile": False} and b["vself"]["path"] == "shared"
    assert body_branch(16, 6400, 0, 0, 1, 114)["v2p"] == {"path": "split_k", "splits": 7}
    assert body_branch(48, 600, 0, 0, 1, 132)["v2p"]["path"] == "shared"
    assert body_branch(20, 65, 0, 0, 1, 132)["p2v"] == {"path": "wgmma", "ragged_tile": True}
    assert body_branch(20, 64, 0, 0, 1, 132)["p2v"]["path"] == "shared"
    assert body_branch(129, 5, 0, 0, 1, 132)["time"]["path"] == "per_warp"
    assert [body_branch(T, 3, 0, 0, 0, 132)["time"]["kb"] for T in (2, 24, 40)] == [16, 32, 64]
    assert body_branch(24, 200, 1, 0, 1, 132)["time"]["path"] == "per_warp"
    assert body_branch(24, 200, 0, 1, 1, 132)["time"] == {"path": "simt"}
