"""Track slabs on the GPU (ct3_loop_shape.slab_tracks, DESIGN.md §4.4.5): coords / vis / conf bit-identical to the call
without slabs for every slab size, call kind, both time-attention routes and the A/B options; nothing outside the
queried workspace is written; the offline predictor under a budget that forces slabs returns what it returns without."""
import pytest
import torch

from cases import CASES, O, case_inputs, compare, load_golden, predictor_kwargs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SIZES = [90, 1, 200]          # ragged groups: slabs of 7, 64 and 129 tracks cross group boundaries


@pytest.fixture(scope="module")
def eng():
    from cotracker_b200 import engine
    engine.lib()
    return engine


@pytest.fixture(scope="module")
def sd():
    from cotracker_b200.synthetic import seeded_state_dict
    return seeded_state_dict(91, offline=True, window_len=60, head_gain=10.0, vis_gain=100.0)


def _inputs(eng, sd, T, H4, W4, seed):
    """A pyramid of T frames, support at random query frames, initial coords at the query points."""
    g = torch.Generator().manual_seed(seed)
    N = sum(SIZES)
    fmaps = torch.randn(T, 128, H4, W4, generator=g).to(DEV)
    qf = torch.randint(0, T, (N,), generator=g)
    qc = torch.stack([torch.rand(N, generator=g) * (W4 - 1), torch.rand(N, generator=g) * (H4 - 1)], dim=1).to(DEV)
    valid = (torch.rand(N, generator=g) < 0.9).to(torch.uint8).to(DEV)
    pyr = eng.prepare_pyramid(fmaps)
    support = eng.sample_support(pyr, T, H4, W4, qf.to(torch.int32).to(DEV).contiguous(), qc)
    c0 = (qc[None] + torch.randn(T, N, 2, generator=g).to(DEV)).contiguous()
    te = O.time_embedding(sd, T)[0].contiguous().to(DEV)
    return pyr, support, valid, c0, te


def _kind_args(kind, T):
    if kind == "plain":
        return None, None
    if kind == "grouped":
        return SIZES, None
    return SIZES, [list(range(T)), list(range(T - 1, -1, -1)), list(range(T))]   # frames: group 1 reversed


def _loop(eng, packed, inp, H4, W4, iters, sizes, frames, slab=None, extra=0):
    pyr, support, valid, c0, te = inp
    T, N, _ = c0.shape
    g = torch.Generator().manual_seed(5)
    coords = c0.clone()
    vis = torch.randn(T, N, generator=g).to(DEV)
    conf = torch.randn(T, N, generator=g).to(DEV)
    G = 1 if sizes is None else len(sizes)
    T_pyr = None if frames is None else eng.pyramid_frames(pyr, H4, W4)
    need = eng.workspace_bytes(T, N, H4, W4, groups=G, frames=T_pyr, slab_tracks=slab)
    ws = torch.full((need + extra,), 0xA5, dtype=torch.uint8, device=DEV)
    eng.update_loop(packed, pyr, H4, W4, support, valid, coords, vis, conf, te, iters, ws, group_sizes=sizes,
                    group_frames=frames, slab_tracks=slab)
    torch.cuda.synchronize()
    return (coords, vis, conf), ws[need:]


def _same(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b))


# T = 1 .. 128: the fused q|k|v + time-attention kernel; T = 160: the separate projection and per-warp attention
# (64, 72): every level >= 8x8, corr_tc3.cu;  (24, 32): level 3 is 3x4, corr_tc.cu
@pytest.mark.parametrize("T,hw", [(1, (64, 72)), (16, (64, 72)), (60, (24, 32)), (128, (64, 72)), (160, (64, 72))])
@pytest.mark.parametrize("kind", ["plain", "grouped", "frames"])
def test_slabbed_bit_identical_to_unslabbed(eng, sd, T, hw, kind):
    H4, W4 = hw
    packed = eng.pack_weights(sd, DEV)
    inp = _inputs(eng, sd, T, H4, W4, seed=T)
    sizes, frames = _kind_args(kind, T)
    want, _ = _loop(eng, packed, inp, H4, W4, 2, sizes, frames)
    N = sum(SIZES)
    for slab in (1, 7, 64, 129, N):
        got, _ = _loop(eng, packed, inp, H4, W4, 2, sizes, frames, slab)
        assert _same(got, want), (T, kind, slab)


@pytest.mark.parametrize("opt", [("attn", 1), ("gemm", 1), ("fuse", 0), ("prec.fc1", 2), ("corr", 1),
                                 ("prec.corr", 3)])
def test_slabbed_bit_identical_under_options(eng, sd, opt):
    """Each A/B option: slabbed against the unslabbed call under the same option."""
    T, H4, W4 = 16, 64, 72
    packed = eng.pack_weights(sd, DEV)
    inp = _inputs(eng, sd, T, H4, W4, seed=3)
    name, value = opt
    old = eng.get_option(name)
    eng.set_option(name, value)
    try:
        for kind in ("grouped", "frames"):
            sizes, frames = _kind_args(kind, T)
            want, _ = _loop(eng, packed, inp, H4, W4, 2, sizes, frames)
            for slab in (7, 129):
                got, _ = _loop(eng, packed, inp, H4, W4, 2, sizes, frames, slab)
                assert _same(got, want), (opt, kind, slab)
    finally:
        eng.set_option(name, old)


@pytest.mark.parametrize("slab", [1, 64])
def test_slabbed_writes_only_its_workspace(eng, sd, slab):
    """The pyramid and support are read-only and no byte past ct3_workspace_bytes(shape) changes."""
    T, H4, W4 = 20, 64, 72
    packed = eng.pack_weights(sd, DEV)
    inp = _inputs(eng, sd, T, H4, W4, seed=4)
    pyr0, sup0 = inp[0].clone(), inp[1].clone()
    sizes, frames = _kind_args("frames", T)
    _, tail = _loop(eng, packed, inp, H4, W4, 2, sizes, frames, slab, extra=1 << 20)
    assert bool((tail == 0xA5).all())
    assert torch.equal(inp[0], pyr0) and torch.equal(inp[1], sup0)


def _predictor_runs(monkeypatch, name):
    """The offline predictor on golden case `name` as grid, queries + support grid and backward tracking, without and
    with a pass budget that forces track slabs; every call that ran in slabs is recorded."""
    import cotracker_b200.model as M
    from cotracker_b200.predictor import CoTrackerPredictor
    cfg = CASES[name]
    sd, video, queries = case_inputs(cfg)
    p = CoTrackerPredictor(checkpoint=None, window_len=cfg["window_len"])
    p.model.load_state_dict(sd)
    p = p.to(DEV)
    video, queries = video.to(DEV), queries.to(DEV)
    calls = [dict(grid_size=4), dict(queries=queries, grid_size=3), predictor_kwargs(cfg, video, queries)]
    with torch.no_grad():
        want = [p(video, **kw) for kw in calls]
        slabs = []
        real = M.engine.update_loop

        def spy(*a, **k):
            slabs.append(k.get("slab_tracks"))
            return real(*a, **k)

        monkeypatch.setattr(M, "pass_budget_bytes", lambda *a, **k: 1)
        monkeypatch.setattr(M.engine, "update_loop", spy)
        got = [p(video, **kw) for kw in calls]
    return want, got, slabs


def test_offline_predictor_with_forced_slabs_matches(monkeypatch):
    name = "pred_backward"
    assert CASES[name].get("backward")
    want, got, slabs = _predictor_runs(monkeypatch, name)
    assert slabs and all(s == 1 for s in slabs)                     # nothing fits a 1-byte budget: one track a slab
    for w, g in zip(want, got):
        assert torch.equal(g[0], w[0]) and torch.equal(g[1], w[1])
    tr, vi = got[2]
    compare(dict(tracks=tr.cpu(), visibility=vi.cpu()), load_golden(name), tol_px=1e-3, tol_logit=1e-3)
