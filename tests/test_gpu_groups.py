"""Grouped calls on the GPU: G independent query sets over one clip in one pass (ct3_loop_shape.G,
ct3_updateformer's groups, forward_groups, single-point EvaluationPredictor).  Each group's outputs must be
bit-identical to a standalone call on that group's tracks alone."""
import numpy as np
import pytest
import torch

from cases import O, load_golden

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# not multiples of 128; groups of <= 64 tracks take the mma.sync point<-virtual kernel, the others the wgmma one
SIZES = [90, 1, 129, 300, 64, 255]


@pytest.fixture(scope="module")
def eng():
    from cotracker_b200 import engine
    engine.lib()
    return engine


@pytest.fixture(scope="module")
def sd():
    from cotracker_b200.synthetic import seeded_state_dict
    return seeded_state_dict(71, offline=True, window_len=60, head_gain=10.0, vis_gain=100.0)


def _bounds(sizes):
    b = np.concatenate([[0], np.cumsum(sizes)]).tolist()
    return list(zip(b[:-1], b[1:]))


def _loop_case(T, sizes, H4=64, W4=72, seed=0):
    """Pyramid, support and initial state of a synthetic update-loop problem (64x72: the production correlation kernel)."""
    g = torch.Generator().manual_seed(seed)
    N = sum(sizes)
    fmaps = torch.randn(T, 128, H4, W4, generator=g)
    qf = torch.randint(0, T, (N,), generator=g)
    qc = torch.stack([torch.rand(N, generator=g) * (W4 - 1), torch.rand(N, generator=g) * (H4 - 1)], dim=1)
    valid = (torch.rand(N, generator=g) < 0.9).to(torch.uint8)
    return fmaps, qf, qc, valid


def _run_loop(eng, packed, pyr, H4, W4, support, valid, c0, te, iters, group_sizes=None):
    T, N, _ = c0.shape
    coords, vis, conf = c0.clone(), torch.zeros(T, N, device=DEV), torch.zeros(T, N, device=DEV)
    G = 1 if group_sizes is None else len(group_sizes)
    ws = torch.empty(eng.workspace_bytes(T, N, H4, W4, groups=G), dtype=torch.uint8, device=DEV)
    eng.update_loop(packed, pyr, H4, W4, support, valid, coords, vis, conf, te, iters, ws, group_sizes=group_sizes)
    return coords, vis, conf


def _loop_inputs(eng, sd, T, sizes, seed=0, H4=64, W4=72):
    fmaps, qf, qc, valid = _loop_case(T, sizes, H4, W4, seed)
    pyr = eng.prepare_pyramid(fmaps.to(DEV))
    support = eng.sample_support(pyr, T, H4, W4, qf.to(torch.int32).to(DEV).contiguous(), qc.to(DEV).contiguous())
    c0 = qc.to(DEV)[None].expand(T, -1, 2).contiguous()
    te = O.time_embedding(sd, T)[0].contiguous().to(DEV)
    return pyr, support, valid.to(DEV), c0, te


@pytest.mark.parametrize("T", [12, 150])   # 150 > 128: the separate time-attention kernels
def test_update_loop_groups_bit_identical_to_standalone(eng, sd, T):
    H4, W4, iters = 64, 72, 2
    pyr, support, valid, c0, te = _loop_inputs(eng, sd, T, SIZES, seed=T)
    packed = eng.pack_weights(sd, DEV)
    got = _run_loop(eng, packed, pyr, H4, W4, support, valid, c0, te, iters, SIZES)
    assert float((got[0] - c0).abs().max()) > 0.25, "case must move"
    for a, b in _bounds(SIZES):
        want = _run_loop(eng, packed, pyr, H4, W4, support[:, :, a:b].contiguous(), valid[a:b].contiguous(),
                         c0[:, a:b].contiguous(), te, iters)
        for x, y in zip(got, want):
            assert torch.equal(x[:, a:b], y), (T, a, b, float((x[:, a:b] - y).abs().max()))


@pytest.mark.parametrize("T", [12, 150])
def test_updateformer_groups_bit_identical_to_standalone(eng, sd, T):
    g = torch.Generator().manual_seed(T + 1)
    x = torch.randn(sum(SIZES), T, 1110, generator=g).to(DEV)
    packed = eng.pack_weights(sd, DEV)
    got = eng.updateformer(packed, x, group_sizes=SIZES)
    for a, b in _bounds(SIZES):
        want = eng.updateformer(packed, x[a:b].contiguous())
        assert torch.equal(got[a:b], want), (T, a, b, float((got[a:b] - want).abs().max()))
    # G = 1 through the grouped entry point is the plain call
    assert torch.equal(eng.updateformer(packed, x, group_sizes=[x.shape[0]]), eng.updateformer(packed, x))


def test_groups_are_isolated(eng, sd):
    """Moving one group's queries changes nothing in any other group."""
    T, H4, W4, iters = 12, 64, 72, 2
    pyr, support, valid, c0, te = _loop_inputs(eng, sd, T, SIZES, seed=5)
    packed = eng.pack_weights(sd, DEV)
    base = _run_loop(eng, packed, pyr, H4, W4, support, valid, c0, te, iters, SIZES)
    a, b = _bounds(SIZES)[2]
    c1 = c0.clone()
    c1[:, a:b] += 3.0
    sup1 = support.clone()
    sup1[:, :, a:b] *= 0.5
    moved = _run_loop(eng, packed, pyr, H4, W4, sup1, valid, c1, te, iters, SIZES)
    assert not torch.equal(moved[0][:, a:b], base[0][:, a:b])
    for k, (a2, b2) in enumerate(_bounds(SIZES)):
        if k == 2:
            continue
        for x, y in zip(moved, base):
            assert torch.equal(x[:, a2:b2], y[:, a2:b2]), k


def test_grouped_tensor_cores_match_simt(eng, sd):
    """The grouped call on the exact-fp32 verification kernels (gemm / corr / attn = 1) within 1e-3 px."""
    T, H4, W4, iters = 12, 64, 72, 2
    pyr, support, valid, c0, te = _loop_inputs(eng, sd, T, SIZES, seed=9)
    packed = eng.pack_weights(sd, DEV)
    tc = _run_loop(eng, packed, pyr, H4, W4, support, valid, c0, te, iters, SIZES)
    for k in ("gemm", "corr", "attn"):
        eng.set_option(k, 1)
    try:
        simt = _run_loop(eng, packed, pyr, H4, W4, support, valid, c0, te, iters, SIZES)
        torch.cuda.synchronize()
    finally:
        for k in ("gemm", "corr", "attn"):
            eng.set_option(k, 0)
    e_c = float((tc[0] - simt[0]).abs().max()) * 4     # pixels
    e_v = float((tc[1] - simt[1]).abs().max())
    e_q = float((tc[2] - simt[2]).abs().max())
    assert e_c < 1e-3 and e_v < 1e-3 and e_q < 1e-3, (e_c, e_v, e_q)


def _group_queries(sizes, T, H, W, seed):
    from cotracker_b200.synthetic import random_queries
    return torch.cat([random_queries(n, T, H, W, seed=seed + k) for k, n in enumerate(sizes)], dim=1)


@pytest.mark.parametrize("online", [False, True])
def test_forward_groups_bit_identical_to_forward(sd, online):
    from cotracker_b200.build import build_cotracker
    from cotracker_b200.synthetic import seeded_state_dict, texture_video
    T, H, W = (12, 256, 288) if not online else (27, 256, 288)
    state = sd if not online else seeded_state_dict(72, offline=False, window_len=16, head_gain=5.0, vis_gain=30.0)
    model = build_cotracker(None, offline=not online, window_len=60 if not online else 16).eval()
    model.load_state_dict(state)
    model = model.to(DEV)
    video = texture_video(T, H, W, seed=3).to(DEV)
    queries = _group_queries(SIZES, T, H, W, seed=40).to(DEV)
    got = model.forward_groups(video, queries, SIZES, iters=2)
    for a, b in _bounds(SIZES):
        want = model(video, queries[:, a:b].contiguous(), iters=2)
        for x, y in zip(got[:3], want[:3]):
            assert torch.equal(x[:, :, a:b], y), (online, a, b, float((x[:, :, a:b] - y).abs().max()))
    # forward is forward_groups with one group
    one = model.forward_groups(video, queries, [queries.shape[1]], iters=2)
    full = model(video, queries, iters=2)
    for x, y in zip(one[:3], full[:3]):
        assert torch.equal(x, y)


def _eval_model():
    from cotracker_b200.build import build_cotracker
    from oracle.make_eval_single_golden import eval_single_inputs
    sd, video, queries = eval_single_inputs()
    model = build_cotracker(None, offline=True, window_len=60).eval()
    model.load_state_dict(sd)
    return model.to(DEV), video.to(DEV), queries.to(DEV)


def test_evaluation_predictor_partition_independent():
    """The single-point predictor gives identical outputs with one group per pass, two passes and one pass."""
    from cotracker_b200.evaluation import EvaluationPredictor, pass_bytes
    model, video, queries = _eval_model()
    n_q, T = queries.shape[1], video.shape[1]
    half = pass_bytes(T, 90 * (n_q // 2), n_q // 2, 96, 128)
    out = {}
    for name, budget in (("each", 1), ("two", half), ("one", 1 << 50)):
        ev = EvaluationPredictor(model, single_point=True, grid_size=5, local_grid_size=8, pass_budget_bytes=budget)
        out[name] = ev(video, queries)
    from cotracker_b200.evaluation import plan_passes
    assert len(plan_passes([90] * n_q, T, 96, 128, half)) == 2
    for name in ("two", "one"):
        assert torch.equal(out[name][0], out["each"][0]) and torch.equal(out[name][1], out["each"][1]), name


def test_evaluation_predictor_single_point_matches_reference_golden():
    """tests/golden/eval_predictor_single_t24.npz: the reference's single-point EvaluationPredictor, 12 queries at
    varied frames over 24 frames (oracle/make_eval_single_golden.py)."""
    from cotracker_b200.evaluation import EvaluationPredictor
    model, video, queries = _eval_model()
    want = load_golden("eval_predictor_single_t24")
    assert len(set(queries[0, :, 0].tolist())) > 4, "query frames must vary"
    ev = EvaluationPredictor(model, single_point=True, grid_size=5, local_grid_size=8)
    tracks, vis = ev(video, queries)
    e_t = float((tracks.cpu() - want["tracks"]).abs().max())
    e_v = float((vis.cpu() - want["vis"]).abs().max())
    assert e_t < 1e-3 and e_v < 1e-3, (e_t, e_v)
