"""GPU tests of clips of different lengths in one update-loop pass (ct3_loop_shape.group_T) and of the predictor's list
call: every group of a padded pass, and every clip of a list call, is bit-identical (torch.equal) to its own pass or
call, under the default kernels, fuse = 0, the exact-fp32 verification options and forced track slabs; a list holding
the clips of reference goldens still meets each golden."""
import numpy as np
import pytest
import torch

from cases import case_inputs, compare, load_golden, predictor_kwargs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
H, W = 96, 128


def _model(seed=41):
    from cotracker_b200.build import build_cotracker
    from cotracker_b200.synthetic import seeded_state_dict
    m = build_cotracker(None, offline=True, window_len=60).eval()
    m.load_state_dict(seeded_state_dict(seed, offline=True, window_len=60, head_gain=10.0, vis_gain=100.0))
    return m.to(DEV)


# ---- loop level ---------------------------------------------------------------------------------------------------
# 130 frames take the unfused time attention; 60 = window_len uses the time embedding as it is, every other length
# interpolates it; 600 tracks at 16 frames make attention_tc_splits split the virtual <- point attention; 70 > 64
# tracks take the wgmma point <- virtual kernel.
LENGTHS = [1, 7, 16, 60, 130]
SIZES = [5, 9, 600, 70, 4]


@pytest.fixture(scope="module")
def loop_case():
    from cotracker_b200 import engine
    from cotracker_b200.synthetic import texture_video
    m = _model()
    first = np.concatenate([[0], np.cumsum(LENGTHS)]).tolist()
    video = torch.cat([texture_video(T, H, W, seed=200 + g, shift=(1 + g, 2)) for g, T in enumerate(LENGTHS)], 1)
    with torch.no_grad():
        pyr = m._encode(2.0 * (video[0].to(DEV).float() / 255.0) - 1.0, 200)
    H4, W4 = H // 4, W // 4
    gen = torch.Generator().manual_seed(5)
    groups = []
    for g, (T_g, n) in enumerate(zip(LENGTHS, SIZES)):
        qf = torch.randint(0, T_g, (n,), generator=gen)
        qc = torch.rand(n, 2, generator=gen) * torch.tensor([W4 - 1.0, H4 - 1.0])
        groups.append((qf, qc, first[g], T_g))
    return m, pyr, H4, W4, groups, engine


def _run(case, idx, slab=None):
    """One pass over the groups `idx`: padded to the longest with group_T (several), or alone (one)."""
    from cotracker_b200.model import ragged_frame_map
    m, pyr, H4, W4, groups, engine = case
    sel = [groups[i] for i in idx]
    T = max(T_g for *_, T_g in sel)
    qframes = torch.cat([qf + f0 for qf, _, f0, _ in sel]).to(torch.int32).to(DEV)
    qcoords = torch.cat([qc for _, qc, _, _ in sel]).float().to(DEV).contiguous()
    T_pyr = engine.pyramid_frames(pyr, H4, W4)
    support = engine.sample_support(pyr, T_pyr, H4, W4, qframes, qcoords)
    N = qcoords.shape[0]
    coords = qcoords[None].expand(T, N, 2).contiguous()
    vis = torch.zeros(T, N, device=DEV)
    conf = torch.zeros(T, N, device=DEV)
    sizes = [qf.shape[0] for qf, *_ in sel]
    lengths = [T_g for *_, T_g in sel] if len(sel) > 1 else None
    fmap = ragged_frame_map(T, [(f0, T_g, False) for _, _, f0, T_g in sel])
    if lengths is None:
        te = m.interpolate_time_embed(T).to(DEV)
    else:
        te = torch.zeros(len(sel), T, 1110, device=DEV)
        for g, t in enumerate(lengths):
            te[g, :t] = m.interpolate_time_embed(t).to(DEV)
    ws = torch.empty(engine.workspace_bytes(T, N, H4, W4, len(sel), T_pyr, slab, lengths), dtype=torch.uint8,
                     device=DEV)
    engine.update_loop(m.packed_weights(DEV), pyr, H4, W4, support, None, coords, vis, conf, te, 2, ws,
                       group_sizes=sizes, group_frames=fmap, slab_tracks=slab, group_T=lengths)
    out, a = [], 0
    for n, (*_, T_g) in zip(sizes, sel):
        out.append((coords[:T_g, a:a + n], vis[:T_g, a:a + n], conf[:T_g, a:a + n]))
        a += n
    return out


@pytest.mark.parametrize("opts,slab", [({}, None), ({"fuse": 0}, None), ({}, 50),
                                       ({"gemm": 1, "attn": 1, "corr": 1}, None)],
                         ids=["default", "fuse0", "slabs", "exact_fp32"])
def test_padded_pass_groups_equal_their_own_passes(loop_case, opts, slab):
    from cotracker_b200 import engine
    old = {k: engine.get_option(k) for k in opts}
    try:
        for k, v in opts.items():
            engine.set_option(k, v)
        with torch.no_grad():
            got = _run(loop_case, range(len(LENGTHS)), slab)
            for g in range(len(LENGTHS)):
                want = _run(loop_case, [g])[0]
                for k, (a, b) in enumerate(zip(got[g], want)):
                    assert a.shape == b.shape and torch.equal(a, b), (opts, g, LENGTHS[g], k)
    finally:
        for k, v in old.items():
            engine.set_option(k, v)


def test_padded_pass_without_the_long_group(loop_case):
    """T <= 128: every group takes the fused time attention with its own length."""
    with torch.no_grad():
        got = _run(loop_case, [0, 2, 3, 1])
        for i, g in enumerate([0, 2, 3, 1]):
            want = _run(loop_case, [g])[0]
            assert all(torch.equal(a, b) for a, b in zip(got[i], want)), g


# ---- predictor level ----------------------------------------------------------------------------------------------
def _predictor(seed=43):
    from cotracker_b200.predictor import CoTrackerPredictor
    from cotracker_b200.synthetic import seeded_state_dict
    p = CoTrackerPredictor(checkpoint=None, window_len=60)
    p.model.load_state_dict(seeded_state_dict(seed, offline=True, window_len=60, head_gain=10.0, vis_gain=100.0))
    return p.to(DEV)


def _clips():
    """Different lengths, frame sizes (the 120x216 apple frames among them), dtypes and devices."""
    from cotracker_b200.synthetic import texture_video
    apple = np.load("tests/golden/apple_frames_120x216.npz")["frames"][:21]
    return [torch.from_numpy(apple).permute(0, 3, 1, 2)[None].contiguous(),             # uint8, host, 21 frames
            texture_video(9, 96, 128, seed=7, shift=(2, 1)).float().to(DEV),            # float, device
            texture_video(33, 64, 80, seed=8, shift=(1, 3)),                            # uint8, host
            texture_video(4, 144, 192, seed=9, shift=(3, 2)).to(DEV).float()]            # float, device


def _queries(clips, counts, seed=300):
    from cotracker_b200.synthetic import random_queries
    return [random_queries(n, c.shape[1], c.shape[3], c.shape[4], seed=seed + b).to(DEV)
            for b, (c, n) in enumerate(zip(clips, counts))]


def _assert_list_equal(got, single):
    tracks, vis = got
    for b in range(len(tracks)):
        t1, v1 = single(b)
        assert tracks[b].shape == t1.shape and torch.equal(tracks[b], t1), b
        assert vis[b].shape == v1.shape and torch.equal(vis[b], v1), b


@pytest.mark.parametrize("budget", [None, 1], ids=["default_bound", "pass_per_clip"])
def test_list_call_queries_backward_equals_single_calls(budget):
    p = _predictor()
    p._list_budget_bytes = budget
    clips = _clips()
    qs = _queries(clips, [11, 3, 25, 6])
    got = p(clips, queries=qs, backward_tracking=True)
    _assert_list_equal(got, lambda b: p(clips[b], queries=qs[b], backward_tracking=True))


@pytest.mark.parametrize("budget", [None, 1], ids=["default_bound", "pass_per_clip"])
def test_list_call_grid_segm_mask_equals_single_calls(budget):
    p = _predictor(seed=47)
    p._list_budget_bytes = budget
    clips = _clips()
    mask = torch.zeros(1, 1, 120, 216)
    mask[..., 20:100, 40:180] = 1
    masks = [mask, None, None, None]
    got = p(clips, grid_size=5, grid_query_frame=2, segm_mask=masks, backward_tracking=True)
    _assert_list_equal(got, lambda b: p(clips[b], grid_size=5, grid_query_frame=2, segm_mask=masks[b],
                                        backward_tracking=True))


def test_list_call_in_one_pass_of_very_different_lengths(monkeypatch):
    """Clips of 4 to 33 frames padded into a single pass (padding bound lifted) still equal their single calls."""
    import cotracker_b200.predictor as P
    seen = []
    plan = P.plan_ragged_passes
    monkeypatch.setattr(P, "RAGGED_PAD_FRACTION", 1e9)
    monkeypatch.setattr(P, "plan_ragged_passes", lambda *a, **k: seen.append(plan(*a, **k)) or seen[-1])
    p = _predictor(seed=51)
    clips = _clips()
    qs = _queries(clips, [11, 3, 25, 6], seed=500)
    got = p(clips, queries=qs, backward_tracking=True)
    assert seen == [[[3, 1, 0, 2]]]
    _assert_list_equal(got, lambda b: p(clips[b], queries=qs[b], backward_tracking=True))


def test_list_call_mixed_queries_and_grid():
    p = _predictor(seed=49)
    clips = _clips()
    qs = _queries(clips, [4, 8, 2, 5], seed=400)
    qs[1] = None
    got = p(clips, queries=qs, grid_size=4)
    _assert_list_equal(got, lambda b: p(clips[b], queries=qs[b], grid_size=4))


# ---- goldens ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["predictor_grid", "c2_grid30", "pred_backward", "pred_segm_mask"])
def test_goldens_in_a_list_meet_their_bounds(name):
    from cases import CASES
    from cotracker_b200.predictor import CoTrackerPredictor
    from cotracker_b200.synthetic import random_queries, texture_video
    cfg = CASES[name]
    sd, video, queries = case_inputs(cfg)
    p = CoTrackerPredictor(checkpoint=None, window_len=cfg["window_len"])
    p.model.load_state_dict(sd)
    p = p.to(DEV)
    kw = predictor_kwargs(cfg, video, queries)
    T = video.shape[1]
    others = [texture_video(T + 5, 96, 128, seed=61), texture_video(max(1, T - 2), 64, 96, seed=62)]
    clips = [others[0], video, others[1]]
    args = {"grid_size": kw.get("grid_size", 0), "grid_query_frame": kw.get("grid_query_frame", 0),
            "backward_tracking": kw.get("backward_tracking", False)}
    if kw.get("queries") is not None:
        args["queries"] = [random_queries(5, c.shape[1], c.shape[3], c.shape[4], seed=70 + i).to(DEV)
                           if c is not video else kw["queries"].to(DEV) for i, c in enumerate(clips)]
    if kw.get("segm_mask") is not None:
        args["segm_mask"] = [None, kw["segm_mask"], None]
    tracks, vis = p(clips, **args)
    compare({"tracks": tracks[1].cpu(), "visibility": vis[1].cpu()}, load_golden(name))
