"""Frame maps on the GPU (ct3_loop_shape.group_frames, forward_groups(reversed_groups=), the predictors' grouped
backward tracking and dense passes).  Every group must be bit-identical to a standalone call on a pyramid holding
exactly the frames its map names, and the predictors bit-identical to their previous one-pass-at-a-time sequence."""
import numpy as np
import pytest
import torch

from cases import O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SIZES = [90, 1, 129, 300, 64]


@pytest.fixture(scope="module")
def eng():
    from cotracker_b200 import engine
    engine.lib()
    return engine


@pytest.fixture(scope="module")
def sd():
    from cotracker_b200.synthetic import seeded_state_dict
    return seeded_state_dict(81, offline=True, window_len=60, head_gain=10.0, vis_gain=100.0)


def _bounds(sizes):
    b = np.concatenate([[0], np.cumsum(sizes)]).tolist()
    return list(zip(b[:-1], b[1:]))


def _maps(T, T_pyr, G, seed):
    """Group g's frame row: identity, reversed (T-1-t), random with repeats over all T_pyr frames, in turn."""
    g = torch.Generator().manual_seed(seed)
    rows = []
    for k in range(G):
        if k % 3 == 0:
            rows.append(list(range(T)))
        elif k % 3 == 1:
            rows.append(list(range(T - 1, -1, -1)))
        else:
            rows.append(torch.randint(0, T_pyr, (T,), generator=g).tolist())
    return rows


def _loop(eng, packed, pyr, H4, W4, support, valid, c0, te, iters, sizes=None, frames=None):
    T, N, _ = c0.shape
    coords, vis, conf = c0.clone(), torch.zeros(T, N, device=DEV), torch.zeros(T, N, device=DEV)
    G = 1 if sizes is None else len(sizes)
    T_pyr = None if frames is None else eng.pyramid_frames(pyr, H4, W4)
    ws = torch.empty(eng.workspace_bytes(T, N, H4, W4, groups=G, frames=T_pyr), dtype=torch.uint8, device=DEV)
    eng.update_loop(packed, pyr, H4, W4, support, valid, coords, vis, conf, te, iters, ws, group_sizes=sizes,
                    group_frames=frames)
    return coords, vis, conf


def _frames_case(eng, sd, T, H4, W4, seed):
    """A pyramid of T + 3 frames, frame maps of every kind, support sampled at each track's mapped query frame."""
    g = torch.Generator().manual_seed(seed)
    T_pyr, N = T + 3, sum(SIZES)
    fmaps = torch.randn(T_pyr, 128, H4, W4, generator=g).to(DEV)
    maps = _maps(T, T_pyr, len(SIZES), seed)
    qf = torch.randint(0, T, (N,), generator=g)
    qc = torch.stack([torch.rand(N, generator=g) * (W4 - 1), torch.rand(N, generator=g) * (H4 - 1)], dim=1).to(DEV)
    valid = (torch.rand(N, generator=g) < 0.9).to(torch.uint8).to(DEV)
    rowof = torch.tensor(maps)[torch.repeat_interleave(torch.arange(len(SIZES)), torch.tensor(SIZES))]   # [N, T]
    mapped = rowof.gather(1, qf[:, None])[:, 0]
    pyr = eng.prepare_pyramid(fmaps)
    support = eng.sample_support(pyr, T_pyr, H4, W4, mapped.to(torch.int32).to(DEV).contiguous(), qc)
    c0 = qc[None].expand(T, -1, 2).contiguous()
    te = O.time_embedding(sd, T)[0].contiguous().to(DEV)
    return fmaps, maps, qf, qc, valid, pyr, support, c0, te


# (64, 72): every level >= 8x8, corr_tc3.cu;  (24, 32): level 3 is 3x4, corr_tc.cu
@pytest.mark.parametrize("hw", [(64, 72), (24, 32)])
@pytest.mark.parametrize("T", [12, 150])
def test_update_loop_frames_bit_identical_to_standalone(eng, sd, T, hw):
    H4, W4 = hw
    iters = 2
    fmaps, maps, qf, qc, valid, pyr, support, c0, te = _frames_case(eng, sd, T, H4, W4, seed=T + H4)
    packed = eng.pack_weights(sd, DEV)
    got = _loop(eng, packed, pyr, H4, W4, support, valid, c0, te, iters, SIZES, maps)
    assert float((got[0] - c0).abs().max()) > 0.25, "case must move"
    for k, (a, b) in enumerate(_bounds(SIZES)):
        # the standalone problem: a pyramid of exactly the group's frames, in order
        pyr_g = eng.prepare_pyramid(fmaps[maps[k]].contiguous())
        sup_g = eng.sample_support(pyr_g, T, H4, W4, qf[a:b].to(torch.int32).to(DEV).contiguous(),
                                   qc[a:b].contiguous())
        assert torch.equal(sup_g, support[:, :, a:b])
        want = _loop(eng, packed, pyr_g, H4, W4, sup_g, valid[a:b].contiguous(), c0[:, a:b].contiguous(), te, iters)
        for x, y in zip(got, want):
            assert torch.equal(x[:, a:b], y), (T, hw, k, float((x[:, a:b] - y).abs().max()))


def test_identity_map_is_the_grouped_call(eng, sd):
    T, H4, W4 = 12, 64, 72
    fmaps, _, qf, qc, valid, _, _, c0, te = _frames_case(eng, sd, T, H4, W4, seed=3)
    pyr = eng.prepare_pyramid(fmaps[:T].contiguous())
    support = eng.sample_support(pyr, T, H4, W4, qf.to(torch.int32).to(DEV).contiguous(), qc)
    packed = eng.pack_weights(sd, DEV)
    ident = [list(range(T))] * len(SIZES)
    got = _loop(eng, packed, pyr, H4, W4, support, valid, c0, te, 2, SIZES, ident)
    want = _loop(eng, packed, pyr, H4, W4, support, valid, c0, te, 2, SIZES)
    for x, y in zip(got, want):
        assert torch.equal(x, y)


# with the sample-then-correlate kernel (corr_tc.cu) and the split-bf16 correlate-then-interpolate kernel (corr_tc2.cu)
@pytest.mark.parametrize("opts", [{"corr": 2}, {"prec.corr": 3}], ids=["corr2", "prec.corr3"])
def test_frames_on_other_tensor_core_kernels(eng, sd, opts):
    T, H4, W4 = 12, 64, 72
    fmaps, maps, qf, qc, valid, pyr, support, c0, te = _frames_case(eng, sd, T, H4, W4, seed=11)
    packed = eng.pack_weights(sd, DEV)
    before = {k: eng.get_option(k) for k in opts}
    for k, v in opts.items():
        eng.set_option(k, v)
    try:
        got = _loop(eng, packed, pyr, H4, W4, support, valid, c0, te, 2, SIZES, maps)
        for k, (a, b) in enumerate(_bounds(SIZES)):
            pyr_g = eng.prepare_pyramid(fmaps[maps[k]].contiguous())
            want = _loop(eng, packed, pyr_g, H4, W4, support[:, :, a:b].contiguous(), valid[a:b].contiguous(),
                         c0[:, a:b].contiguous(), te, 2)
            for x, y in zip(got, want):
                assert torch.equal(x[:, a:b], y), (opts, k)
    finally:
        for k, v in before.items():
            eng.set_option(k, v)


def test_frames_simt_cross_check(eng, sd):
    """corr = 1 (exact-fp32 SIMT correlation, with the SIMT GEMM and attention) against the tensor-core run, and the
    SIMT run's groups bit-identical to standalone SIMT calls."""
    T, H4, W4 = 12, 64, 72
    fmaps, maps, qf, qc, valid, pyr, support, c0, te = _frames_case(eng, sd, T, H4, W4, seed=9)
    packed = eng.pack_weights(sd, DEV)
    tc = _loop(eng, packed, pyr, H4, W4, support, valid, c0, te, 2, SIZES, maps)
    for k in ("gemm", "corr", "attn"):
        eng.set_option(k, 1)
    try:
        simt = _loop(eng, packed, pyr, H4, W4, support, valid, c0, te, 2, SIZES, maps)
        for k, (a, b) in enumerate(_bounds(SIZES)):
            if k % 3 == 0:
                continue
            pyr_g = eng.prepare_pyramid(fmaps[maps[k]].contiguous())
            want = _loop(eng, packed, pyr_g, H4, W4, support[:, :, a:b].contiguous(), valid[a:b].contiguous(),
                         c0[:, a:b].contiguous(), te, 2)
            for x, y in zip(simt, want):
                assert torch.equal(x[:, a:b], y), k
        torch.cuda.synchronize()
    finally:
        for k in ("gemm", "corr", "attn"):
            eng.set_option(k, 0)
    e_c = float((tc[0] - simt[0]).abs().max()) * 4
    e_v = float((tc[1] - simt[1]).abs().max())
    e_q = float((tc[2] - simt[2]).abs().max())
    assert e_c < 1e-3 and e_v < 1e-3 and e_q < 1e-3, (e_c, e_v, e_q)


# ---- models -----------------------------------------------------------------------------------------------------
def _group_queries(sizes, T, H, W, seed):
    from cotracker_b200.synthetic import random_queries
    return torch.cat([random_queries(n, T, H, W, seed=seed + k) for k, n in enumerate(sizes)], dim=1)


@pytest.mark.parametrize("online,T", [(False, 12), (True, 16), (True, 37)])
def test_forward_groups_reversed_equals_forward_on_flipped_clip(online, T):
    """A reversed group equals `forward` on video.flip(1); the sliding-window model with T not a multiple of S pads the
    reversed clip with copies of the original frame 0 and gathers each window's frames from the forward pyramid."""
    from cotracker_b200.build import build_cotracker
    from cotracker_b200.synthetic import seeded_state_dict, texture_video
    S = 16 if online else 60
    sizes, flags = [90, 1, 129, 64], [False, True, True, False]
    state = seeded_state_dict(82, offline=not online, window_len=S, head_gain=5.0, vis_gain=30.0)
    model = build_cotracker(None, offline=not online, window_len=S).eval()
    model.load_state_dict(state)
    model = model.to(DEV)
    H, W = 256, 288
    video = texture_video(T, H, W, seed=T).to(DEV)
    queries = _group_queries(sizes, T, H, W, seed=T).to(DEV)
    with torch.no_grad():
        got = model.forward_groups(video, queries, sizes, iters=2, reversed_groups=flags)
        flipped = video.flip(1).contiguous()
        for (a, b), r in zip(_bounds(sizes), flags):
            want = model(flipped if r else video, queries[:, a:b], iters=2)
            for x, y in zip(got[:3], want[:3]):
                assert torch.equal(x[:, :, a:b], y), (online, T, a, r, float((x[:, :, a:b] - y).abs().max()))


# ---- predictors -------------------------------------------------------------------------------------------------
def _predictor(offline, seed=91):
    from cotracker_b200.predictor import CoTrackerPredictor
    from cotracker_b200.synthetic import seeded_state_dict
    S = 60 if offline else 16
    p = CoTrackerPredictor(checkpoint=None, offline=offline, window_len=S)
    p.model.load_state_dict(seeded_state_dict(seed, offline=offline, window_len=S, head_gain=10.0, vis_gain=100.0))
    return p.to(DEV)


def _sequential(p, clip, video_shape, queries=None, grid_size=0, grid_query_frame=0, backward_tracking=False,
                add_support_grid=False):
    """The previous sparse path: one model pass for the forward queries and, for backward tracking, a second one on
    the pyramid reversed in place (and restored afterwards)."""
    T = clip.T
    q = p._model_queries(clip, video_shape, queries, None, grid_size, add_support_grid, grid_query_frame)
    m = p.model
    fwd = m._track_pyramid(clip.pyr, T, clip.H, clip.W, q, clip.ITERS, [q.shape[1]])[:2]
    bwd = None
    if backward_tracking:
        inv = q.clone()
        inv[:, :, 0] = T - inv[:, :, 0] - 1
        m._reverse_clip_pyramid_(clip.pyr, T, clip.H, clip.W)
        bwd = m._track_pyramid(clip.pyr, T, clip.H, clip.W, inv, clip.ITERS, [q.shape[1]])[:2]
        m._reverse_clip_pyramid_(clip.pyr, T, clip.H, clip.W)
    return p._finish(q, fwd, bwd, video_shape, add_support_grid)


@pytest.mark.parametrize("one_pass", [True, False])
@pytest.mark.parametrize("offline", [True, False])
def test_backward_tracking_equals_sequential_passes(offline, one_pass, monkeypatch):
    """Both directions as groups of one pass, and (above BACKWARD_GROUP_TRACK_FRAMES) as two passes."""
    import cotracker_b200.predictor as P
    from cotracker_b200.predictor import _EncodedClip
    from cotracker_b200.synthetic import random_queries, texture_video
    if not one_pass:
        monkeypatch.setattr(P, "BACKWARD_GROUP_TRACK_FRAMES", 0)
    p = _predictor(offline)
    T, H, W = 21, 144, 192
    video = texture_video(T, H, W, seed=5).to(DEV)
    queries = random_queries(13, T, H, W, seed=6).to(DEV)
    with torch.no_grad():
        clip = _EncodedClip(p.model, video, p.interp_shape)
        for kw, call in [(dict(queries=queries, add_support_grid=True), dict(queries=queries)),
                         (dict(grid_size=7), dict(grid_size=7)),
                         (dict(grid_size=7, grid_query_frame=T - 3), dict(grid_size=7, grid_query_frame=T - 3))]:
            got = p(video, backward_tracking=True, **call)
            want = _sequential(p, clip, video.shape, backward_tracking=True, **kw)
            assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]), (offline, kw)


def _dense_sequential(p, video, grid_query_frame, backward):
    from cotracker_b200.predictor import _EncodedClip
    H, W = video.shape[3:]
    step = W // 80
    gw, gh = W // step, H // step
    clip = _EncodedClip(p.model, video, p.interp_shape)
    base_x = (torch.arange(gw, device=DEV).repeat(gh) * step).float()
    base_y = (torch.arange(gh, device=DEV).repeat_interleave(gw) * step).float()
    parts = []
    for offset in range(step * step):
        pts = torch.zeros(1, gw * gh, 3, device=DEV)
        pts[:, :, 0] = grid_query_frame
        pts[:, :, 1] = base_x + offset % step
        pts[:, :, 2] = base_y + offset // step
        parts.append(_sequential(p, clip, video.shape, queries=pts, backward_tracking=backward))
    return torch.cat([t for t, _ in parts], dim=2), torch.cat([v for _, v in parts], dim=2)


@pytest.mark.parametrize("offline", [True, False])
@pytest.mark.parametrize("backward", [False, True])
def test_dense_equals_sequential_passes(offline, backward, monkeypatch, capsys):
    """Dense mode in grouped passes equals the per-offset passes, whatever the budget: one pass for every group, or
    a budget so small that every group is a pass of its own."""
    import cotracker_b200.predictor as P
    from cotracker_b200.synthetic import texture_video
    p = _predictor(offline, seed=93)
    T, H, W = 8, 96, 160          # grid step 2: 4 offsets of 48 x 80 tracks
    video = texture_video(T, H, W, seed=7).to(DEV)
    gq = T - 1 if backward else 0
    with torch.no_grad():
        want = _dense_sequential(p, video, gq, backward)
        capsys.readouterr()
        got = p(video, grid_query_frame=gq, backward_tracking=backward)
        lines = capsys.readouterr().out.split("\n")
        monkeypatch.setattr(P, "pass_budget_bytes", lambda *a, **k: 1)
        tiny = p(video, grid_query_frame=gq, backward_tracking=backward)
    assert [ln for ln in lines if ln.startswith("step")] == [f"step {i} / 4" for i in range(4)]
    for out in (got, tiny):
        assert torch.equal(out[0], want[0]) and torch.equal(out[1], want[1]), (offline, backward)


# ---- memory -----------------------------------------------------------------------------------------------------
def test_grouped_backward_tracking_peak_memory():
    """One grouped pass holds the update-loop workspace of both directions; nothing else grows."""
    from cotracker_b200 import engine
    from cotracker_b200.synthetic import texture_video
    p = _predictor(True, seed=95)
    T, H, W, grid = 48, 480, 640, 30
    video = texture_video(T, H, W, seed=8).to(DEV)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    with torch.no_grad():
        tracks, vis = p(video, grid_size=grid, backward_tracking=True)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    assert tracks.shape == (1, T, grid * grid, 2)
    ih, iw = p.interp_shape
    N = 2 * grid * grid                    # forward and reversed groups
    frames = T * 3 * ih * iw * 4
    pyramid = engine.pyramid_layout(T, ih // 4, iw // 4)[3] * 4
    bound = (frames + pyramid + engine.encoder_workspace_bytes(T, ih, iw)
             + engine.workspace_bytes(T, N, ih // 4, iw // 4, groups=2, frames=T) + N * 4 * 49 * 128 * 4
             + engine.packed_weights_bytes() + (64 << 20)                     # packed weights (both nets) < 64 MiB
             + N * T * 16 * 4 + (64 << 20))                                   # state, outputs, small temporaries
    print(f"peak {peak / 2**20:.0f} MiB, bound {bound / 2**20:.0f} MiB")
    assert peak <= bound
