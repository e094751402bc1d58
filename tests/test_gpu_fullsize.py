"""GPU, BASELINE.json's full sizes (N=6400; T=16 and T=48; online grid 50): the CPU oracle would need minutes to hours
here, so parity is carried by size-independent properties of the path:
  * determinism           -- two runs of the same call are bit-identical (no atomics / racy reductions anywhere)
  * duplicated queries    -- the same query listed twice yields the same track (the virtual-token coupling is symmetric)
  * tensor-core vs SIMT   -- the production kernels (wgmma GEMMs, wgmma correlation, mma attention) against the
                             exact-fp32 SIMT verification kernels on the same inputs, within the 1e-3 px budget
  * query-frame identity  -- predictor output at the query frame is the query itself and visible (reference :173-185)
"""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _predictor(offline=True, window_len=60, seed=1234, head_gain=10.0, vis_gain=100.0):
    from cotracker_b200.predictor import CoTrackerOnlinePredictor, CoTrackerPredictor
    from cotracker_b200.synthetic import seeded_state_dict
    cls = CoTrackerPredictor if offline else CoTrackerOnlinePredictor
    p = cls(checkpoint=None, window_len=window_len)
    p.model.load_state_dict(seeded_state_dict(seed, offline=offline, window_len=window_len, head_gain=head_gain,
                                              vis_gain=vis_gain))
    return p.to(DEV)


def test_headline_shape_determinism_and_query_identity():
    from cotracker_b200.synthetic import texture_video
    p = _predictor()
    video = texture_video(16, 512, 512, seed=0).to(DEV)
    t1, v1 = p(video, grid_size=80)
    t2, v2 = p(video, grid_size=80)
    assert t1.shape == (1, 16, 6400, 2) and v1.shape == (1, 16, 6400) and v1.dtype == torch.bool
    assert torch.isfinite(t1).all()
    assert torch.equal(t1, t2) and torch.equal(v1, v2), "the path must be bit-deterministic"
    from cotracker_b200.predictor import get_points_on_a_grid
    q = get_points_on_a_grid(80, (384, 512), device=DEV)[0] * torch.tensor([511 / 511, 511 / 383], device=DEV)
    assert float((t1[0, 0] - q).abs().max()) < 1e-3 and bool(v1[0, 0].all())
    assert float((t1[0, -1] - t1[0, 0]).abs().max()) > 1.0, "amplified heads: tracks must move"


def test_headline_shape_duplicated_queries_agree():
    from cotracker_b200.synthetic import random_queries, texture_video
    p = _predictor()
    video = texture_video(16, 512, 512, seed=1).to(DEV)
    q = random_queries(3200, 16, 512, 512, seed=5).to(DEV)
    qq = torch.cat([q, q], dim=1)                       # 6400 tracks + the predictor's 36 support points
    tr, vi = p(video, queries=qq)
    assert tr.shape[2] == 6400
    d = float((tr[:, :, :3200] - tr[:, :, 3200:]).abs().max())
    assert d < 1e-4, d
    assert torch.equal(vi[:, :, :3200], vi[:, :, 3200:])


@pytest.mark.parametrize("T", [16, 48])
def test_loop_tensor_core_vs_simt_full_size(T):
    """N=6400 (T=48 = config 3): production kernels vs the SIMT fp32 verification kernels, 2 iterations."""
    from cotracker_b200 import engine as eng
    from cotracker_b200.synthetic import seeded_state_dict
    from cases import O
    sd = seeded_state_dict(7, offline=True, window_len=60, head_gain=10.0, vis_gain=100.0)
    N, H4, W4, iters = 6400, 96, 128, 2
    g = torch.Generator().manual_seed(3)
    fmaps = torch.randn(T, 128, H4, W4, generator=g).to(DEV)
    pyr = eng.prepare_pyramid(fmaps)
    del fmaps
    qf = torch.randint(0, T, (N,), generator=g).to(torch.int32).to(DEV)
    qc = (torch.rand(N, 2, generator=g) * torch.tensor([W4 - 1.0, H4 - 1.0])).to(DEV)
    support = eng.sample_support(pyr, T, H4, W4, qf, qc)
    packed = eng.pack_weights(sd, DEV)
    te = O.time_embedding(sd, T)[0].contiguous().to(DEV)
    ws = torch.empty(eng.workspace_bytes(T, N, H4, W4), dtype=torch.uint8, device=DEV)
    out = {}
    for mode in (0, 1):
        coords = qc[None].expand(T, N, 2).contiguous().clone()
        vis, conf = torch.zeros(T, N, device=DEV), torch.zeros(T, N, device=DEV)
        for opt in ("gemm", "corr", "attn"):
            eng.set_option(opt, mode)
        try:
            eng.update_loop(packed, pyr, H4, W4, support, None, coords, vis, conf, te, iters, ws)
            torch.cuda.synchronize()
        finally:
            for opt in ("gemm", "corr", "attn"):
                eng.set_option(opt, 0)
        out[mode] = (coords.cpu(), vis.cpu(), conf.cpu())
    assert torch.isfinite(out[0][0]).all()
    assert float((out[1][0] - qc.cpu()[None]).abs().max()) > 0.25, "case must move"
    e_c = float((out[0][0] - out[1][0]).abs().max()) * 4
    e_v = float((out[0][1] - out[1][1]).abs().max())
    e_q = float((out[0][2] - out[1][2]).abs().max())
    print(f"T={T}: tensor-core vs SIMT  d_tracks {e_c:.2e} px, d_vis {e_v:.2e}, d_conf {e_q:.2e}")
    assert e_c < 1e-3 and e_v < 1e-3 and e_q < 1e-3


def test_online_stream_config4_shape():
    """cotracker3_online, 512x512 stream, window 16 / step 8, grid 50 (N=2500): runs, deterministic, consistent growth."""
    from cotracker_b200.synthetic import texture_video
    video = texture_video(40, 512, 512, seed=2).to(DEV)
    outs = []
    for rep in range(2):
        p = _predictor(offline=False, window_len=16, seed=77, head_gain=5.0, vis_gain=30.0)
        p(video_chunk=video, is_first_step=True, grid_size=50)
        res = []
        for ind in range(0, video.shape[1] - p.step, p.step):
            tr, vi = p(video_chunk=video[:, ind:ind + p.step * 2])
            res.append((tr.clone(), vi.clone()))
        outs.append(res)
    assert [r[0].shape[1] for r in outs[0]] == [16, 24, 32, 40]
    assert outs[0][-1][0].shape == (1, 40, 2500, 2)
    for (a, av), (b, bv) in zip(outs[0], outs[1]):
        assert torch.equal(a, b) and torch.equal(av, bv)
    # frames finalised by an earlier window (older than the current window) never change afterwards
    assert torch.equal(outs[0][1][0][:, :8], outs[0][2][0][:, :8])
