"""GPU stage-level parity: every CUDA kernel against the CPU oracle (called through the C ABI).
Amplified inputs/weights are used where end-to-end parity is blind (SURVEY.md Appendix A)."""
import math

import pytest
import torch

from cases import O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def eng():
    from cotracker_b200 import engine
    engine.lib()
    engine.set_option("gemm", 0)
    return engine


def _rel_err(got, want):
    return float((got.double().cpu() - want.double().cpu()).abs().max() / (want.double().abs().max() + 1e-30))


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("M,K,N", [(128, 64, 128), (300, 384, 384), (1000, 2401, 384), (257, 1110, 384),
                                   (640, 1536, 384), (4100, 384, 1536), (129, 384, 256), (64, 384, 1152),
                                   (38000, 384, 384), (40100, 1110, 256)])   # many tiles per persistent CTA, odd tile count
def test_linear_matches_fp64(eng, impl, M, K, N):
    g = torch.Generator().manual_seed(M * 7 + K)
    x = torch.randn(M, K, generator=g)
    w = torch.randn(N, K, generator=g) / math.sqrt(K)
    b = torch.randn(N, generator=g)
    want = x.double() @ w.double().t() + b.double()
    eng.set_option("gemm", impl)
    try:
        got = eng.linear(x.to(DEV), w.to(DEV), b.to(DEV), act=0)
        torch.cuda.synchronize()
    finally:
        eng.set_option("gemm", 0)
    # split-bf16x3: ~2^-17 per product; fp32 accumulate.  fp32 SIMT: ~1e-6.
    assert _rel_err(got, want) < 2e-5, (impl, M, K, N, _rel_err(got, want))


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("products,fp16,tol", [(3, 1, 1e-5), (2, 1, 6e-4), (1, 1, 1.2e-3), (2, 0, 8e-3), (1, 0, 1.6e-2)])
@pytest.mark.parametrize("M,K,N", [(300, 384, 384), (1000, 2401, 384), (40100, 2401, 384)])
def test_linear_precision_variants(eng, impl, products, fp16, tol, M, K, N):
    """The GEMM engine's precision switches against fp64: fp16 planes x3 ~2^-22, x2 = activation rounded to fp16
    (2^-12, weights exact), x1 = both rounded; bf16 planes: 2^-9.  Bounds are a few times the rounding of ONE operand
    element relative to the output scale (errors average over K).  Also checks tensor-core == SIMT restatement."""
    g = torch.Generator().manual_seed(M + K + products)
    x = torch.rand(M, K, generator=g) * 2 - 1                      # correlations live in [-1, 1]
    w = torch.randn(N, K, generator=g) / math.sqrt(K)
    b = torch.randn(N, generator=g)
    want = x.double() @ w.double().t() + b.double()
    eng.set_option("gemm", impl)
    try:
        got = eng.linear(x.to(DEV), w.to(DEV), b.to(DEV), act=0, products=products, fp16=bool(fp16))
        torch.cuda.synchronize()
    finally:
        eng.set_option("gemm", 0)
    err = _rel_err(got, want)
    assert err < tol, (impl, products, fp16, M, K, N, err)
    if products < 3:
        assert err > tol / 200, "suspiciously exact: is the lo plane still being multiplied?"


@pytest.mark.parametrize("act,approx", [(1, "none"), (2, "tanh")])
def test_linear_gelu_epilogues(eng, act, approx):
    g = torch.Generator().manual_seed(act)
    x = torch.randn(513, 384, generator=g) * 3
    w = torch.randn(384, 384, generator=g) / 10
    b = torch.randn(384, generator=g)
    want = torch.nn.functional.gelu((x.double() @ w.double().t() + b.double()), approximate=approx)
    got = eng.linear(x.to(DEV), w.to(DEV), b.to(DEV), act=act)
    assert _rel_err(got, want) < 2e-5


def _pyramid_case(T=3, H4=24, W4=32, seed=0):
    g = torch.Generator().manual_seed(seed)
    fmaps = torch.randn(T, 128, H4, W4, generator=g) * 2.5
    fmaps[0, :, 0, 0] = 0.0  # zero vector -> the 1e-12 clamp path
    return fmaps


def test_prepare_pyramid(eng):
    T, H4, W4 = 3, 25, 33  # odd sizes: avg-pool floors
    fmaps = _pyramid_case(T, H4, W4)
    want = O.normalized_pyramid(fmaps)
    pyr = eng.prepare_pyramid(fmaps.to(DEV))
    levels = eng.pyramid_levels(pyr, T, H4, W4)
    for l in range(4):
        got = levels[l].permute(0, 3, 1, 2).cpu()
        assert got.shape == want[l].shape
        assert float((got - want[l]).abs().max()) < 1e-6, l


def _coords_case(T, N, H4, W4, seed):
    g = torch.Generator().manual_seed(seed)
    c = torch.rand(T, N, 2, generator=g) * torch.tensor([W4 - 1.0, H4 - 1.0])
    c[:, 0] = torch.tensor([-7.3, -2.0])                 # far outside: everything clamps
    c[:, 1] = torch.tensor([W4 + 5.5, H4 + 9.25])
    c[:, 2] = torch.tensor([0.0, 0.0])
    c[:, 3] = torch.tensor([W4 - 1.0, H4 - 1.0])         # exactly on the last texel
    c[:, 4] = torch.tensor([2.5, H4 - 1.75])
    return c


def test_sample_support(eng):
    T, H4, W4, N = 4, 24, 32, 40
    fmaps = _pyramid_case(T, H4, W4, seed=1)
    want_pyr = O.normalized_pyramid(fmaps)
    pyr = eng.prepare_pyramid(fmaps.to(DEV))
    g = torch.Generator().manual_seed(3)
    qf = torch.randint(0, T, (N,), generator=g)
    qc = _coords_case(1, N, H4, W4, 5)[0]
    got = eng.sample_support(pyr, T, H4, W4, qf.to(torch.int32).to(DEV), qc.to(DEV)).cpu()
    for l in range(4):
        want = O.support_features(want_pyr[l], qf, qc / 2 ** l)
        assert float((got[l] - want).abs().max()) < 2e-5, l
    # online accumulation: masked add
    acc = torch.ones(4, 49, N, 128, device=DEV)
    mask = (torch.arange(N) % 3 == 0).to(torch.uint8)
    eng.sample_support(pyr, T, H4, W4, qf.to(torch.int32).to(DEV), qc.to(DEV), support=acc, accumulate_mask=mask.to(DEV))
    acc = acc.cpu()
    sel = mask.bool()
    assert float((acc[:, :, sel] - 1 - got[:, :, sel]).abs().max()) < 1e-6
    assert bool((acc[:, :, ~sel] == 1).all())


# impl 0: tensor-core product path (correlate-then-interpolate kernel when every level is >= 8x8, i.e. the
# 64x64 / 64x72 / 96x128 cases; sample-then-correlate otherwise), 1: exact-fp32 SIMT cross-check,
# 2: sample-then-correlate tensor-core kernel forced
@pytest.mark.parametrize("impl", [0, 1, 2])
@pytest.mark.parametrize("T,N,H4,W4", [(3, 16, 24, 32), (2, 9, 8, 8), (5, 33, 96, 128), (1, 5, 16, 24), (16, 300, 96, 128),
                                       (2, 40, 64, 64), (3, 150, 64, 72)])
def test_corr_sample(eng, impl, T, N, H4, W4):
    fmaps = _pyramid_case(T, H4, W4, seed=2)
    want_pyr = O.normalized_pyramid(fmaps)
    pyr = eng.prepare_pyramid(fmaps.to(DEV))
    g = torch.Generator().manual_seed(11)
    support = torch.randn(4, 49, N, 128, generator=g)
    support = support / support.norm(dim=-1, keepdim=True)
    coords = _coords_case(T, N, H4, W4, 13)
    valid = torch.ones(N, dtype=torch.uint8)
    dead = min(5, N - 1)
    valid[dead] = 0
    eng.set_option("corr", impl)
    try:
        got = eng.corr_sample(pyr, H4, W4, support.to(DEV), valid.to(DEV), coords.to(DEV)).cpu()   # [N,T,4,2401]
    finally:
        eng.set_option("corr", 0)
    for l in range(4):
        want = O.correlation_volume(want_pyr[l], support[l] * valid[None, :, None].float(), coords / 2 ** l)  # [T,N,2401]
        err = float((got[:, :, l].permute(1, 0, 2) - want).abs().max())
        # |corr| <= 1; grid_sample normalise/denormalise noise ~1e-5, bf16x3 ~1e-5; the default precision of the
        # correlate-then-interpolate kernels (prec.corr = 2) rounds the texels to fp16: + ~3e-5
        assert err < (1.2e-4 if impl == 0 else 5e-5), (impl, l, err)
    assert bool((got[dead] == 0).all())


# precision switches of the correlate-then-interpolate kernels: products of the contraction x volume format
# (prec.corr 3 on corr_tc2.cu, 1 and 2 on corr_tc3.cu).
# tolerances: texels rounded to fp16 -> ~2^-12 * sqrt(128) * |f||s| / 128 ~ 3e-5 on top of the 5e-5 above;
# a single fp16 volume plane rounds |v| <= 1 to 2^-12 relative -> 2.5e-4.
@pytest.mark.parametrize("corr,fc1,tol", [(3, 3, 1.2e-4), (2, 3, 1.2e-4), (1, 3, 1.5e-4), (3, 2, 3.2e-4), (2, 2, 3.6e-4),
                                          (1, 1, 4e-4)])
@pytest.mark.parametrize("T,N,H4,W4", [(2, 9, 8, 8), (5, 33, 96, 128), (16, 300, 96, 128), (3, 150, 64, 72)])
def test_corr_sample_precision_modes(eng, corr, fc1, tol, T, N, H4, W4):
    fmaps = _pyramid_case(T, H4, W4, seed=2)
    want_pyr = O.normalized_pyramid(fmaps)
    pyr = eng.prepare_pyramid(fmaps.to(DEV))
    g = torch.Generator().manual_seed(11)
    support = torch.randn(4, 49, N, 128, generator=g)
    support = support / support.norm(dim=-1, keepdim=True)
    coords = _coords_case(T, N, H4, W4, 13)
    valid = torch.ones(N, dtype=torch.uint8)
    valid[min(5, N - 1)] = 0
    c0, f0 = eng.get_option("prec.corr"), eng.get_option("prec.fc1")
    eng.set_option("prec.corr", corr)
    eng.set_option("prec.fc1", fc1)
    try:
        patch = min(H4, W4) // 8 >= 8    # coarsest level >= 8x8 texels: the correlate-then-interpolate kernel runs;
        # otherwise the sample-then-correlate kernel computes split x split whatever the switches say
        assert eng.precision_info(T, H4, W4) == ((corr, fc1, 4 if fc1 == 3 else 2) if patch else (3, 3, 4))
        got = eng.corr_sample(pyr, H4, W4, support.to(DEV), valid.to(DEV), coords.to(DEV)).cpu()
    finally:
        eng.set_option("prec.corr", c0)
        eng.set_option("prec.fc1", f0)
    worst = 0.0
    for l in range(4):
        want = O.correlation_volume(want_pyr[l], support[l] * valid[None, :, None].float(), coords / 2 ** l)
        worst = max(worst, float((got[:, :, l].permute(1, 0, 2) - want).abs().max()))
    assert worst < tol, (corr, fc1, worst)
    assert bool((got[min(5, N - 1)] == 0).all())


def _amplified_sd(seed=1234, **kw):
    from cotracker_b200.synthetic import seeded_state_dict
    return seeded_state_dict(seed, offline=True, window_len=60, **kw)


def _with_norm_context(sd, seed=8, token_scale=3e-3):
    """sd with a trained-like affine norm_context in every cross block (gamma ~ 1 + 0.7 N(0, 1), some negative; beta ~
    0.5 N(0, 1); a fresh module has 1 and 0) and the point tokens scaled down by token_scale (input_transform and every
    time block's to_out and fc2), so that the tokens the first virtual<-point block normalises have a variance of about
    1e-6, below norm_context's eps of 1e-5: eps then decides that LayerNorm."""
    g = torch.Generator().manual_seed(seed)
    sd = dict(sd)
    for k in [k for k in sd if k.endswith("norm_context.weight")]:
        sd[k] = 1 + 0.7 * torch.randn(sd[k].shape, generator=g)
        sd[k[:-len("weight")] + "bias"] = 0.5 * torch.randn(sd[k].shape, generator=g)
    for k in [k for k in sd if k.startswith("updateformer.input_transform.") or
              (k.startswith("updateformer.time_blocks.") and (".attn.to_out." in k or ".mlp.fc2." in k))]:
        sd[k] = sd[k] * token_scale
    return sd


@pytest.mark.parametrize("impl", [0, 1])
def test_updateformer_stage(eng, impl):
    """Also with non-trivial norm_context weights (every seeded state dict has gamma = 1, beta = 0 there) on tokens
    whose variance is below its eps: the affine and the eps must each move the oracle's output far beyond the tolerance,
    so that the case cannot pass without them."""
    sd0 = _amplified_sd(head_gain=100.0, vis_gain=100.0)
    g = torch.Generator().manual_seed(21)
    N, T = 70, 6
    x = torch.randn(N, T, 1110, generator=g)
    sd_nc = _with_norm_context(sd0)
    for sd in (sd0, sd_nc):
        with torch.no_grad():
            want = O.updateformer(sd, x[None])[0]
        packed = eng.pack_weights(sd, DEV)
        eng.set_option("gemm", impl)
        try:
            got = eng.updateformer(packed, x.to(DEV)).cpu()
        finally:
            eng.set_option("gemm", 0)
        scale = float(want.abs().max())
        err = float((got - want).abs().max())
        assert err < 2e-4 * max(scale, 1.0), (sd is sd_nc, err, scale)
    # the same tokens with norm_context back at gamma = 1, beta = 0, and with eps 1e-6 in place of its 1e-5
    plain = {k: (torch.ones_like(v) if k.endswith("norm_context.weight") else
                 torch.zeros_like(v) if k.endswith("norm_context.bias") else v) for k, v in sd_nc.items()}
    ln = O.ln
    with torch.no_grad():
        moved_affine = float((O.updateformer(plain, x[None])[0] - want).abs().max())
        O.ln = lambda xx, eps, w=None, b=None: ln(xx, 1e-6 if eps == 1e-5 else eps, w, b)
        try:
            moved_eps = float((O.updateformer(sd_nc, x[None])[0] - want).abs().max())
        finally:
            O.ln = ln
    tol = 2e-4 * max(scale, 1.0)
    assert moved_affine > 100 * tol and moved_eps > 100 * tol, (moved_affine, moved_eps, tol)


# 0: product kernels (fused wgmma time attention, wgmma + TMA point<-virtual attention for more than 64 points,
#    mma.sync kernels for the other space patterns), 1: exact-fp32 SIMT cross-check
@pytest.mark.parametrize("attn", [0, 1])
@pytest.mark.parametrize("N,T", [(70, 6), (600, 20), (130, 40), (1030, 16), (129, 5), (3, 2)])
def test_updateformer_attention_shapes(eng, attn, N, T):
    """Exercises every attention variant: per-warp time attention with KB=16/32/64, shared K/V, split-K + combine
    (N >= 512 keys), ragged query/key tails."""
    sd = _amplified_sd(seed=3, head_gain=100.0, vis_gain=100.0)
    g = torch.Generator().manual_seed(N + T)
    x = torch.randn(N, T, 1110, generator=g)
    with torch.no_grad():
        want = O.updateformer(sd, x[None])[0]
    packed = eng.pack_weights(sd, DEV)
    eng.set_option("attn", attn)
    try:
        got = eng.updateformer(packed, x.to(DEV)).cpu()
    finally:
        eng.set_option("attn", 0)
    scale = float(want.abs().max())
    err = float((got - want).abs().max())
    assert err < 2e-4 * max(scale, 1.0), (attn, N, T, err, scale)


@pytest.mark.parametrize("N,T", [(70, 6), (333, 16), (130, 40), (50, 48), (21, 100), (9, 128), (5, 129)])
def test_fused_time_attention(eng, N, T):
    """gemm_qkv_time_attn_kernel (projection + per-track attention in one kernel; tile = floor(128/T) whole tracks,
    ragged last tile, T = 128 -> one track per tile; T = 129 falls back to the separate kernels) against the oracle
    and against the unfused path (`fuse` = 0)."""
    sd = _amplified_sd(seed=5, head_gain=100.0, vis_gain=100.0)
    g = torch.Generator().manual_seed(N * 131 + T)
    x = torch.randn(N, T, 1110, generator=g)
    with torch.no_grad():
        want = O.updateformer(sd, x[None])[0]
    packed = eng.pack_weights(sd, DEV)
    got = {}
    for fuse in (1, 0):     # 1: fused time attention (default), 0: separate projection and attention kernels
        eng.set_option("fuse", fuse)
        try:
            got[fuse] = eng.updateformer(packed, x.to(DEV)).cpu()
        finally:
            eng.set_option("fuse", 1)
    scale = max(float(want.abs().max()), 1.0)
    assert float((got[1] - want).abs().max()) < 2e-4 * scale, (N, T, float((got[1] - want).abs().max()), scale)
    assert float((got[1] - got[0]).abs().max()) < 1e-4 * scale


def test_corr_mlp_gelu_variant_is_erf(eng):
    """Mutation guard (SURVEY Appendix A): with volume x10 the erf and tanh GELUs differ by >1e-3."""
    sd = _amplified_sd()
    g = torch.Generator().manual_seed(5)
    vol = (torch.rand(256, 2401, generator=g) * 2 - 1) * 10
    with torch.no_grad():
        h_erf = torch.nn.functional.gelu(torch.nn.functional.linear(vol, sd["corr_mlp.fc1.weight"], sd["corr_mlp.fc1.bias"]))
        h_tanh = torch.nn.functional.gelu(torch.nn.functional.linear(vol, sd["corr_mlp.fc1.weight"], sd["corr_mlp.fc1.bias"]), approximate="tanh")
    assert float((h_erf - h_tanh).abs().max()) > 1e-4
    got = eng.linear(vol.to(DEV), sd["corr_mlp.fc1.weight"].to(DEV), sd["corr_mlp.fc1.bias"].to(DEV), act=1).cpu()
    # mean abs distance: GEMM rounding (~1e-5) is far below the erf/tanh gap (~2e-4)
    d_erf, d_tanh = float((got - h_erf).abs().mean()), float((got - h_tanh).abs().mean())
    assert d_erf < 0.2 * d_tanh, (d_erf, d_tanh)


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("H4,W4", [(24, 32), (64, 72)])   # 64x72: every level >= 8x8 -> correlate-then-interpolate kernel
def test_update_loop_vs_oracle(eng, impl, H4, W4):
    """The hot loop alone: identical pyramid/support on both sides, amplified heads (several px of motion)."""
    sd = _amplified_sd(seed=7, head_gain=10.0, vis_gain=100.0)
    T, N, iters = 7, 37, 4
    fmaps = _pyramid_case(T, H4, W4, seed=4)
    pyr_cpu = O.normalized_pyramid(fmaps)
    g = torch.Generator().manual_seed(31)
    qf = torch.randint(0, T, (N,), generator=g)
    qc = _coords_case(1, N, H4, W4, 17)[0]
    sup_cpu = [O.support_features(pyr_cpu[l], qf, qc / 2 ** l) for l in range(4)]
    c0 = qc[None].expand(T, N, 2).contiguous()
    with torch.no_grad():
        wc, wv, wq = O.update_loop(sd, pyr_cpu, sup_cpu, c0, torch.zeros(T, N), torch.zeros(T, N), iters)
    pyr = eng.prepare_pyramid(fmaps.to(DEV))
    support = torch.stack(sup_cpu).to(DEV).contiguous()
    packed = eng.pack_weights(sd, DEV)
    coords, vis, conf = c0.to(DEV).clone(), torch.zeros(T, N, device=DEV), torch.zeros(T, N, device=DEV)
    ws = torch.empty(eng.workspace_bytes(T, N, H4, W4), dtype=torch.uint8, device=DEV)
    te = O.time_embedding(sd, T)[0].contiguous().to(DEV)
    eng.set_option("gemm", impl)
    try:
        eng.update_loop(packed, pyr, H4, W4, support, None, coords, vis, conf, te, iters, ws)
        torch.cuda.synchronize()
    finally:
        eng.set_option("gemm", 0)
    assert float((wc - c0).abs().max()) > 0.25, "case must move"
    e_c = float((coords.cpu() - wc).abs().max()) * 4  # pixels
    e_v = float((vis.cpu() - wv).abs().max())
    e_q = float((conf.cpu() - wq).abs().max())
    print("loop parity", impl, e_c, e_v, e_q)
    assert e_c < 1e-3 and e_v < 1e-3 and e_q < 1e-3


def test_update_loop_cluster_gemm_vs_simt_at_scale(eng):
    """N=2400, T=16: every big GEMM runs many tiles per persistent CTA; the SIMT fp32 GEMM is the on-GPU yardstick."""
    sd = _amplified_sd(seed=9, head_gain=10.0, vis_gain=100.0)
    T, N, H4, W4, iters = 16, 2400, 48, 64, 2
    fmaps = _pyramid_case(T, H4, W4, seed=6)
    pyr = eng.prepare_pyramid(fmaps.to(DEV))
    g = torch.Generator().manual_seed(41)
    qf = torch.randint(0, T, (N,), generator=g).to(torch.int32).to(DEV)
    qc = (torch.rand(N, 2, generator=g) * torch.tensor([W4 - 1.0, H4 - 1.0])).to(DEV)
    support = eng.sample_support(pyr, T, H4, W4, qf, qc)
    packed = eng.pack_weights(sd, DEV)
    te = O.time_embedding(sd, T)[0].contiguous().to(DEV)
    ws = torch.empty(eng.workspace_bytes(T, N, H4, W4), dtype=torch.uint8, device=DEV)
    out = {}
    for impl in (0, 1):
        coords = qc[None].expand(T, N, 2).contiguous().clone()
        vis, conf = torch.zeros(T, N, device=DEV), torch.zeros(T, N, device=DEV)
        eng.set_option("gemm", impl)
        try:
            eng.update_loop(packed, pyr, H4, W4, support, None, coords, vis, conf, te, iters, ws)
            torch.cuda.synchronize()
        finally:
            eng.set_option("gemm", 0)
        out[impl] = (coords.cpu(), vis.cpu(), conf.cpu())
    assert float((out[1][0] - qc.cpu()[None]).abs().max()) > 0.25, "case must move"
    e_c = float((out[0][0] - out[1][0]).abs().max()) * 4
    e_v = float((out[0][1] - out[1][1]).abs().max())
    print("cluster-vs-simt", e_c, e_v)
    assert e_c < 5e-4 and e_v < 5e-4


def test_encoder_matches_torch(eng):
    """The whole BasicEncoder + L2-normalise + pyramid in libct3_b200 (conv1 SIMT, implicit-GEMM 3x3 convolutions on
    TMA-shifted NHWC boxes, gather + GEMM for the strided ones, InstanceNorm/ReLU/residual kernels, fused
    resize + concat) vs the fp32 PyTorch module holding the same weights (cuDNN, TF32 off) on the same GPU.  Odd map
    sizes exercise partial tiles, zero padding through TMA out-of-bounds fill and the strided-conv size arithmetic;
    18 frames = two 16-frame chunks."""
    from cotracker_b200.build import build_cotracker
    from cotracker_b200.synthetic import seeded_state_dict, texture_video
    m = build_cotracker(None, offline=True, window_len=60)
    m.load_state_dict(seeded_state_dict(5))
    m = m.to(DEV).eval()
    for (T, H, W) in [(3, 96, 128), (2, 384, 512), (18, 100, 132)]:
        x = (2 * (texture_video(T, H, W, seed=T)[0] / 255) - 1).to(DEV)
        prev = torch.backends.cudnn.allow_tf32
        torch.backends.cudnn.allow_tf32 = False
        try:
            with torch.no_grad():
                want_fm = m.fnet(x)
        finally:
            torch.backends.cudnn.allow_tf32 = prev
        want = O.normalized_pyramid(want_fm.cpu())
        with torch.no_grad():
            pyr = m._encode(x, 200)
        levels = eng.pyramid_levels(pyr, T, H // 4, W // 4)
        for l in range(4):
            got = levels[l].permute(0, 3, 1, 2).cpu()
            err = float((got - want[l]).abs().max())
            assert err < 2e-5, (T, H, W, l, err)     # unit-norm features: 2e-5 abs ~ bf16x3 + fp32 ordering noise


def test_upsample_concat_matches_torch(eng):
    import torch.nn.functional as F
    g = torch.Generator().manual_seed(8)
    for (T, H, W) in [(2, 24, 32), (3, 25, 33), (1, 96, 128)]:
        shapes = [(64, 2 * H, 2 * W), (96, H, W), (128, (H + 1) // 2, (W + 1) // 2), (128, (H + 3) // 4, (W + 3) // 4)]
        feats = [torch.randn(T, c, h, w, generator=g).to(DEV) for (c, h, w) in shapes]
        want = torch.cat([F.interpolate(f, (H, W), mode="bilinear", align_corners=True) for f in feats], dim=1)
        got = eng.upsample_concat(feats, H, W)
        assert got.shape == want.shape
        assert float((got - want).abs().max()) < 2e-5
