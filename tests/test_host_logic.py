"""CPU tests of the host side: ABI surface, state-dict contract, query construction, replica sharding (gloo)."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    from cotracker_b200 import engine
    lib = engine.lib()  # raises if the .so is missing: build it first (__graft_entry__.build)
    header = open(os.path.join(ROOT, "include", "ct3_b200.h")).read()
    declared = set(re.findall(r"\b(ct3_[a-z0-9_]+)\s*\(", header))
    declared -= {"ct3_update_iter"}  # mentioned in a comment only
    assert declared == set(engine.EXPORTED_SYMBOLS), declared ^ set(engine.EXPORTED_SYMBOLS)
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.ct3_version() >= 100


def test_abi_argument_validation_with_loop_shapes_without_gpu():
    from cotracker_b200 import engine
    lib = engine.lib()
    n = ctypes.c_size_t(0)

    def ws(shape, out=ctypes.byref(n)):
        return lib.ct3_workspace_bytes(None if shape is None else ctypes.byref(shape), out)

    assert ws(engine._loop_shape(16, 6400, 96, 128)) == 0 and n.value > 6e9
    assert ws(engine._loop_shape(0, 10, 0, 0)) == -1                           # CT3_EINVAL
    assert b"T and N" in lib.ct3_last_error()
    assert ws(engine._loop_shape(4, 4, 0, 0), None) == -1
    assert ws(None) == -1 and b"null shape" in lib.ct3_last_error()
    off, h, w, total = engine.pyramid_layout(16, 96, 128)
    assert h == [96, 48, 24, 12] and w == [128, 64, 32, 16] and total == 16 * 16320 * 128
    with pytest.raises(engine.EngineError):
        engine.pyramid_layout(2, 4, 4)                                      # level 3 would be 0x0
    assert lib.ct3_set_option(b"nope", 1) == -1
    assert engine.get_option("gemm") == 0
    assert lib.ct3_update_loop(None, None, None, None, None, None, None, None, 1, None, None, 0, None) == -1
    one = ctypes.c_void_p(256)
    assert lib.ct3_update_loop(one, one, one, None, one, one, one, one, 1, None, one, 1 << 40, None) == -1
    assert b"null shape" in lib.ct3_last_error()
    # the split-bf16 pyramid copy of the correlation kernel is part of the workspace iff every level is >= 8x8 texels
    *_, total = engine.pyramid_layout(16, 96, 128)
    assert engine.workspace_bytes(16, 6400, 96, 128) - engine.workspace_bytes(16, 6400) == total * 4
    assert engine.workspace_bytes(4, 10, 24, 32) == engine.workspace_bytes(4, 10)       # level 3 is 3x4
    assert ws(engine._loop_shape(4, 10, 4, 4)) == -1                                     # level 3 would be 0x0
    # stage entry: argument checks come before any launch
    assert lib.ct3_corr_sample(None, 96, 128, one, None, one, 2, 5, one, None, 0, None) == -1
    assert lib.ct3_corr_sample(one, 96, 128, one, None, one, 2, 5, one, ctypes.c_void_p(264), 1 << 30, None) == -1
    assert b"256-byte aligned" in lib.ct3_last_error()
    assert lib.ct3_corr_sample(one, 96, 128, one, None, one, 2, 5, one, ctypes.c_void_p(512), 1024, None) == -3   # CT3_ENOSPC


def test_attention_stage_argument_validation_without_gpu():
    """ct3_attention / ct3_attention_workspace_bytes reject bad arguments with CT3_EINVAL / CT3_ENOSPC before any
    launch (the pointers below are never dereferenced)."""
    from cotracker_b200 import engine
    lib = engine.lib()
    n, m = ctypes.c_size_t(0), ctypes.c_size_t(0)
    assert lib.ct3_attention_workspace_bytes(16, 6400, 1, ctypes.byref(n)) == 0 and n.value > 0
    assert lib.ct3_attention_workspace_bytes(16, 6400, 8, ctypes.byref(m)) == 0 and m.value > n.value   # + group table
    assert lib.ct3_attention_workspace_bytes(16, 6400, 1, None) == -1
    assert lib.ct3_attention_workspace_bytes(0, 10, 1, ctypes.byref(n)) == -1
    assert lib.ct3_attention_workspace_bytes(4, 10, 11, ctypes.byref(n)) == -1          # G > N
    assert lib.ct3_attention_workspace_bytes(4, 10, 0, ctypes.byref(n)) == -1
    assert lib.ct3_attention_workspace_bytes(4, 10, 1, ctypes.byref(n)) == 0
    need = n.value
    p, ws = ctypes.c_void_p(1 << 20), ctypes.c_void_p(1 << 21)
    one = (ctypes.c_int32 * 1)(10)

    def call(kind=1, q=p, kv=p, T=4, N=10, sizes=one, G=1, out=p, w=ws, nbytes=need):
        return lib.ct3_attention(kind, q, kv, T, N, sizes, G, out, w, nbytes, None)

    assert call(q=None) == -1 and call(kv=None) == -1 and call(out=None) == -1 and call(w=None) == -1
    assert call(kind=-1) == -1 and call(kind=4) == -1 and b"kind" in lib.ct3_last_error()
    assert call(T=0) == -1 and call(N=0) == -1
    assert call(sizes=None) == -1 and call(G=0) == -1
    assert call(sizes=(ctypes.c_int32 * 2)(4, 5), G=2) == -1 and b"sum to N" in lib.ct3_last_error()
    assert call(sizes=(ctypes.c_int32 * 2)(10, 0), G=2, N=10) == -1
    assert call(q=ctypes.c_void_p((1 << 20) + 4)) == -1 and b"16-byte" in lib.ct3_last_error()
    assert call(out=ctypes.c_void_p((1 << 20) + 8)) == -1
    assert call(w=ctypes.c_void_p((1 << 21) + 16)) == -1 and b"256-byte" in lib.ct3_last_error()
    assert call(nbytes=need - 1) == -3                                                   # CT3_ENOSPC


def test_loop_tokens_and_update_loop_argument_validation_without_gpu():
    """ct3_loop_tokens rejects bad arguments with update_loop's checks and messages (CT3_EINVAL / CT3_ENOSPC) before
    any launch (the pointers below are never dereferenced)."""
    from cotracker_b200 import engine
    lib = engine.lib()
    T, N, H4, W4 = 4, 10, 64, 72
    need = engine.workspace_bytes(T, N, H4, W4)
    p, ws = ctypes.c_void_p(1 << 20), ctypes.c_void_p(1 << 21)

    def call(packed=p, pyr=p, H4=H4, W4=W4, support=p, coords=p, vis=p, conf=p, te=p, T=T, N=N, w=ws, nbytes=need,
             outs=(None, None, None)):
        return lib.ct3_loop_tokens(packed, pyr, H4, W4, support, None, coords, vis, conf, te, T, N, *outs, w, nbytes,
                                   None)

    for k in ("packed", "pyr", "support", "coords", "vis", "conf", "te", "w"):
        assert call(**{k: None}) == -1 and b"null argument" in lib.ct3_last_error(), k
    assert call(T=0) == -1 and b"T and N" in lib.ct3_last_error()
    assert call(N=0) == -1 and b"T and N" in lib.ct3_last_error()
    assert call(N=1 << 30) == -1 and b"too large" in lib.ct3_last_error()
    assert call(H4=4, W4=4) == -1                                                       # level 3 would be 0x0
    assert call(w=ctypes.c_void_p((1 << 21) + 16)) == -1 and b"256-byte" in lib.ct3_last_error()
    assert call(nbytes=need - 1) == -3 and b"workspace too small" in lib.ct3_last_error()   # CT3_ENOSPC
    # the same messages as ct3_update_loop for the same faults
    shape = engine._loop_shape(T, N, H4, W4)
    assert lib.ct3_update_loop(p, p, p, None, p, p, p, p, 1, ctypes.byref(shape), ws, need - 1, None) == -3
    assert b"workspace too small" in lib.ct3_last_error()


def test_loop_tokens_branch_map_matches_library():
    """The branch map of test_gpu_tokens.py (which correlation kernel, volume format, fc1 weights and products a call
    runs) against what the compiled library reports, across the options and pyramid shapes (every level >= 8x8 or not)."""
    import itertools
    from cotracker_b200 import engine
    from test_gpu_tokens import loop_branch
    lib = engine.lib()
    flag = ctypes.c_int(0)
    try:
        for corr, pc, pf, (H4, W4) in itertools.product(range(3), (1, 2, 3), (1, 2, 3),
                                                        [(24, 32), (64, 72), (96, 128), (64, 63), (63, 64), (8, 8)]):
            for k, v in (("corr", corr), ("prec.corr", pc), ("prec.fc1", pf)):
                engine.set_option(k, v)
            b = loop_branch(16, H4, W4, corr, pc, pf)
            assert engine.precision_info(16, H4, W4) == (b["corr_products"], b["products"],
                                                         2 if b["volume"] == "fp16" else 4), (corr, pc, pf, H4, W4)
            assert lib.ct3_volume_is_support_major(16, H4, W4, ctypes.byref(flag)) == 0
            assert bool(flag.value) == b["support_major"], (corr, pc, pf, H4, W4)
    finally:
        for k, v in (("corr", 0), ("prec.corr", 2), ("prec.fc1", 3)):
            engine.set_option(k, v)
    assert loop_branch(16, 96, 128)["weights"] == "corr_fc1_t"
    assert loop_branch(16, 96, 128, prec_fc1=2)["weights"] == "corr_fc1_th"
    assert loop_branch(16, 96, 128, prec_corr=3, prec_fc1=1)["weights"] == "corr_fc1_h"
    assert loop_branch(16, 24, 32, prec_fc1=1) == loop_branch(16, 24, 32, corr=2)    # no patch kernel: split x split


def test_weight_names_match_state_dict():
    from cotracker_b200 import engine
    from cotracker_b200.build import build_cotracker
    names = engine.weight_names()
    sd = build_cotracker(None, offline=True, window_len=60).state_dict()
    hot = [k for k in sd if k.startswith(("updateformer.", "corr_mlp."))]
    assert sorted(names) == sorted(hot)
    assert len(names) == 143
    assert sum(sd[k].numel() for k in sd if k != "time_emb") == 25385700      # SURVEY Appendix B
    assert sd["time_emb"].shape == (1, 60, 1110)
    assert "updateformer.virual_tracks" in sd                                   # (sic)


def test_v2_and_training_are_rejected():
    from cotracker_b200.build import build_cotracker
    with pytest.raises(NotImplementedError):
        build_cotracker(None, v2=True)


def test_grid_queries_match_reference_contract():
    from cotracker_b200.predictor import get_points_on_a_grid
    g = get_points_on_a_grid(80, (384, 512))
    assert g.shape == (1, 6400, 2)
    assert float(g[0, :, 0].min()) == 8.0 and float(g[0, :, 0].max()) == 504.0   # margin W/64
    assert float(g[0, :, 1].min()) == 8.0 and float(g[0, :, 1].max()) == 376.0
    assert torch.equal(g[0, 1] - g[0, 0], torch.tensor([g[0, 1, 0] - 8.0, 0.0]))     # row-major, x fastest
    assert get_points_on_a_grid(1, (384, 512)).tolist() == [[[256.0, 192.0]]]


def test_grid_and_time_embedding_match_live_reference():
    """Against the reference's get_points_on_a_grid / sincos embedding (tests/golden/reference_host.npz)."""
    from cotracker_b200.model import sincos_time_embedding
    from cotracker_b200.predictor import get_points_on_a_grid
    with np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_host.npz")) as z:
        for i, size in ((2, 1), (1, 5), (3, 30)):
            assert torch.equal(get_points_on_a_grid(size, (384, 512)), torch.from_numpy(z[f"grid_{i}"]))
        for L in (16, 60):
            assert torch.equal(sincos_time_embedding(1110, L), torch.from_numpy(z[f"sincos_{L}"]))


def test_shard_clips():
    from cotracker_b200.sharding import shard_clips
    assert [shard_clips(8, 8, r) for r in range(8)] == [[r] for r in range(8)]
    assert shard_clips(10, 4, 1) == [1, 5, 9]
    assert sorted(sum((shard_clips(13, 4, r) for r in range(4)), [])) == list(range(13))


_WORKER = r"""
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1])
from cotracker_b200.build import build_cotracker
from cotracker_b200.sharding import broadcast_state_dict, shard_clips, gather_results
dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
torch.manual_seed(100 + rank)                      # different random weights per rank before the broadcast
m = build_cotracker(None, offline=False, window_len=16)
sent = broadcast_state_dict(m, src=0)
ref = torch.cat([v.reshape(-1).float() for _, v in sorted(m.state_dict().items())])
chk = ref.clone(); dist.broadcast(chk, src=0)
assert torch.equal(ref, chk), "weights differ after broadcast"
assert sent >= 25385700 * 4
mine = shard_clips(5, world, rank)
tr = torch.full((1, 2, 3, 2), float(rank)); vi = torch.ones(1, 2, 3, dtype=torch.bool)
tl, vl = gather_results(tr, vi, dst=0)
if rank == 0:
    assert [float(t.mean()) for t in tl] == [0.0, 1.0] and all(v.all() for v in vl)
print("OK", rank, mine)
"""


def test_replica_sharding_world_size_2_gloo(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(_WORKER)
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", "29613", str(script), ROOT],
                       capture_output=True, text=True, timeout=240, env=env)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "OK 0 [0, 2, 4]" in r.stdout and "OK 1 [1, 3]" in r.stdout


def test_corr_patch_taps_stay_in_box():
    """fp32 restatement of box_origin8 / tap_pair (csrc/corr_tc2.cu): for every map size >= 8 and every coordinate --
    far outside, on texel centres, one ulp either side of them -- both bilinear taps of all 7 border-clamped samples
    lie inside the 8-texel box the TMA load fetches, once a zero-weight second tap is folded onto the first (the case
    `c + offset` rounding up to an integer in fp32).  The kernel relies on this to index the box without a fallback."""
    import numpy as np
    f32 = np.float32
    rng = np.random.default_rng(0)
    for size in (8, 9, 12, 16, 24, 48, 96, 128, 1000):
        ints = np.arange(-6, size + 7).astype(f32)
        near = [ints]
        lo, hi = ints.copy(), ints.copy()
        for _ in range(6):
            lo, hi = np.nextafter(lo, f32(-1e9)), np.nextafter(hi, f32(1e9))
            near += [lo.copy(), hi.copy()]
        c = np.concatenate([rng.uniform(-40, size + 40, 100000).astype(f32), np.array([-1e9, 1e9], dtype=f32)] + near)
        cc = np.minimum(np.maximum(c, f32(-16)), f32(size + 16)).astype(f32)
        origin = np.clip(np.floor(cc).astype(np.int64) - 3, 0, size - 8)
        for a in range(7):
            x = np.minimum(np.maximum((c + f32(a - 3)).astype(f32), f32(0)), f32(size - 1)).astype(f32)
            xf = np.floor(x)
            x0 = xf.astype(np.int64)
            w = (x - xf).astype(f32)
            x1 = np.minimum(x0 + 1, size - 1)
            s0 = x0 - origin
            s1 = np.where(w > 0, x1 - origin, s0)
            assert s0.min() >= 0 and s0.max() <= 7 and s1.min() >= 0 and s1.max() <= 7, (size, a)


def test_dropin_package_and_hub_entry_points():
    """The import-path shim (dropin/cotracker/...) and hubconf.py expose the reference's names (INTEGRATION.md 1):
    `from cotracker.predictor import CoTrackerPredictor`, `build_cotracker`, `torch.hub.load(..., source="local")`."""
    code = (
        "import torch, cotracker\n"
        "from cotracker.predictor import CoTrackerPredictor, CoTrackerOnlinePredictor\n"
        "from cotracker.models.build_cotracker import build_cotracker\n"
        "from cotracker.models.core.cotracker.cotracker3_offline import CoTrackerThreeOffline\n"
        "from cotracker.models.core.cotracker.cotracker3_online import CoTrackerThreeOnline\n"
        "import cotracker_b200.predictor as P\n"
        "assert CoTrackerPredictor is P.CoTrackerPredictor and CoTrackerOnlinePredictor is P.CoTrackerOnlinePredictor\n"
        "m = build_cotracker(None, offline=False, window_len=16)\n"
        "assert isinstance(m, CoTrackerThreeOnline) and m.window_len == 16 and m.model_resolution == (384, 512)\n"
        "on = torch.hub.load(%r, 'cotracker3_online', source='local', pretrained=False)\n"
        "off = torch.hub.load(%r, 'cotracker3_offline', source='local', pretrained=False)\n"
        "assert type(on).__name__ == 'CoTrackerOnlinePredictor' and on.step == 8 and on.model.window_len == 16\n"
        "assert type(off).__name__ == 'CoTrackerPredictor' and off.model.window_len == 60 and off.interp_shape == (384, 512)\n"
        "print('HUB_OK')\n" % (ROOT, ROOT))
    env = dict(os.environ, PYTHONPATH=os.path.join(ROOT, "dropin") + os.pathsep + ROOT)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=240, env=env, cwd="/tmp")
    assert r.returncode == 0 and "HUB_OK" in r.stdout, r.stdout + r.stderr


def test_non_default_model_resolution_is_rejected():
    """tokens.cu normalises the relative-motion posenc by (128, 96) = (512, 384)/4 (ADVICE r1)."""
    from cotracker_b200.model import CoTrackerThreeOffline
    with pytest.raises(NotImplementedError):
        CoTrackerThreeOffline(window_len=60, model_resolution=(256, 320))


def test_options_are_validated_and_thread_local():
    import threading
    from cotracker_b200 import engine
    lib = engine.lib()
    assert lib.ct3_set_option(b"corr", 7) == -1 and b"out of range" in lib.ct3_last_error()
    assert lib.ct3_set_option(b"attn", -1) == -1
    assert lib.ct3_set_option(b"corr", 3) == -1 and b"out of range" in lib.ct3_last_error()
    assert lib.ct3_set_option(b"attn", 2) == -1 and b"out of range" in lib.ct3_last_error()
    assert engine.get_option("corr") == 0 and engine.get_option("attn") == 0
    assert engine.get_option("fuse") == 1
    assert lib.ct3_set_option(b"fuse", 2) == -1 and b"out of range" in lib.ct3_last_error()
    assert lib.ct3_set_option(b"fuse", 0) == 0 and engine.get_option("fuse") == 0
    assert lib.ct3_set_option(b"fuse", 1) == 0
    assert lib.ct3_set_option(b"gemm", 1) == 0 and engine.get_option("gemm") == 1
    seen = []
    t = threading.Thread(target=lambda: seen.append(engine.get_option("gemm")))   # another host thread: defaults
    t.start(); t.join()
    assert seen == [0]
    assert lib.ct3_set_option(b"gemm", 0) == 0


def test_corr_shift_pattern_covers_every_sample():
    """fp32 restatement of box_origin8 / tap_weights (csrc/corr_tc3.cu; tests/corr_cases.py).  The transposed
    correlation kernel blends the 8x8 raw correlations with STATIC register indices: per frame and axis the two taps of
    sample a are box entries clamp07(a + d) and clamp07(a + d + 1) for one shift d = clamp(floor(clamp(c)) - 3 - origin,
    -7, 7).  This test brute-forces, for every map size >= 8 and every coordinate class (far outside, on texel centres,
    a few ulps either side), that the border-clamped bilinear taps of all 7 samples -- computed exactly as grid_sample
    does -- ARE that pattern with weights (1 - w, w), or (0, 1) when c + offset rounded up to an integer; and that the
    blend value equals the straightforward two-tap evaluation.  The kernel traps otherwise; this is the proof that it
    never does."""
    import numpy as np
    from corr_cases import box_origin8, tap_weights
    f32 = np.float32
    rng = np.random.default_rng(1)
    for size in (8, 9, 12, 16, 24, 48, 96, 128, 1000):
        ints = np.arange(-20, size + 21).astype(f32)
        near = [ints]
        lo, hi = ints.copy(), ints.copy()
        for _ in range(6):
            lo, hi = np.nextafter(lo, f32(-1e9)), np.nextafter(hi, f32(1e9))
            near += [lo.copy(), hi.copy()]
        c = np.concatenate([rng.uniform(-40, size + 40, 200000).astype(f32), np.array([-1e9, 1e9, 0.5, size - 0.5], dtype=f32)] + near)
        origin, d = box_origin8(c, size)
        box = rng.standard_normal((len(c), 8)).astype(f32)            # the 8 box entries along this axis
        rows = np.arange(len(c))
        for a in range(7):
            branch, u, w, s0, s1, i0, i1, fr = tap_weights(c, a, size, origin, d)
            assert bool((branch != 0).all()), (size, a, c[branch == 0][:5])
            want = (f32(1) - fr) * box[rows, s0] + fr * box[rows, s1]
            got = u * box[rows, i0] + w * box[rows, i1]
            assert np.array_equal(want.astype(f32), got.astype(f32)), (size, a)
