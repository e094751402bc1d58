"""CPU tests of clip ingestion: the ct3_prepare_frames symbol and its argument validation before any launch, the
host-clip chunk plan and staging bound, and the CUDA-only contract of the predictors for host clips."""
import ctypes
import os
import re

import pytest
import torch

from cotracker_b200 import engine, ingest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_prepare_frames_exported_and_declared():
    lib = engine.lib()
    assert hasattr(lib, "ct3_prepare_frames") and "ct3_prepare_frames" in engine.EXPORTED_SYMBOLS
    with open(os.path.join(ROOT, "include", "ct3_b200.h")) as f:
        header = f.read()
    assert re.search(r"int ct3_prepare_frames\(", header)
    assert "CT3_FRAMES_U8 = 0" in header and "CT3_FRAMES_F32 = 1" in header
    assert engine.FRAME_DTYPES == {torch.uint8: 0, torch.float32: 1}


def test_prepare_frames_rejects_bad_arguments_without_gpu():
    """Each invalid argument returns CT3_EINVAL with a message before any launch (fake pointers, legacy stream:
    reaching a launch would fail differently)."""
    lib = engine.lib()
    src, out = ctypes.c_void_p(1 << 20), ctypes.c_void_p(1 << 24)
    big = 2 ** 62
    ok = dict(src=src, dtype=0, T=4, H=90, W=120, st=3 * 90 * 120, sc=90 * 120, sh=120, sw=1, oh=384, ow=512, out=out)

    def call(**kw):
        a = dict(ok, **kw)
        return lib.ct3_prepare_frames(a["src"], a["dtype"], a["T"], a["H"], a["W"], a["st"], a["sc"], a["sh"], a["sw"],
                                      a["oh"], a["ow"], a["out"], None)

    cases = [
        (dict(src=None), b"null argument"),
        (dict(out=None), b"null argument"),
        (dict(T=0), b"must be >= 1"), (dict(H=0), b"must be >= 1"), (dict(W=-1), b"must be >= 1"),
        (dict(oh=0), b"must be >= 1"), (dict(ow=0), b"must be >= 1"),
        (dict(dtype=2), b"unknown frame dtype"), (dict(dtype=-1), b"unknown frame dtype"),
        (dict(st=big), b"stride extent"),                          # 3 * 2^62 elements
        (dict(sh=-(2 ** 63)), b"stride extent"),
        (dict(dtype=1, sc=2 ** 61), b"stride extent"),             # fits in elements, not in bytes
        (dict(oh=65536, ow=32768), b"output plane too large"),    # 2^31 pixels: beyond the kernel's int index
        (dict(T=2 ** 31 - 1, oh=1, ow=2 ** 31 - 1, st=0), b"output too large"),
    ]
    for kw, msg in cases:
        assert call(**kw) == -1, kw
        assert msg in lib.ct3_last_error(), (kw, lib.ct3_last_error())


def test_prepare_frames_wrapper_rejects_host_and_bad_tensors():
    with pytest.raises(engine.EngineError):
        engine.prepare_frames(torch.zeros(2, 3, 8, 8, dtype=torch.uint8), (4, 4))


def test_chunk_plan_and_staging_bound():
    fb = 3 * 1080 * 1920                                           # one uint8 1080p frame
    slot = ingest.STAGING_SLOT_BYTES
    k = ingest.chunk_frames(120, fb)
    assert k == slot // fb and k >= 1
    for T in (1, 2, 5, 7, 48, 120):
        for frame_bytes in (1, 1000, fb, 4 * fb, slot, slot + 1, 3 * slot):
            plan = ingest.plan_chunks(T, frame_bytes)
            assert [t for a, b in plan for t in range(a, b)] == list(range(T))     # every frame once, in order
            k = ingest.chunk_frames(T, frame_bytes)
            assert all(b - a == k for a, b in plan[:-1]) and 1 <= plan[-1][1] - plan[-1][0] <= k
            sb = ingest.staging_bytes(T, frame_bytes)
            assert sb == 2 * k * frame_bytes
            assert sb <= 2 * max(slot, frame_bytes)                                 # the documented bound
            assert sb <= 2 * T * frame_bytes
    assert ingest.chunk_frames(3, 100, slot_bytes=1000) == 3                        # never more than T
    assert ingest.plan_chunks(7, 10, slot_bytes=30) == [(0, 3), (3, 6), (6, 7)]
    with pytest.raises(ValueError):
        ingest.chunk_frames(0, 10)


def test_frame_density():
    x = torch.zeros(5, 3, 6, 7)
    assert ingest.frame_is_dense(x.shape[1:], x.stride()[1:])
    thwc = torch.zeros(5, 6, 7, 3).permute(0, 3, 1, 2)
    assert ingest.frame_is_dense(thwc.shape[1:], thwc.stride()[1:])
    assert ingest.frame_is_dense(x[::2].shape[1:], x[::2].stride()[1:])
    for v in (x[:, :, :, :5], x[:, :, ::2], thwc[:, :, :, 1:5], x[:, ::2]):
        assert not ingest.frame_is_dense(v.shape[1:], v.stride()[1:])
    rows = thwc[:, :, 1:5]                     # a run of whole rows of a THWC frame is still one block
    assert ingest.frame_is_dense(rows.shape[1:], rows.stride()[1:])
    one = torch.zeros(2, 3, 1, 7)
    assert ingest.frame_is_dense(one.shape[1:], one.stride()[1:])


def test_host_clip_with_cpu_model_raises_engine_error():
    """A host-resident clip never reaches eager PyTorch: with the model on the CPU every predictor raises EngineError,
    for uint8 and float clips."""
    from cotracker_b200.build import build_cotracker
    from cotracker_b200.evaluation import EvaluationPredictor
    from cotracker_b200.predictor import CoTrackerOnlinePredictor, CoTrackerPredictor
    for clip in (torch.zeros(1, 4, 3, 64, 64, dtype=torch.uint8), torch.zeros(1, 4, 3, 64, 64)):
        p = CoTrackerPredictor(checkpoint=None, window_len=8)
        with pytest.raises(engine.EngineError):
            p(clip, grid_size=2)
        with pytest.raises(engine.EngineError):
            p(clip, queries=torch.zeros(1, 1, 3), backward_tracking=True)
        op = CoTrackerOnlinePredictor(checkpoint=None, window_len=4)
        op(video_chunk=clip, is_first_step=True, grid_size=2)
        with pytest.raises(engine.EngineError):
            op(video_chunk=clip)
        ev = EvaluationPredictor(build_cotracker(None, offline=True, window_len=8), single_point=False)
        with pytest.raises(engine.EngineError):
            ev(clip, torch.zeros(1, 1, 3))
    with pytest.raises(engine.EngineError):
        ingest.prepare_video(torch.zeros(1, 2, 3, 8, 8, dtype=torch.uint8), (8, 8), "cpu")
