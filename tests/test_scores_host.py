"""CPU tests of the probability outputs (`return_scores`): the ABI of ct3_finish_tracks_scores and
ct3_online_window_end_scores and their rejections before any launch, the library version, the default of every public
`return_scores` argument, its check before any device work, and the `TrackScores` exports."""
import ctypes
import importlib.util
import inspect
import os

import pytest
import torch

from cotracker_b200 import engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("ct3_finish_tracks_scores", "ct3_online_window_end_scores")


def test_scores_entry_points_are_exported_and_the_version_stays():
    lib = engine.lib()
    with open(os.path.join(ROOT, "include", "ct3_b200.h")) as f:
        header = f.read()
    for name in NEW:
        assert name in engine.EXPORTED_SYMBOLS and hasattr(lib, name)
        assert f"int {name}(" in header
    assert lib.ct3_version() == 102
    assert ctypes.sizeof(engine.OnlineScores) == 16


def test_finish_tracks_scores_rejects_bad_arguments():
    """Every ct3_finish_tracks rejection, and the scores' own, return CT3_EINVAL before any launch (the fake pointers
    would fail on the device otherwise)."""
    lib = engine.lib()
    p, f = ctypes.c_void_p(256), ctypes.c_float
    ok = dict(B=2, T=5, N=7, n_keep=7)

    def call(fwd_t=p, fwd_v=p, fwd_c=p, bwd_t=None, bwd_v=None, bwd_c=None, q=p, out_t=p, out_v=p, sv=p, sc=p, **kw):
        a = {**ok, **kw}
        return lib.ct3_finish_tracks_scores(fwd_t, fwd_v, fwd_c, bwd_t, bwd_v, bwd_c, q, a["B"], a["T"], a["N"],
                                            a["n_keep"], f(0.9), f(1.0), f(1.0), out_t, out_v, sv, sc, None)

    for bad in (dict(fwd_t=None), dict(fwd_v=None), dict(q=None), dict(out_t=None), dict(out_v=None),
                dict(fwd_c=None), dict(sv=None), dict(sc=None)):
        assert call(**bad) == -1 and b"null argument" in lib.ct3_last_error(), bad
    assert call(bwd_t=p, bwd_c=p) == -1 and b"given together" in lib.ct3_last_error()
    assert call(bwd_t=p, bwd_v=p) == -1 and b"bwd_conf" in lib.ct3_last_error()     # backward pair without conf
    assert call(bwd_c=p) == -1 and b"bwd_conf" in lib.ct3_last_error()              # conf without the pair
    for bad in (dict(B=0), dict(T=0), dict(N=0)):
        assert call(**bad) == -1 and b"must be >= 1" in lib.ct3_last_error()
    for bad in (dict(n_keep=0), dict(n_keep=8)):
        assert call(**bad) == -1 and b"n_keep" in lib.ct3_last_error()
    assert call(fwd_t=ctypes.c_void_p(260)) == -1 and b"8-byte aligned" in lib.ct3_last_error()
    assert call(B=1 << 20, T=1 << 20, N=1 << 10) == -1 and b"too large" in lib.ct3_last_error()


def test_online_window_end_scores_rejects_bad_arguments():
    lib = engine.lib()
    p = ctypes.c_void_p(1 << 20)
    stream_bytes, scores_bytes = ctypes.sizeof(engine.OnlineStream), ctypes.sizeof(engine.OnlineScores)

    def entry(**kw):
        e = engine.OnlineStream(p.value, p.value, p.value, 64, 0, p.value, p.value, 0, 16, 10, 0, 0, 10, 1.0, 1.0)
        for k, v in kw.items():
            setattr(e, k, v)
        return e

    def end(entries, scores=None, ws=4096, N=None):
        arr = (engine.OnlineStream * len(entries))(*entries)
        sc = None if scores is False else (engine.OnlineScores * len(entries))(
            *(scores or [engine.OnlineScores(p.value, p.value)] * len(entries)))
        N = sum(e.n for e in entries) if N is None else N
        return lib.ct3_online_window_end_scores(arr, len(entries), 16, 4, p, p, p, N, ctypes.c_float(0.6), sc, p, ws,
                                                None)

    assert end([entry()], scores=False) == -1 and b"null" in lib.ct3_last_error()
    assert end([entry()], scores=[engine.OnlineScores(p.value, None)]) == -1 and b"both" in lib.ct3_last_error()
    assert end([entry()], scores=[engine.OnlineScores(None, p.value)]) == -1
    assert end([entry(tracks=None, visibility=None)]) == -1 and b"output" in lib.ct3_last_error()
    assert end([entry()], scores=[engine.OnlineScores(p.value + 2, p.value)]) == -1 and b"aligned" in lib.ct3_last_error()
    # the workspace holds the streams and then the scores
    assert end([entry(), entry(first=10)], ws=2 * stream_bytes) == -3
    assert end([entry(), entry(first=10)], ws=2 * (stream_bytes + scores_bytes) - 1) == -3
    # window_end's own checks come first
    assert end([entry(ind=50, len=50)]) == -1 and b"ind + T" in lib.ct3_last_error()
    assert end([entry(tracks=p.value, visibility=None)]) == -1 and b"visibility" in lib.ct3_last_error()
    assert end([entry()], N=11) == -1 and b"tile" in lib.ct3_last_error()
    assert end([entry(vis=None)]) == -1


def test_return_scores_defaults_to_false():
    from cotracker_b200.predictor import CoTrackerOnlinePredictor, CoTrackerPredictor
    from cotracker_b200.streams import OnlineStreams
    for fn in (CoTrackerPredictor.forward, CoTrackerOnlinePredictor.forward, OnlineStreams.step):
        assert inspect.signature(fn).parameters["return_scores"].default is False, fn


@pytest.mark.parametrize("bad", [1, 0, None, "yes", torch.tensor(True)])
def test_return_scores_must_be_a_bool_before_any_device_work(bad):
    """A wrong value raises ValueError on a CPU model: the check runs before anything reaches the device (which would
    raise EngineError here)."""
    from cotracker_b200.predictor import CoTrackerOnlinePredictor, CoTrackerPredictor
    from cotracker_b200.streams import OnlineStreams
    p = CoTrackerPredictor(checkpoint=None, window_len=8)
    clip = torch.zeros(1, 4, 3, 64, 64, dtype=torch.uint8)
    with pytest.raises(ValueError, match="return_scores"):
        p(clip, grid_size=3, return_scores=bad)
    with pytest.raises(ValueError, match="return_scores"):
        p([clip, clip], grid_size=3, return_scores=bad)
    with pytest.raises(ValueError, match="return_scores"):
        p(clip, return_scores=bad)                                        # dense mode
    op = CoTrackerOnlinePredictor(checkpoint=None, window_len=4)
    with pytest.raises(ValueError, match="return_scores"):
        op(video_chunk=clip, is_first_step=True, grid_size=2, return_scores=bad)
    with pytest.raises(ValueError, match="return_scores"):
        OnlineStreams(op).step(return_scores=bad)


def test_first_online_step_keeps_the_arity():
    from cotracker_b200.predictor import CoTrackerOnlinePredictor
    op = CoTrackerOnlinePredictor(checkpoint=None, window_len=4)
    clip = torch.zeros(1, 4, 3, 64, 64, dtype=torch.uint8)
    assert op(video_chunk=clip, is_first_step=True, grid_size=2) == (None, None)
    assert op(video_chunk=clip, is_first_step=True, grid_size=2, return_scores=True) == (None, None, None)


def test_an_empty_hub_step_returns_nothing_with_scores():
    from cotracker_b200.predictor import CoTrackerOnlinePredictor
    from cotracker_b200.streams import OnlineStreams
    assert OnlineStreams(CoTrackerOnlinePredictor(checkpoint=None, window_len=4)).step(return_scores=True) == {}


def test_track_scores_exports():
    import cotracker_b200
    from cotracker_b200.predictor import TrackScores
    assert cotracker_b200.TrackScores is TrackScores
    assert TrackScores._fields == ("visibility", "confidence")
    spec = importlib.util.spec_from_file_location("dropin_predictor",
                                                  os.path.join(ROOT, "dropin", "cotracker", "predictor.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    assert mod.TrackScores is TrackScores


def test_finish_tracks_wrapper_needs_the_confidence_with_scores():
    z = torch.zeros(1, 2, 3)
    with pytest.raises(engine.EngineError, match="confidence"):
        engine.finish_tracks((torch.zeros(1, 2, 3, 2), z), None, torch.zeros(1, 3, 3), 3, 0.9, (1, 1), scores=True)
