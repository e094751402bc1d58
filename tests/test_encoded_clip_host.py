"""CPU tests of `EncodedClip`: the checks a predictor makes on a clip before any work and the TypeErrors of every entry
point that takes pixels, on a clip built without a device, and the ABI surface of `ct3_pyramid_pools` with its
rejections before any launch."""
import ctypes
import os
import re

import pytest
import torch

from cotracker_b200 import EncodedClip, detect_corners, engine
from cotracker_b200.evaluation import EvaluationPredictor
from cotracker_b200.predictor import CoTrackerOnlinePredictor, CoTrackerPredictor, _EncodedClip, _loop
from cotracker_b200.streams import OnlineStreams
from cotracker_b200.visualizer import Visualizer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _clip(p, B=1, T=8, H=96, W=128, **kw):
    """An EncodedClip as `p.encode` records it, on the model's device, without a pyramid or a device."""
    c = EncodedClip.__new__(EncodedClip)
    c.model, c.device, c.weights = p.model, torch.device("cpu"), p.model.weights_fingerprint()
    c.video_shape, c.B, c.T = torch.Size((B, T, 3, H, W)), B, T
    c.H, c.W = p.interp_shape
    c.interp_shape, c.stride, c.loop, c.pad = tuple(p.interp_shape), p.model.stride, _loop(p.model), 0
    c.host, c.pyr = None, torch.zeros(1)
    for k, v in kw.items():
        setattr(c, k, v)
    return c


@pytest.fixture(scope="module")
def predictor():
    return CoTrackerPredictor(checkpoint=None)


def test_public_names(predictor):
    import sys
    sys.path.insert(0, os.path.join(ROOT, "dropin"))
    from cotracker.predictor import EncodedClip as dropin_clip
    assert dropin_clip is EncodedClip and _EncodedClip is EncodedClip
    c = _clip(predictor, B=2, T=5, H=120, W=176)
    assert c.input_hw == (120, 176) and not c.parked and c.nbytes == 4
    assert "EncodedClip" in repr(c)


def test_predictor_checks_the_clip_before_any_work(predictor):
    p = predictor
    q = torch.zeros(1, 3, 3)
    cases = [
        (dict(pyr=None, device=torch.device("cpu")), "parked"),
        (dict(interp_shape=(192, 256)), "interp_shape"),
        (dict(stride=8), "stride"),
        (dict(loop="sliding-window (window_len 16)"), "sliding-window"),
        (dict(device=torch.device("cuda", 0)), "cuda:0"),
        (dict(weights="0" * 64), "weights"),
        (dict(weights=None), "weights"),
    ]
    for kw, msg in cases:
        with pytest.raises(ValueError, match=re.escape(msg)):
            p(_clip(p, **kw), queries=q)
    with pytest.raises(ValueError, match="B == 1"):
        p(_clip(p, B=2), grid_size=5, segm_mask=torch.ones(1, 1, 96, 128))
    with pytest.raises(ValueError, match="return_scores"):
        p(_clip(p), queries=q, return_scores=1)


def test_entry_points_that_take_pixels_reject_a_clip(predictor):
    p = predictor
    c = _clip(p)
    online = CoTrackerOnlinePredictor(checkpoint=None, window_len=16)
    calls = {
        "CoTrackerOnlinePredictor": lambda: online(c, is_first_step=True, grid_size=5),
        "OnlineStreams.push": lambda: OnlineStreams(online).push(0, c),
        "entry 0 of a list call": lambda: p([c], grid_size=5),
        "entry 1 of a list call": lambda: p([torch.zeros(1, 4, 3, 32, 32), c], grid_size=5),
        "EvaluationPredictor": lambda: EvaluationPredictor(p.model)(c, torch.zeros(1, 1, 3)),
        "detect_corners": lambda: detect_corners(c, 10),
        "Visualizer.visualize": lambda: Visualizer().visualize(c, torch.zeros(1, 8, 2, 2), save_video=False),
        "Visualizer.draw_tracks_on_video": lambda: Visualizer().draw_tracks_on_video(c, torch.zeros(1, 8, 2, 2)),
    }
    for where, call in calls.items():
        with pytest.raises(TypeError, match=re.escape(where) + ".*EncodedClip"):
            call()
    for bad in (c, [torch.zeros(1, 4, 3, 32, 32)], (c,)):
        with pytest.raises(TypeError, match="encode takes one clip"):
            p.encode(bad)
    with pytest.raises(ValueError, match="not meta"):
        c.to("meta")
    c.pyr = None   # parked: parking again is a no-op
    assert c.to("cpu") is c and c.parked and c.nbytes == 0


def test_pyramid_pools_exported_and_declared():
    lib = engine.lib()
    with open(os.path.join(ROOT, "include", "ct3_b200.h")) as f:
        header = f.read()
    assert re.search(r"int ct3_pyramid_pools\(int T, int H4, int W4, float\* pyr, ct3_stream_t stream\);", header)
    assert hasattr(lib, "ct3_pyramid_pools") and "ct3_pyramid_pools" in engine.EXPORTED_SYMBOLS
    assert lib.ct3_version() == 102


def test_pyramid_pools_rejects_bad_arguments_in_the_library():
    """Each invalid argument returns CT3_EINVAL with a message before any launch (a fake pointer and the legacy stream:
    reaching a launch would fail differently)."""
    lib = engine.lib()
    pyr = ctypes.c_void_p(1 << 24)
    cases = [
        (dict(pyr=None), b"null argument"), (dict(T=0), b"bad pyramid shape"), (dict(H4=0), b"bad pyramid shape"),
        (dict(W4=-3), b"bad pyramid shape"), (dict(H4=7), b"feature map too small"), (dict(W4=4), b"too small"),
    ]
    for kw, msg in cases:
        a = dict(dict(T=4, H4=96, W4=128, pyr=pyr), **kw)
        assert lib.ct3_pyramid_pools(a["T"], a["H4"], a["W4"], a["pyr"], None) == -1, kw
        assert msg in lib.ct3_last_error(), (kw, lib.ct3_last_error())


def test_pyramid_pools_binding_checks_its_tensor():
    with pytest.raises(engine.EngineError, match="CUDA tensor"):
        engine.pyramid_pools(torch.zeros(16), 1, 8, 8)
