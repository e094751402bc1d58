"""torch.hub entry points -- same names as the reference's hubconf.py:104-119.

    torch.hub.load("<this repo>", "cotracker3_offline", source="local", pretrained=False)

`pretrained=True` downloads the released CoTracker3 checkpoints (same URLs as the reference) and loads them
with strict=True; the CoTracker2 entry points are outside the H100 hot path and raise NotImplementedError.
"""
import torch

dependencies = ["torch"]

_COTRACKER3_SCALED_OFFLINE_URL = "https://huggingface.co/facebook/cotracker3/resolve/main/scaled_offline.pth"
_COTRACKER3_SCALED_ONLINE_URL = "https://huggingface.co/facebook/cotracker3/resolve/main/scaled_online.pth"


def _make(online: bool, pretrained: bool):
    from cotracker_b200.predictor import CoTrackerOnlinePredictor, CoTrackerPredictor

    if online:
        predictor = CoTrackerOnlinePredictor(checkpoint=None, window_len=16, v2=False)
        url = _COTRACKER3_SCALED_ONLINE_URL
    else:
        predictor = CoTrackerPredictor(checkpoint=None, window_len=60, v2=False)
        url = _COTRACKER3_SCALED_OFFLINE_URL
    if pretrained:
        state_dict = torch.hub.load_state_dict_from_url(url, map_location="cpu")
        predictor.model.load_state_dict(state_dict)
    return predictor


def cotracker3_offline(*, pretrained: bool = True, **kwargs):
    """Scaled offline CoTracker3 (stride 4, whole clip as one window of up to 60 time embeddings)."""
    return _make(online=False, pretrained=pretrained)


def cotracker3_online(*, pretrained: bool = True, **kwargs):
    """Scaled online CoTracker3 (stride 4, sliding window of 16 frames, step 8)."""
    return _make(online=True, pretrained=pretrained)


def _v2(*args, **kwargs):
    raise NotImplementedError("CoTracker2 entry points are not provided by the H100 hot-path build")


cotracker2 = cotracker2_online = cotracker2v1 = cotracker2v1_online = _v2
