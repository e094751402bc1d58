"""Model factory -- mirror of the reference's cotracker/models/build_cotracker.py:26-45.

Same signature and checkpoint handling (flat state dict or {"model": ...}); `v2=True` (CoTracker2) is
outside the north-star path and raises NotImplementedError.
"""
from __future__ import annotations

import torch

from .model import CoTrackerThreeOffline, CoTrackerThreeOnline


def build_cotracker(checkpoint=None, offline=True, window_len=16, v2=False):
    if v2:
        raise NotImplementedError("CoTracker2 is not part of the H100 hot path (SURVEY.md §2, row 3b)")
    cls = CoTrackerThreeOffline if offline else CoTrackerThreeOnline
    cotracker = cls(stride=4, corr_radius=3, window_len=window_len)
    if checkpoint is not None:
        with open(checkpoint, "rb") as f:
            state_dict = torch.load(f, map_location="cpu")
        if "model" in state_dict:
            state_dict = state_dict["model"]
        cotracker.load_state_dict(state_dict)
    return cotracker
