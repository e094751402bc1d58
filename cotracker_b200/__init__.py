"""cotracker_b200 -- H100-native (sm_90a) implementation of CoTracker3's iterative update loop behind the
reference's `cotracker.predictor` API.  See DESIGN.md and include/ct3_b200.h."""
from .build import build_cotracker  # noqa: F401
from .corners import detect_corners  # noqa: F401
from .ingest import Crop, YUVClip  # noqa: F401
from .predictor import CoTrackerOnlinePredictor, CoTrackerPredictor, EncodedClip, TrackScores  # noqa: F401
from .streams import OnlineStreams  # noqa: F401

__version__ = "0.1.0"
