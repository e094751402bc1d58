from cotracker_b200.predictor import CoTrackerOnlinePredictor, CoTrackerPredictor, EncodedClip, TrackScores  # noqa: F401
