from cotracker_b200.predictor import CoTrackerOnlinePredictor, CoTrackerPredictor, TrackScores  # noqa: F401
