from cotracker_b200.visualizer import Visualizer, read_video_from_path  # noqa: F401
