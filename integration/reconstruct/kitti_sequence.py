"""One-file replacement of DSP-SLAM's `reconstruct/kitti_sequence.py` whose detections are built on the H100.

Copy this file over `reconstruct/kitti_sequence.py` in a DSP-SLAM checkout (with `dsp_slam_b200/` on PYTHONPATH, as for
the optimizer).  The Tracking thread keeps calling `get_frame_by_id(frame_id)` (src/Tracking_util.cc:35) and reading
the same attributes; files, calibration and detectors are read as before.
"""
from dsp_slam_b200.lidar_frame import KITIISequence  # noqa: F401

__all__ = ["KITIISequence"]
