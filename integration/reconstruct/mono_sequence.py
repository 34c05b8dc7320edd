"""One-file replacement of DSP-SLAM's `reconstruct/mono_sequence.py` whose detection is built on the H100.

Copy this file over `reconstruct/mono_sequence.py` in a DSP-SLAM checkout (with `dsp_slam_b200/` on PYTHONPATH, as for
the optimizer).  The Tracking thread keeps calling `get_frame_by_id(frame_id)` (src/Tracking_util.cc:166) and reading
the same attributes; the yaml, images, labels and detector are read as before.
"""
from dsp_slam_b200.mono_frame import MonoSequence  # noqa: F401

__all__ = ["MonoSequence"]
