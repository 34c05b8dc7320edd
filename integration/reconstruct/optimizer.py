"""One-file replacement of DSP-SLAM's `reconstruct/optimizer.py` (222 lines of PyTorch) by the H100 path.

Copy this file over `reconstruct/optimizer.py` in a DSP-SLAM checkout and put `dsp_slam_b200/` (with the built
`libdspgn.so`) on PYTHONPATH.  The C++ side is untouched: it keeps importing `reconstruct.optimizer`
(src/LocalMapping.cc:38) and calling `Optimizer(decoder, configs)`, `.reconstruct_object(...)`,
`.estimate_pose_cam_obj(...)`, `.code_len` and `MeshExtractor(decoder, code_len, voxels_dim)
.extract_mesh_from_code(code)` (src/LocalMapping.cc:39-40, src/LocalMapping_util.cc:109-110,179-196,390-428).
Everything else of the `reconstruct` package (utils, sequences, detectors) stays the reference's.
"""
from dsp_slam_b200.optimizer import Optimizer, MeshExtractor  # noqa: F401

__all__ = ["Optimizer", "MeshExtractor"]
