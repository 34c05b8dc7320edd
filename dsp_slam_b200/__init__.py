"""dsp_slam_b200: DSP-SLAM's per-object shape-prior Gauss-Newton reconstruction, H100-native.

Public surface (mirrors reconstruct/optimizer.py of the reference):
    from dsp_slam_b200.optimizer import Optimizer, MeshExtractor
The CUDA library (libdspgn.so, C ABI in include/dspgn.h) is loaded lazily on first use.
"""
import json as _json
import os as _os

__all__ = ["load_config", "CONFIG_DIR"]

CONFIG_DIR = _os.path.join(_os.path.dirname(_os.path.abspath(__file__)), "configs")


def load_config(name):
    """Load one of the bundled optimiser configs ('config_kitti.json', 'config_redwood_01053.json')."""
    with open(_os.path.join(CONFIG_DIR, name)) as f:
        return _json.load(f)
