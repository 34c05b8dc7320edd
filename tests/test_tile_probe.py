"""The tile probe build (tools/tile_probe.py): the cycle counters exist only in a library compiled with
-DDSPGN_STALL_PROBE.  The shipped library exports no probe entry point; the probe build compiles and exports one."""
import ctypes
import os
import shutil
import subprocess

import pytest

import __graft_entry__ as g
from dsp_slam_b200 import _lib


def test_shipped_library_has_no_probe():
    assert not hasattr(ctypes.CDLL(_lib.LIB_PATH), "dspgn_debug_stall_probe")


def test_probe_build_compiles(tmp_path):
    nvcc = os.environ.get("NVCC", "nvcc")
    if shutil.which(nvcc) is None:
        pytest.skip("nvcc is not available")
    lib = str(tmp_path / "libdspgn_probe.so")
    subprocess.run([nvcc] + g.NVCC_FLAGS + ["-DDSPGN_STALL_PROBE", "-o", lib, os.path.join(g.CSRC, "dspgn_api.cu")],
                   cwd=g.CSRC, check=True, capture_output=True, timeout=900)
    assert hasattr(ctypes.CDLL(lib), "dspgn_debug_stall_probe")
