"""Long rays (num_depth_samples > 64) without a GPU: the oracle against the reference's long-ray goldens
(tests/golden/make_long_ray_golden.py), a host model of the 8-bit first-sample field of the valid-sample range words
(dspgn_common.cuh: kRangeSampleBits; written by valid_sample_ranges, read by ray_sample_row, scan_chunk and mega_rows),
and the accepted range of dspgn_solver_create."""
import copy
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import valid_ranges_model as VR  # noqa: E402

BITS = 8                       # kRangeSampleBits
LONG_RUNS = [(128, "recon_long128"), (256, "recon_long256")]


def rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


@pytest.mark.parametrize("D,name", LONG_RUNS)
def test_oracle_whole_runs_vs_long_ray_goldens(oracle, oracle_decoders, cfg_kitti, golden_dir, D, name):
    """At the tolerances of test_oracle_vs_golden.test_whole_runs for recon_kitti250 (same object, same config but D):
    iteration 0 tight, the end state to the noise floor of a 10-iteration run with the render term."""
    d = np.load(os.path.join(golden_dir, name + ".npz"))
    assert int(d["num_depth_samples"]) == D
    cfg = copy.deepcopy(cfg_kitti)
    cfg["optimizer"]["num_depth_samples"] = D
    ocfg = oracle.GNConfig.from_json_dict(cfg)
    ocfg.num_iterations = 10
    trace = []
    out = oracle.reconstruct_object(oracle_decoders["cars"], ocfg, d["in_t_cam_obj"], d["in_pts"], d["in_rays"],
                                    d["in_depth"], trace=trace)
    assert out["is_good"] and bool(d["is_good"])
    assert trace[0]["V"] == int(d["V_iters"][0]) and trace[0]["m"] == int(d["m_iters"][0])
    assert rel(trace[0]["H"], d["H_iters"][0]) < 5e-5
    assert rel(trace[0]["b"], d["b_iters"][0]) < 5e-5
    assert np.abs(trace[0]["dx"] - d["dx_iters"][0]).max() < 1e-4
    assert np.abs(out["t_cam_obj"] - d["t_cam_obj"]).max() < 3e-2
    assert np.abs(out["code"] - d["code"]).max() < 1.5e-2
    assert abs(float(out["loss"]) - float(d["loss"])) < 0.05 * abs(float(d["loss"])) + 1e-5


# ---- range words ------------------------------------------------------------------------------------------------------
def pack(first, cnt, bits=BITS):
    """valid_sample_ranges' words: (exclusive prefix of the hull lengths << bits) | first sample, then total << bits."""
    pre = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
    w = (pre[:-1] << bits) | first
    assert pre[-1] << bits < 2 ** 31                        # an int32 word
    return np.concatenate([w, [pre[-1] << bits]]).astype(np.int32)


def decode(words, rows, bits=BITS):
    """ray_sample_row on compact rows: the largest ray whose hull starts at or before the row (its bisection over the
    prefixes, vectorised), and the row's sample."""
    n_rays = len(words) - 1
    pre = words[:n_rays] >> bits
    ray = np.clip(np.searchsorted(pre, rows, side="right") - 1, 0, n_rays - 1)
    return ray, (words[ray] & ((1 << bits) - 1)) + (rows - pre[ray])


def bisect(words, row, bits=BITS):
    """ray_sample_row's loop, literally."""
    lo, hi = 0, len(words) - 1
    while hi - lo > 1:
        mid = (lo + hi) >> 1
        if (int(words[mid]) >> bits) <= row:
            lo = mid
        else:
            hi = mid
    return lo, (int(words[lo]) & ((1 << bits) - 1)) + (row - (int(words[lo]) >> bits))


def hulls(rng, D, n_rays):
    """Hulls [first, first + cnt) of every kind the words must carry: empty, the whole ray, one sample at each end, random."""
    first = rng.integers(0, D, n_rays)
    cnt = np.array([rng.integers(0, D - f + 1) for f in first])
    k = np.arange(n_rays) % 8
    first[k == 0], cnt[k == 0] = 0, 0
    first[k == 1], cnt[k == 1] = 0, D
    first[k == 2], cnt[k == 2] = D - 1, 1
    first[k == 3], cnt[k == 3] = 0, 1
    return first, cnt


@pytest.mark.parametrize("D", [65, 128, 255, 256])
def test_range_words_carry_every_hull(D):
    """Every compact row decodes to its own (ray, sample) with the 8-bit field, at the largest ray count at D = 256
    (8192 rays, n_rays x D = 2^21 rows: the prefix field's bound); the 7-bit field of D <= 64 would not hold these hulls.
    The windowed hull search of the pre-pass also equals the exhaustive one at this D."""
    rng = np.random.default_rng(D)
    n_rays = 8192 if D == 256 else 600
    first, cnt = hulls(rng, D, n_rays)
    words = pack(first, cnt)
    rows = np.arange(int(cnt.sum()))
    want_ray = np.repeat(np.arange(n_rays), cnt)
    want_j = np.concatenate([np.arange(f, f + c) for f, c in zip(first, cnt)])
    ray, j = decode(words, rows)
    np.testing.assert_array_equal(ray, want_ray)
    np.testing.assert_array_equal(j, want_j)
    for r in rng.choice(rows, 300, replace=False):
        assert bisect(words, int(r)) == (want_ray[r], want_j[r])
    assert int(words[-1]) >> BITS == len(rows)              # mega_rows: the object's row count
    if D > 128:
        _, j7 = decode(pack(first, cnt, bits=7), rows, bits=7)
        assert not np.array_equal(j7, want_j)
    bad, nonempty, _ = VR.run(300, seed=D, D=D)
    assert bad == 0 and nonempty > 50


# ---- accepted range ---------------------------------------------------------------------------------------------------
def test_solver_create_accepts_256_depth_samples_and_refuses_257():
    """The argument checks of dspgn_solver_create run before any CUDA call or decoder access.  D = 257 is refused with a
    message naming the range; D = 256 passes that check (the call then fails on the next one, num_iterations = 0)."""
    from dsp_slam_b200 import _lib
    lib = _lib.load()
    classes = (C.c_void_p * 1)(C.c_void_p(8))                # never dereferenced: the checks below fail first
    out = C.c_void_p(0)

    def create(D, iters):
        cfg = _lib.Config(num_iterations=iters, code_len=64, num_depth_samples=D, cut_off=0.01)
        rc = lib.dspgn_solver_create(C.byref(cfg), classes, 1, 0, C.byref(out))
        return rc, lib.dspgn_last_error().decode()

    for D in (1, 257, 1024):
        assert create(D, 1) == (_lib.E_ARG, "num_depth_samples must be in [2,256]"), D
    for D in (2, 65, 128, 256):
        assert create(D, 0) == (_lib.E_ARG, "num_iterations must be >= 1"), D
    assert not out.value
