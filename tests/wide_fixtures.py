"""The 512-wide decoder fixtures, built from committed data and fixed seeds instead of stored weights (8 x 512 floats
are 7 MB).

* decoder_wide: DeepSDF's own network -- 8 hidden layers of 512, latent_in = [4], weight-norm, a 64-long code -- whose
  first 256 units of every layer are the fitted 8 x 256 car decoder (decoder_cars.npz) and whose other units have
  seeded random weights.  The new units read every unit of the layer below and feed every unit of the layer above
  (scale ALPHA against the core's own weights), so each of the 512 columns enters the SDF and its Jacobian, while the
  zero level set of the car decoder survives (the reference's joint run on it succeeds).
* decoder_wide_variant: a 512-wide decoder with LayerNorm and xyz_in_all, two hidden layers, seeded random weights.

Both are plain state dicts in the fixture format (npz with spec_json), so they go through DecoderWeights.from_npz like
the committed ones.  tests/golden/make_wide_golden.py built the reference's goldens from exactly these weights and
stored their digest beside them (wide_stages.npz / wide_variant.npz: weights_sha256), which the tests check.  The
construction is numpy only, with correctly rounded row norms, so it does not depend on a summation order.
"""
import hashlib
import json
import math
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
WIDTH = 512
ALPHA = 0.2          # the new units' share of a core unit's input, relative to 1/sqrt(fan-in)
SEED_WIDE, SEED_VARIANT = 512, 513


def _rownorm(A):
    """|row| of a float64 matrix, each sum of squares correctly rounded (math.fsum): no summation order to differ."""
    return np.array([[math.sqrt(math.fsum(np.square(r)))] for r in A])


def _wn(W):
    """weight-norm parameters (g, v) of a folded matrix: v = W, g = |W| per row (fold: g v / |v|)."""
    v = W.astype(np.float32)
    return _rownorm(v.astype(np.float64)).astype(np.float32), v


def wide_state_dict():
    """(spec, state dict) of decoder_wide."""
    d = np.load(os.path.join(GOLDEN, "decoder_cars.npz"))
    spec = json.loads(bytes(d["spec_json"]).decode())
    spec["dims"] = [WIDTH] * 8
    rng = np.random.default_rng(SEED_WIDE)
    L3 = 64 + 3
    sd = {}
    for k in range(9):
        if k < 8:
            v = d[f"lin{k}.weight_v"].astype(np.float64)
            Wc = d[f"lin{k}.weight_g"].astype(np.float64) * v / _rownorm(v)
        else:
            Wc = d["lin8.weight"].astype(np.float64)
        bc = d[f"lin{k}.bias"].astype(np.float64)
        n_out = 1 if k == 8 else (WIDTH - L3 if k == 3 else WIDTH)
        n_in = L3 if k == 0 else WIDTH
        # columns of the car layer in the wide one: layer 4 reads [layer-3 units | decoder input]
        cols = np.arange(Wc.shape[1])
        if k == 4:
            cols = np.where(cols < 256 - L3, cols, WIDTH - L3 + (cols - (256 - L3)))
        W = rng.standard_normal((n_out, n_in)) * (np.sqrt(2.0 / n_in))
        core_rows = Wc.shape[0]
        W[:core_rows] *= ALPHA                  # a core unit: the car weights, plus ALPHA from the new units below
        W[:core_rows, cols] = Wc
        b = np.zeros(n_out)
        b[:core_rows] = bc
        b[core_rows:] = 0.01 * rng.standard_normal(n_out - core_rows)
        if k < 8:
            sd[f"lin{k}.weight_g"], sd[f"lin{k}.weight_v"] = _wn(W)
        else:
            sd["lin8.weight"] = W.astype(np.float32)
        sd[f"lin{k}.bias"] = b.astype(np.float32)
    return spec, sd


def wide_variant_state_dict():
    """(spec, state dict) of decoder_wide_variant: dims [512, 512], LayerNorm after both hidden layers, xyz_in_all."""
    spec = dict(latent_size=64, dims=[WIDTH, WIDTH], dropout=None, dropout_prob=0.0, norm_layers=[0, 1], latent_in=[],
                weight_norm=False, xyz_in_all=True, use_tanh=False, latent_dropout=False)
    rng = np.random.default_rng(SEED_VARIANT)
    sd = {}
    for k, (n_in, n_out) in enumerate([(67, WIDTH - 3), (WIDTH, WIDTH - 3), (WIDTH, 1)]):
        scale = np.sqrt(2.0 / n_in) if k < 2 else 0.15 / np.sqrt(n_in)
        sd[f"lin{k}.weight"] = (rng.standard_normal((n_out, n_in)) * scale).astype(np.float32)
        sd[f"lin{k}.bias"] = (0.05 * rng.standard_normal(n_out)).astype(np.float32)
        if k < 2:
            sd[f"bn{k}.weight"] = (1.0 + 0.3 * rng.standard_normal(n_out)).astype(np.float32)
            sd[f"bn{k}.bias"] = (0.2 * rng.standard_normal(n_out)).astype(np.float32)
    return spec, sd


BUILDERS = {"wide": wide_state_dict, "wide_variant": wide_variant_state_dict}


def digest(sd):
    """sha256 over the state dict's arrays in key order (stored with the goldens made from them)."""
    h = hashlib.sha256()
    for k in sorted(sd):
        h.update(k.encode()); h.update(np.ascontiguousarray(sd[k]).tobytes())
    return h.hexdigest()


def write(name, directory):
    """Writes decoder_<name>.npz into directory (fixture format) and returns its path."""
    spec, sd = BUILDERS[name]()
    path = os.path.join(directory, f"decoder_{name}.npz")
    np.savez(path, spec_json=np.frombuffer(json.dumps(spec).encode(), dtype=np.uint8), **sd)
    return path
