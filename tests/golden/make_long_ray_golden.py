"""Generate the goldens of long rays (num_depth_samples > 64) by running the UNMODIFIED reference (PyTorch-CPU, via
tools/ref_harness.py), in the authoring container only:

    python tests/golden/make_long_ray_golden.py

For D = 128 and D = 256, on the fitted cars decoder, a KITTI-shaped object (250 points, 250 + 200 rays: the shape of
recon_kitti250.npz) and the shipped config_kitti.json values otherwise, writes
  recon_long<D>.npz   a whole joint run with H, b, dx, V, m of every iteration (make_golden.run_reconstruct) and
                      num_depth_samples; a second run of the reference must reproduce it bit for bit
  states_long<D>.npz  the reference's state at every iteration of that run (teacher-forced tests)
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as MG  # noqa: E402

synth = MG.synth
DEPTH_SAMPLES = (128, 256)


def main():
    cars = MG.load_ref_decoder("cars")
    o = synth.make_object(1, 250, 250, 200)
    for D in DEPTH_SAMPLES:
        cfg = MG.cfg_with("config_kitti.json")
        cfg.optimizer.num_depth_samples = D
        states = {}
        r = MG.run_reconstruct(cars, cfg, o, states=states)
        again = MG.run_reconstruct(cars, cfg, o)
        for k in ("H_iters", "b_iters", "dx_iters", "V_iters", "m_iters", "t_cam_obj", "code", "loss"):
            assert np.array_equal(r[k], again[k]), k
        np.savez_compressed(os.path.join(HERE, f"recon_long{D}.npz"), **MG.pack_inputs(o), **r,
                            num_depth_samples=np.array(D))
        np.savez_compressed(os.path.join(HERE, f"states_long{D}.npz"), **states)
        print(f"recon_long{D}.npz: V", r["V_iters"].tolist(), "m", r["m_iters"].tolist())


if __name__ == "__main__":
    main()
