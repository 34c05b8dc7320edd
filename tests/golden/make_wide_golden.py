"""Generate the goldens of the 512-wide decoders (tests/wide_fixtures.py) by running the UNMODIFIED reference
(PyTorch-CPU, via tools/ref_harness.py), in the authoring container only:

    python tests/golden/make_wide_golden.py

Writes, for decoder_wide (DeepSDF's 8 x 512 network with a 64-long code):
  wide_stages.npz    forward, input Jacobian, SDF-term rows and render band rows at one state
  recon_wide.npz     a whole joint run with the render term on the KITTI hyper-parameters (the shape of
                     recon_kitti250.npz), with H, b, dx, V, m of every iteration
  states_wide.npz    the reference's state at every iteration of that run (teacher-forced tests); a second run of the
                     reference must reproduce recon_wide bit for bit
  pose_only_wide.npz a pose-only run (estimate_pose_cam_obj)
and for decoder_wide_variant (LayerNorm + xyz_in_all at width 512): wide_variant.npz, its stages.  Each stage file
carries weights_sha256, the digest of the weights it was made from.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden as MG  # noqa: E402
import wide_fixtures as WF  # noqa: E402

ns, synth = MG.ns, MG.synth


def ref_decoder(name):
    spec, sd = WF.BUILDERS[name]()
    dec = ns.decoder.Decoder(**spec)
    dec.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    return dec.eval(), WF.digest(sd)


def stages(dec, obj, z):
    """What make_golden.main records as stages.npz, for decoder dec: object obj (100 foreground + 20 background rays)
    at code z."""
    lu, lo = ns.loss_utils, ns.loss
    st = {}
    t_oc = torch.inverse(torch.from_numpy(np.array(obj["t_cam_obj_init"])))
    pts = torch.from_numpy(np.ascontiguousarray(obj["pts"]))
    x_obj = (pts[..., None, :] * t_oc[:3, :3]).sum(-1) + t_oc[:3, 3]
    inp = torch.cat([z.expand(x_obj.shape[0], -1), x_obj], 1)
    with torch.no_grad():
        st["dec_in"] = inp.numpy().copy()
        st["dec_y"] = dec(inp).squeeze(-1).numpy().copy()
    y, g = lu.get_batch_sdf_jacobian(dec, z, x_obj, 1)
    st["jac_y"] = y.reshape(-1).numpy().copy()
    st["jac_g"] = g.reshape(-1, 67).numpy().copy()
    jt, jc, res = lo.compute_sdf_loss(dec, pts, t_oc, z)
    st["sdf_t_obj_cam"] = t_oc.numpy().copy()
    st["sdf_z"] = z.numpy().copy()
    st["sdf_pts"] = pts.numpy().copy()
    st["sdf_J"] = torch.cat([jt, jc], -1).reshape(-1, 71).numpy().copy()
    st["sdf_res"] = res.reshape(-1).numpy().copy()
    t_co = torch.inverse(t_oc)
    scale = torch.det(t_co[:3, :3]) ** (1 / 3)
    dmin, dmax = t_co[2, 3] - scale, t_co[2, 3] + scale
    depths = torch.linspace(dmin, dmax, 50)
    rays = torch.from_numpy(np.ascontiguousarray(obj["rays"]))
    dobs = torch.cat([torch.from_numpy(np.array(obj["depth"])), torch.full((20,), float(1.1 * dmax))])
    dobs[100:] = 1.1 * dmax
    rr = lo.compute_render_loss(dec, rays, dobs, t_oc, depths, z, th=0.01)
    st["rnd_rays"] = rays.numpy().copy()
    st["rnd_depth_obs"] = dobs.numpy().copy()
    st["rnd_depths"] = depths.numpy().copy()
    st["rnd_J"] = torch.cat([rr[0], rr[1]], -1).reshape(-1, 71).numpy().copy()
    st["rnd_res"] = rr[2].reshape(-1).numpy().copy()
    return st


def main():
    rng = np.random.default_rng(17)
    wide, h = ref_decoder("wide")
    st = stages(wide, synth.make_object(23, 300, 100, 20), torch.from_numpy((0.05 * rng.standard_normal(64)).astype(np.float32)))
    np.savez_compressed(os.path.join(HERE, "wide_stages.npz"), weights_sha256=np.array(h), **st)
    print("wide_stages.npz:", st["sdf_J"].shape, st["rnd_J"].shape)
    cfgk = MG.cfg_with("config_kitti.json")
    o = synth.make_object(1, 250, 250, 200)
    states = {}
    r = MG.run_reconstruct(wide, cfgk, o, states=states)
    again = MG.run_reconstruct(wide, cfgk, o)
    for k in ("H_iters", "b_iters", "dx_iters", "V_iters", "m_iters", "t_cam_obj", "code", "loss"):
        assert np.array_equal(r[k], again[k]), k
    np.savez_compressed(os.path.join(HERE, "recon_wide.npz"), **MG.pack_inputs(o), **r)
    np.savez_compressed(os.path.join(HERE, "states_wide.npz"), **states)
    print("recon_wide.npz: V", r["V_iters"].tolist(), "m", r["m_iters"].tolist())
    o = synth.make_object(6, 250, 0, 0)
    T = np.array(o["t_cam_obj_init"], dtype=np.float32)
    s = float(np.cbrt(np.linalg.det(T[:3, :3].astype(np.float64))))
    se3 = T.copy(); se3[:3, :3] /= s
    code = (0.8 * o["code_gt"]).astype(np.float32)
    Tout = ns.optimizer.Optimizer(wide, cfgk).estimate_pose_cam_obj(se3.copy(), s, MG.np_f(o["pts"]), code.copy())
    np.savez_compressed(os.path.join(HERE, "pose_only_wide.npz"), in_t_co_se3=se3, in_scale=np.array(s, dtype=np.float32),
                        in_pts=o["pts"], in_code=code, t_cam_obj=Tout.numpy())
    variant, h = ref_decoder("wide_variant")
    st = stages(variant, synth.make_object(29, 200, 100, 20), torch.from_numpy((0.3 * rng.standard_normal(64)).astype(np.float32)))
    np.savez_compressed(os.path.join(HERE, "wide_variant.npz"), weights_sha256=np.array(h), **st)
    print("wide_variant.npz: sdf range", float(st["dec_y"].min()), float(st["dec_y"].max()), "band rows", st["rnd_J"].shape[0])


if __name__ == "__main__":
    main()
