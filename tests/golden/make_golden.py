"""Generate the golden vectors under tests/golden/ by running the UNMODIFIED reference
(/root/reference, PyTorch-CPU, via tools/ref_harness.py) on seeded synthetic inputs.

The reference has no tests or golden vectors of its own (SURVEY.md s4), and it cannot travel to
the GPU box, so these files are what pins the oracle (oracle/dsp_oracle.py) and, through it, the
CUDA path.  Run in the authoring container only:

    python tools/fit_fixture_decoder.py cars chairs      # once, ~5 min
    python tests/golden/make_golden.py

Writes stages.npz (single-stage inputs/outputs at a fixed state) and recon_*.npz (whole GN runs,
with the 71x71 system of every iteration captured by wrapping torch.mv).

    python tests/golden/make_golden.py --states

re-runs every whole-run golden from its stored inputs, asserts that the reference reproduces it bit for bit, and writes
states_*.npz (the reference's state at every iteration) and pose_only_cut.npz for the teacher-forced tests.
"""
import os
import sys
import json
import copy
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import ref_harness  # noqa: E402
from dsp_slam_b200 import synth  # noqa: E402

ns = ref_harness.load()
torch.set_num_threads(os.cpu_count())


def load_ref_decoder(name):
    d = np.load(os.path.join(HERE, f"decoder_{name}.npz"))
    spec = json.loads(bytes(d["spec_json"]).decode())
    dec = ns.decoder.Decoder(**spec)
    dec.load_state_dict({k: torch.from_numpy(d[k]) for k in d.files if k != "spec_json"})
    return dec.eval()


def cfg_with(name, **joint_overrides):
    cfg = ref_harness.load_config(name)
    for k, v in joint_overrides.items():
        cfg.optimizer.joint_optim[k] = v
    return cfg


class SolveRecorder:
    """Captures (H, b, dx) of every  dx = mv(inverse(H), b)  the reference performs."""

    def __enter__(self):
        self.H, self.b, self.dx = [], [], []
        self._inv, self._mv = torch.inverse, torch.mv
        rec = self

        def inv(a):
            r = rec._inv(a)
            if a.shape[0] > 4:
                rec.H.append(a.detach().clone().numpy())
            return r

        def mv(a, b):
            r = rec._mv(a, b)
            if a.shape[0] > 4:
                rec.b.append(b.detach().clone().numpy())
                rec.dx.append(r.detach().clone().numpy())
            return r

        torch.inverse, torch.mv = inv, mv
        return self

    def __exit__(self, *a):
        torch.inverse, torch.mv = self._inv, self._mv


class RenderRecorder:
    """Per-iteration counters of the render term, captured without touching the reference: V = number of
    query points handed to the no-grad decode_sdf inside compute_render_loss (loss.py:77-78), m = rows of
    the render Jacobian it returns (loss.py:143-150); -1 where the call returned None."""

    def __enter__(self):
        self.V, self.m = [], []
        self._crl = ns.optimizer.compute_render_loss
        self._dec = ns.loss.decode_sdf
        rec = self

        def dec(decoder, latent, pts, *a, **k):
            rec._lastV = int(pts.shape[0])
            return rec._dec(decoder, latent, pts, *a, **k)

        def crl(*a, **k):
            rec._lastV = -1
            r = rec._crl(*a, **k)
            rec.V.append(rec._lastV)
            rec.m.append(-1 if r is None else int(r[0].shape[0]))
            return r

        ns.loss.decode_sdf = dec
        ns.optimizer.compute_render_loss = crl
        return self

    def __exit__(self, *a):
        ns.loss.decode_sdf = self._dec
        ns.optimizer.compute_render_loss = self._crl


class StateRecorder:
    """The state the reference's loop starts each iteration from, captured without touching the reference: the
    t_obj_cam and latent_vector handed to compute_sdf_loss (optimizer.py:62-65,129; cloned, because the code is
    updated in place), the number of surface points, the SDF residuals, and the loss of every get_robust_res call
    (sdf then render in reconstruct_object, sdf only in estimate_pose_cam_obj)."""

    def __enter__(self):
        self.Toc, self.z, self.n_pts, self.res, self.losses = [], [], [], [], []
        self._csl = ns.optimizer.compute_sdf_loss
        self._grr = ns.optimizer.get_robust_res
        rec = self

        def csl(decoder, pts, t_obj_cam, latent, *a, **k):
            rec.Toc.append(t_obj_cam.detach().clone().numpy())
            rec.z.append(latent.detach().clone().numpy())
            rec.n_pts.append(int(pts.shape[0]))
            r = rec._csl(decoder, pts, t_obj_cam, latent, *a, **k)
            rec.res.append(None if r is None else r[2].detach().reshape(-1).clone().numpy())
            return r

        def grr(res, b, *a, **k):
            r = rec._grr(res, b, *a, **k)
            rec.losses.append(np.float32(r[1].item()))
            return r

        ns.optimizer.compute_sdf_loss = csl
        ns.optimizer.get_robust_res = grr
        return self

    def __exit__(self, *a):
        ns.optimizer.compute_sdf_loss = self._csl
        ns.optimizer.get_robust_res = self._grr


def np_f(x):
    return np.asfortranarray(np.array(x, dtype=np.float32))


def run_reconstruct(dec, cfg, obj, with_code=False, states=None):
    """One reference reconstruct_object run with its per-iteration systems.  With states={} the per-iteration
    state is also captured into that dict (StateRecorder), plus the final state after the last update."""
    opt = ns.optimizer.Optimizer(dec, cfg)
    code = None if not with_code else np.array(obj["code_init"], dtype=np.float32)
    with SolveRecorder() as rec, RenderRecorder() as rr, StateRecorder() as sr:
        out = opt.reconstruct_object(np_f(obj["t_cam_obj_init"]), np_f(obj["pts"]),
                                     np_f(obj["rays"]), np.array(obj["depth"], dtype=np.float32),
                                     code)
    if states is not None:
        n = len(rec.dx)
        assert out.is_good and len(sr.Toc) == n and len(sr.losses) == 2 * n
        # the update the reference applies after its last solve (optimizer.py:187-192), with its own functions
        dx = torch.from_numpy(rec.dx[-1])
        Toc_end = torch.mm(ns.loss_utils.exp_sim3(opt.lr * dx[:7]), torch.from_numpy(sr.Toc[-1]))
        assert np.array_equal(torch.inverse(Toc_end).numpy(), out.t_cam_obj)
        states.update(Toc_iters=np.stack(sr.Toc + [Toc_end.numpy()]),
                      z_iters=np.stack(sr.z + [np.asarray(out.code)]),
                      sdf_loss_iters=np.array(sr.losses[0::2], np.float32),
                      render_loss_iters=np.array(sr.losses[1::2], np.float32))
    res = dict(is_good=np.array(bool(out.is_good)), loss=np.array(float(out.loss), dtype=np.float32))
    if out.is_good:
        res["t_cam_obj"] = np.ascontiguousarray(out.t_cam_obj)
        res["code"] = np.ascontiguousarray(out.code)
    if rec.H:
        res["H_iters"] = np.stack(rec.H)
        res["b_iters"] = np.stack(rec.b)
        res["dx_iters"] = np.stack(rec.dx)
    res["V_iters"] = np.array(rr.V, dtype=np.int64)
    res["m_iters"] = np.array(rr.m, dtype=np.int64)
    return res


def pack_inputs(obj, with_code=False):
    d = dict(in_t_cam_obj=obj["t_cam_obj_init"], in_pts=obj["pts"], in_rays=obj["rays"],
             in_depth=obj["depth"], gt_t_cam_obj=obj["t_cam_obj_gt"], gt_code=obj["code_gt"])
    if with_code:
        d["in_code"] = obj["code_init"]
    return d


def sdf_only_composed(dec, cfg, obj, states=None):
    """optimizer.py:118-192 with the render block removed, built from the reference's own
    functions (BASELINE config 2 'surface-SDF loss' mode; SURVEY.md 8d).  states={} also captures
    the state of every iteration, as run_reconstruct does."""
    lu, lo = ns.loss_utils, ns.loss
    o = cfg.optimizer
    j = o.joint_optim
    L = o.code_len
    z = torch.zeros(L)
    t_obj_cam = torch.inverse(torch.from_numpy(np.array(obj["t_cam_obj_init"])))
    pts = torch.from_numpy(np.ascontiguousarray(obj["pts"]))
    Hs, bs, dxs = [], [], []
    Tocs, zs, sdf_losses = [], [], []
    loss = 0.0
    for _ in range(j.num_iterations):
        Tocs.append(t_obj_cam.clone().numpy()); zs.append(z.clone().numpy())
        jt, jc, res = lo.compute_sdf_loss(dec, pts, t_obj_cam, z)
        rr, sdf_loss, _ = lu.get_robust_res(res, j.b2)
        sdf_losses.append(np.float32(sdf_loss.item()))
        drot, res_rot = lo.compute_rotation_loss_sim3(t_obj_cam)
        loss = j.k2 * sdf_loss
        J = torch.cat([jt, jc], dim=-1)
        n = J.shape[0]
        H = j.k2 * torch.bmm(J.transpose(-2, -1), J).sum(0).squeeze() / n
        b = -j.k2 * torch.bmm(J.transpose(-2, -1), rr).sum(0).squeeze() / n
        H[7:7 + L, 7:7 + L] += j.k3 * torch.eye(L)
        b[7:7 + L] -= j.k3 * z
        drot = drot.unsqueeze(0)
        H[:7, :7] += j.k4 * torch.mm(drot.transpose(-2, -1), drot)
        b[:7] -= j.k4 * (-(drot.transpose(-2, -1) * res_rot).squeeze())
        H[:7, :7] += torch.eye(7)
        H[6, 6] += j.scale_damping
        dx = torch.mv(torch.inverse(H), b)
        Hs.append(H.clone().numpy()); bs.append(b.clone().numpy()); dxs.append(dx.clone().numpy())
        t_obj_cam = torch.mm(lu.exp_sim3(j.learning_rate * dx[:7]), t_obj_cam)
        z = z + j.learning_rate * dx[7:7 + L]
    if states is not None:
        states.update(Toc_iters=np.stack(Tocs + [t_obj_cam.numpy()]), z_iters=np.stack(zs + [z.numpy()]),
                      sdf_loss_iters=np.array(sdf_losses, np.float32),
                      render_loss_iters=np.zeros(len(sdf_losses), np.float32))
    return dict(t_cam_obj=torch.inverse(t_obj_cam).numpy(), code=z.numpy(),
                loss=np.array(float(loss), dtype=np.float32), is_good=np.array(True),
                H_iters=np.stack(Hs), b_iters=np.stack(bs), dx_iters=np.stack(dxs))


def main():
    cars = load_ref_decoder("cars")
    chairs = load_ref_decoder("chairs")
    lu, lo = ns.loss_utils, ns.loss
    rng = np.random.default_rng(7)

    # ------------------------------------------------------------------ single stages
    st = {}
    # folded weights as torch's own weight_norm hook computes them (checked against our fold)
    with torch.no_grad():
        cars(torch.zeros(1, 67))
    for k in range(9):
        st[f"cars_W{k}"] = getattr(cars, f"lin{k}").weight.detach().numpy().copy()
    obj = synth.make_object(3, 300, 100, 20)
    t_oc = torch.inverse(torch.from_numpy(np.array(obj["t_cam_obj_init"])))
    z = torch.from_numpy((0.05 * rng.standard_normal(64)).astype(np.float32))
    pts = torch.from_numpy(np.ascontiguousarray(obj["pts"]))
    x_obj = (pts[..., None, :] * t_oc[:3, :3]).sum(-1) + t_oc[:3, 3]
    inp = torch.cat([z.expand(x_obj.shape[0], -1), x_obj], 1)
    with torch.no_grad():
        st["dec_in"] = inp.numpy().copy()
        st["dec_y"] = cars(inp).squeeze(-1).numpy().copy()
    y, g = lu.get_batch_sdf_jacobian(cars, z, x_obj, 1)
    st["jac_y"] = y.reshape(-1).numpy().copy()
    st["jac_g"] = g.reshape(-1, 67).numpy().copy()
    jt, jc, res = lo.compute_sdf_loss(cars, pts, t_oc, z)
    st["sdf_t_obj_cam"] = t_oc.numpy().copy()
    st["sdf_z"] = z.numpy().copy()
    st["sdf_pts"] = pts.numpy().copy()
    st["sdf_J"] = torch.cat([jt, jc], -1).reshape(-1, 71).numpy().copy()
    st["sdf_res"] = res.reshape(-1).numpy().copy()
    # render term at the same state
    t_co = torch.inverse(t_oc)
    scale = torch.det(t_co[:3, :3]) ** (1 / 3)
    dmin, dmax = t_co[2, 3] - scale, t_co[2, 3] + scale
    depths = torch.linspace(dmin, dmax, 50)
    rays = torch.from_numpy(np.ascontiguousarray(obj["rays"]))
    dobs = torch.cat([torch.from_numpy(np.array(obj["depth"])), torch.full((20,), float(1.1 * dmax))])
    dobs[100:] = 1.1 * dmax
    rr = lo.compute_render_loss(cars, rays, dobs, t_oc, depths, z, th=0.01)
    st["rnd_rays"] = rays.numpy().copy()
    st["rnd_depth_obs"] = dobs.numpy().copy()
    st["rnd_depths"] = depths.numpy().copy()
    st["rnd_J"] = torch.cat([rr[0], rr[1]], -1).reshape(-1, 71).numpy().copy()
    st["rnd_res"] = rr[2].reshape(-1).numpy().copy()
    # rotation prior: upright-ish initial pose and a 3 degree tilt about x
    a = np.deg2rad(3.0)
    Rx = np.array([[1, 0, 0, 0], [0, np.cos(a), -np.sin(a), 0], [0, np.sin(a), np.cos(a), 0],
                   [0, 0, 0, 1]], dtype=np.float32)
    for nm, T in (("up", t_oc), ("tilt", torch.inverse(torch.from_numpy(Rx) @ torch.inverse(t_oc)))):
        Jr, rrot = lo.compute_rotation_loss_sim3(T.clone())
        st[f"rot_{nm}_T"] = T.numpy().copy()
        st[f"rot_{nm}_J"] = Jr.numpy().copy()
        st[f"rot_{nm}_r"] = np.array(float(rrot), dtype=np.float32)
    # exponential maps
    xs = np.array([[0.1, -0.2, 0.05, 0.02, -0.03, 0.04, 0.01],
                   [0.1, -0.2, 0.05, 0.02, -0.03, 0.04, -0.02],
                   [0.3, 0.1, -0.1, 0, 0, 0, 0.05],
                   [0.3, 0.1, -0.1, 0, 0, 0, 0.0],
                   [0, 0, 0, 0, 0, 0, 0],
                   [-0.5, 0.2, 0.7, 0.4, -0.6, 0.3, 0.0]], dtype=np.float32)
    st["exp_x"] = xs
    st["exp_sim3"] = np.stack([lu.exp_sim3(torch.from_numpy(x)).numpy() for x in xs])
    st["exp_se3"] = np.stack([lu.exp_se3(torch.from_numpy(x[:6])).numpy() for x in xs])
    # Huber
    r = torch.from_numpy(np.concatenate([rng.standard_normal(50) * 0.05, [0.0, 0.025, -0.025]]).astype(np.float32))
    rb, ls, w = lu.get_robust_res(r.clone(), 0.025)
    st["hub_r"] = r.numpy().copy()
    st["hub_rr"] = rb.reshape(-1).numpy().copy()
    st["hub_loss"] = np.array(float(ls), dtype=np.float32)
    st["lin_ab"] = np.array([float(dmin), float(dmax)], dtype=np.float32)
    st["lin_out"] = depths.numpy().copy()
    np.savez_compressed(os.path.join(HERE, "stages.npz"), **st)
    print("stages.npz:", {k: v.shape for k, v in st.items() if k.startswith(("sdf_J", "rnd_J"))})

    # ------------------------------------------------------------------ whole runs
    # config 1: 1 car, 500 pts, 700 rays, 5 iterations
    cfg1 = cfg_with("config_kitti.json", num_iterations=5)
    o = synth.make_object(0, 500, 500, 200)
    np.savez_compressed(os.path.join(HERE, "recon_cfg1.npz"), **pack_inputs(o),
                        **run_reconstruct(cars, cfg1, o))
    # KITTI-like real shape: 250 pts, 450 rays, 10 iterations
    cfgk = cfg_with("config_kitti.json")
    o = synth.make_object(1, 250, 250, 200)
    np.savez_compressed(os.path.join(HERE, "recon_kitti250.npz"), **pack_inputs(o),
                        **run_reconstruct(cars, cfgk, o))
    # config 3 shape: chairs, 256 pts, 64+18 rays, initial code, 10 iterations, redwood params
    cfg3 = cfg_with("config_redwood_01053.json", num_iterations=10)
    o = synth.make_object(2, 256, 64, 18, cls="chairs", init_code_frac=0.5)
    np.savez_compressed(os.path.join(HERE, "recon_cfg3.npz"), **pack_inputs(o, True),
                        **run_reconstruct(chairs, cfg3, o, with_code=True))
    # config 2 FULL size: 2048 pts, 2048 fg + 200 bg rays (V ~ 1e5, m in the thousands), 10 iterations
    o = synth.make_object(7, 2048, 2048, 200)
    np.savez_compressed(os.path.join(HERE, "recon_cfg2full.npz"), **pack_inputs(o),
                        **run_reconstruct(cars, cfgk, o))
    # config 3 at B = 8: exactly the batch bench.py --workload cfg3 builds (seeds 0..7)
    objs = synth.make_batch(8, 256, 64, 18, cls="chairs", seed0=0, init_code_frac=0.5)
    per = [dict(**pack_inputs(ob, True), **run_reconstruct(chairs, cfg3, ob, with_code=True)) for ob in objs]
    keys = sorted(set.intersection(*[set(p) for p in per]))
    np.savez_compressed(os.path.join(HERE, "recon_cfg3_b8.npz"), **{k: np.stack([p[k] for p in per]) for k in keys})
    # sdf_only composition, 512 pts, 10 iterations
    o = synth.make_object(4, 512, 0, 0)
    o["rays"] = np.zeros((0, 3), np.float32); o["depth"] = np.zeros((0,), np.float32)
    np.savez_compressed(os.path.join(HERE, "recon_sdf_only.npz"), **pack_inputs(o),
                        **sdf_only_composed(cars, cfgk, o))
    # failure: rays that never enter the unit sphere -> V < 10 -> is_good False
    o = synth.make_object(5, 200, 50, 10)
    o["rays"] = np.asfortranarray((o["rays"] * np.array([[-1, -1, 1]], dtype=np.float32) + np.array([[3, 3, 0]], dtype=np.float32)).astype(np.float32))
    np.savez_compressed(os.path.join(HERE, "recon_fail_few.npz"), **pack_inputs(o),
                        **run_reconstruct(cars, cfgk, o))
    # pose-only GN (estimate_pose_cam_obj), 250 pts, 5 iterations
    o = synth.make_object(6, 250, 0, 0)
    T = np.array(o["t_cam_obj_init"], dtype=np.float32)
    s = float(np.cbrt(np.linalg.det(T[:3, :3].astype(np.float64))))
    se3 = T.copy(); se3[:3, :3] /= s
    code = (0.8 * o["code_gt"]).astype(np.float32)
    opt = ns.optimizer.Optimizer(cars, cfgk)
    Tout = opt.estimate_pose_cam_obj(se3.copy(), s, np_f(o["pts"]), code.copy())
    np.savez_compressed(os.path.join(HERE, "pose_only.npz"), in_t_co_se3=se3, in_scale=np.array(s, dtype=np.float32),
                        in_pts=o["pts"], in_code=code, t_cam_obj=Tout.numpy())
    print("done")


def voxel_golden():
    """reconstruct/utils.py:97-117 voxel grid (with its true-division quirk) and decode_sdf on it."""
    cars = load_ref_decoder("cars")
    grid = ns.utils.create_voxel_grid(vol_dim=8)
    z = torch.from_numpy(np.load(os.path.join(HERE, "stages.npz"))["sdf_z"])
    sdf = ns.loss_utils.decode_sdf(cars, z, grid)
    np.savez_compressed(os.path.join(HERE, "voxel.npz"), vox8=grid.numpy(), vox8_sdf=sdf.numpy(), z=z.numpy())
    print("voxel.npz written")


def variant_golden():
    """A decoder with every optional feature of deep_sdf_decoder.py switched on -- LayerNorm instead of weight-norm
    (:58-63,96-102), xyz_in_all (:41-47,89-90), use_tanh (:93-94), TWO latent_in layers -- random weights (seeded),
    run through the reference: forward, input Jacobian (loss_utils.get_batch_sdf_jacobian) and the SDF term."""
    lu, lo = ns.loss_utils, ns.loss
    spec = dict(latent_size=64, dims=[128, 160, 128, 192, 128], dropout=None, dropout_prob=0.0, norm_layers=[0, 1, 2, 3, 4],
                latent_in=[2, 4], weight_norm=False, xyz_in_all=True, use_tanh=True, latent_dropout=False)
    torch.manual_seed(11)
    dec = ns.decoder.Decoder(**spec).eval()
    with torch.no_grad():
        for k in range(6):
            lin = getattr(dec, f"lin{k}")
            lin.weight.mul_(2.0)                      # keep activations alive through the ReLUs
            if hasattr(dec, f"bn{k}"):
                bn = getattr(dec, f"bn{k}")
                bn.weight.copy_(1.0 + 0.3 * torch.randn_like(bn.weight))
                bn.bias.copy_(0.2 * torch.randn_like(bn.bias))
    sd = {k: v.detach().numpy().copy() for k, v in dec.state_dict().items()}
    np.savez_compressed(os.path.join(HERE, "decoder_variant.npz"), spec_json=np.frombuffer(json.dumps(spec).encode(), dtype=np.uint8), **sd)
    rng = np.random.default_rng(12)
    obj = synth.make_object(13, 200, 0, 0)
    t_oc = torch.inverse(torch.from_numpy(np.array(obj["t_cam_obj_init"])))
    z = torch.from_numpy((0.3 * rng.standard_normal(64)).astype(np.float32))
    pts = torch.from_numpy(np.ascontiguousarray(obj["pts"]))
    x_obj = (pts[..., None, :] * t_oc[:3, :3]).sum(-1) + t_oc[:3, 3]
    inp = torch.cat([z.expand(x_obj.shape[0], -1), x_obj], 1)
    st = {}
    with torch.no_grad():
        st["dec_in"] = inp.numpy().copy()
        st["dec_y"] = dec(inp).squeeze(-1).numpy().copy()
    y, g = lu.get_batch_sdf_jacobian(dec, z, x_obj, 1)
    st["jac_y"] = y.reshape(-1).numpy().copy()
    st["jac_g"] = g.reshape(-1, 67).numpy().copy()
    jt, jc, res = lo.compute_sdf_loss(dec, pts, t_oc, z)
    st["sdf_t_cam_obj"] = np.array(obj["t_cam_obj_init"])
    st["sdf_z"] = z.numpy().copy()
    st["sdf_pts"] = pts.numpy().copy()
    st["sdf_J"] = torch.cat([jt, jc], -1).reshape(-1, 71).numpy().copy()
    st["sdf_res"] = res.reshape(-1).numpy().copy()
    np.savez_compressed(os.path.join(HERE, "variant.npz"), **st)
    print("variant.npz written; sdf range", float(st["dec_y"].min()), float(st["dec_y"].max()))


HYPER = dict(num_depth_samples=24, cut_off_threshold=0.02,
             joint_optim=dict(k1=0.7, k2=80.0, k3=0.05, k4=2000.0, b1=0.15, b2=0.03, learning_rate=0.8, scale_damping=2.0,
                              num_iterations=6))


def hyper_cfg():
    cfg = ref_harness.load_config("config_kitti.json")
    cfg.optimizer.num_depth_samples = HYPER["num_depth_samples"]
    cfg.optimizer.cut_off_threshold = HYPER["cut_off_threshold"]
    for k, v in HYPER["joint_optim"].items():
        cfg.optimizer.joint_optim[k] = v
    return cfg


def pose_only_cut_golden(cars):
    """estimate_pose_cam_obj (optimizer.py:45-86) for 8 iterations on a 300-point car with 10 % gross outliers, so that
    the inlier cut after iteration index 4 (:76-78) removes points: the 6x6 system and the state of every iteration,
    the inlier mask the reference applies and the final pose."""
    cfg = cfg_with("config_kitti.json")
    cfg.optimizer.pose_only_optim.num_iterations = 8
    o = synth.make_object(41, 300)
    pts = np.array(o["pts"], dtype=np.float32)
    rng = np.random.default_rng(41)
    bad = rng.choice(300, 30, replace=False)
    pts[bad] += rng.normal(0, 0.6, size=(30, 3)).astype(np.float32)
    T = np.array(o["t_cam_obj_init"], dtype=np.float32)
    s = np.float32(np.cbrt(np.linalg.det(T[:3, :3].astype(np.float64))))
    se3 = T.copy(); se3[:3, :3] /= s
    code = (0.8 * o["code_gt"]).astype(np.float32)
    opt = ns.optimizer.Optimizer(cars, cfg)
    with SolveRecorder() as rec, StateRecorder() as sr:
        Tout = opt.estimate_pose_cam_obj(se3.copy(), float(s), np_f(pts), code.copy()).numpy()
    assert len(rec.dx) == len(sr.Toc) == 8 and sr.n_pts[:5] == [300] * 5
    mask = np.abs(sr.res[4]) <= 0.05
    assert sr.n_pts[5:] == [int(mask.sum())] * 3 and mask.sum() < 300
    Toc_end = torch.mm(ns.loss_utils.exp_se3(torch.from_numpy(rec.dx[-1])), torch.from_numpy(sr.Toc[-1]))
    T_end = torch.inverse(Toc_end)
    T_end[:3, :3] /= float(s)
    assert np.array_equal(T_end.numpy(), Tout)
    np.savez_compressed(os.path.join(HERE, "pose_only_cut.npz"), in_t_co_se3=se3, in_scale=s, in_pts=pts, in_code=code,
                        H_iters=np.stack(rec.H), b_iters=np.stack(rec.b), dx_iters=np.stack(rec.dx),
                        Toc_iters=np.stack(sr.Toc + [Toc_end.numpy()]), sdf_loss_iters=np.array(sr.losses, np.float32),
                        inlier_mask=mask, t_cam_obj=Tout)
    print("pose_only_cut.npz written:", int(mask.sum()), "inliers")


def states_golden():
    """Re-runs every whole-run golden from its stored inputs, asserts that the reference reproduces the committed
    arrays bit for bit, and writes states_<name>.npz with the reference's state at every iteration:
    Toc_iters (iters+1, 4, 4) = t_obj_cam before each update and after the last one, z_iters (iters+1, L),
    sdf_loss_iters and render_loss_iters (iters,).  Teacher-forced tests start one step from each of these states."""
    cars, chairs = load_ref_decoder("cars"), load_ref_decoder("chairs")
    cfgk = cfg_with("config_kitti.json")
    cfg3 = cfg_with("config_redwood_01053.json", num_iterations=10)
    runs = [("recon_cfg1", cars, cfg_with("config_kitti.json", num_iterations=5), False),
            ("recon_kitti250", cars, cfgk, False), ("recon_cfg2full", cars, cfgk, False),
            ("recon_cfg3", chairs, cfg3, True), ("recon_cfg3_b8", chairs, cfg3, True),
            ("recon_hyper", cars, hyper_cfg(), False), ("recon_sdf_only", cars, cfgk, False)]
    for name, dec, cfg, with_code in runs:
        d = np.load(os.path.join(HERE, name + ".npz"))
        if name == "recon_hyper":
            assert json.loads(bytes(d["hyper_json"]).decode()) == HYPER
        stacked = d["in_pts"].ndim == 3
        n = d["in_pts"].shape[0] if stacked else 1
        per_res, per_st = [], []
        for i in range(n):
            g = (lambda k: d[k][i]) if stacked else (lambda k: d[k])
            o = dict(t_cam_obj_init=g("in_t_cam_obj"), pts=g("in_pts"))
            st = {}
            if name == "recon_sdf_only":
                per_res.append(sdf_only_composed(dec, cfg, o, states=st))
            else:
                o.update(rays=g("in_rays"), depth=g("in_depth"))
                if with_code:
                    o["code_init"] = g("in_code")
                per_res.append(run_reconstruct(dec, cfg, o, with_code, states=st))
            per_st.append(st)
        for k in ("H_iters", "b_iters", "dx_iters", "V_iters", "m_iters", "t_cam_obj", "code", "is_good", "loss"):
            if k in d.files:
                got = np.stack([r[k] for r in per_res]) if stacked else per_res[0][k]
                assert got.dtype == d[k].dtype and np.array_equal(got, d[k]), (name, k)
        out = {k: np.stack([s[k] for s in per_st]) if stacked else per_st[0][k] for k in per_st[0]}
        np.savez_compressed(os.path.join(HERE, "states_" + name[len("recon_"):] + ".npz"), **out)
        print(f"states_{name[len('recon_'):]}.npz: bit-identical re-run, {out['Toc_iters'].shape}")
    pose_only_cut_golden(cars)


def hyper_golden():
    """A whole run with EVERY hyper-parameter of the `optimizer` block moved off the shipped configs' values (D = 24
    depth samples instead of 50, band half-width, all weights, both Huber thresholds, learning rate, scale damping,
    iteration count): pins that the restatement reads each of them where the reference does."""
    cfg = hyper_cfg()
    cars = load_ref_decoder("cars")
    o = synth.make_object(11, 400, 300, 100)
    a = np.deg2rad(3.0)                              # tilted 3 degrees about the object's own x axis: the rotation prior is active
    Rx = np.array([[1, 0, 0, 0], [0, np.cos(a), -np.sin(a), 0], [0, np.sin(a), np.cos(a), 0], [0, 0, 0, 1]], np.float32)
    o["t_cam_obj_init"] = (o["t_cam_obj_init"] @ Rx).astype(np.float32)
    np.savez_compressed(os.path.join(HERE, "recon_hyper.npz"), **pack_inputs(o), **run_reconstruct(cars, cfg, o),
                        hyper_json=np.frombuffer(json.dumps(HYPER).encode(), dtype=np.uint8))
    print("recon_hyper.npz written")


if __name__ == "__main__":
    if "--voxel-only" in sys.argv:
        voxel_golden()
    elif "--variant-only" in sys.argv:
        variant_golden()
    elif "--hyper-only" in sys.argv:
        hyper_golden()
    elif "--states" in sys.argv:
        states_golden()
    else:
        main()
        voxel_golden()
        variant_golden()
        hyper_golden()
