"""The hot path's Python run the reference's way on the CPU -- the loop body of the reference's train.py:140-211 with
update_learning_rate / oneupSHdegree, render(), l1 + fused_ssim and PerPointAdam -- with the three native packages it
imports replaced by tests/cpu_standins (same surface as shims/, oracle inside).

Two arms over the same seeded scene, N_IT iterations each, must agree with what the reference's OWN modules
(gaussian_renderer.render, scene.gaussian_model.GaussianModel, scene.per_point_adam.PerPointAdam, utils.loss_utils)
computed on the same inputs, stored in tests/golden/ref_loop.npz by oracle/make_golden_ref_loop.py:
  mirror  instantsplat_b200.model.GaussianModel + instantsplat_b200.renderer.render(FUSED=False) on the stand-ins
  oracle  oracle/gs_oracle.py end to end (render_instantsplat + training_loss + per_point_adam_step)

Launched by tests/test_reference_shims_cpu.py (a subprocess: the stand-in packages must not leak into the test
session); oracle/make_golden_ref_loop.py imports the shared set-up (scene, cameras, loop body) from here.
"""
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "tests", "cpu_standins"), os.path.join(ROOT, "tests", "stubs"), ROOT):
    sys.path.insert(0, p) if p not in sys.path else None
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_loop.npz")

import numpy as np  # noqa: E402
import torch  # noqa: E402

torch.set_num_threads(4)

import instantsplat_b200.model as M  # noqa: E402
import instantsplat_b200.renderer as RD  # noqa: E402
from instantsplat_b200.camera import SimpleCamera  # noqa: E402
from instantsplat_b200.scenes import surface_scene  # noqa: E402
from oracle import gs_oracle as O  # noqa: E402
import diff_gaussian_rasterization as dgr  # noqa: E402  (stand-in)
from fused_ssim import fused_ssim  # noqa: E402  (stand-in)

N_IT = 6
sc = surface_scene(300, 3, 48, 32, seed=7, sh_degree=3)
gts = torch.rand(3, 3, sc.height, sc.width, generator=torch.Generator().manual_seed(3))
opt_args = M.optimization_defaults(iterations=1000)
pipe = types.SimpleNamespace(convert_SHs_python=False, compute_cov3D_python=False, debug=False)
bg = torch.zeros(3)
cams = []
for v in range(3):
    c = SimpleCamera(sc.width, sc.height, sc.fovx, sc.fovy, device="cpu")
    c.uid = v
    cams.append(c)
views = [it % 3 for it in range(N_IT)]
START_SH = 2       # start below the maximum and place the iteration counter so that oneupSHdegree fires inside the run
FIRST_ITER = 997
PCD_ATTRS = ("_xyz", "_features_dc", "_features_rest", "_scaling", "_rotation", "_opacity")


def fill(model):
    for attr, key in (("_xyz", "xyz"), ("_features_dc", "f_dc"), ("_features_rest", "f_rest"), ("_opacity", "opacity"),
                      ("_scaling", "scaling"), ("_rotation", "rotation")):
        setattr(model, attr, torch.nn.Parameter(sc.params[key].clone().requires_grad_(True)))
    model.P = sc.poses.clone().requires_grad_(True)
    model.active_sh_degree = START_SH
    model.spatial_lr_scale = 1.0
    model.max_radii2D = torch.zeros(sc.P)


def loop(model, render, l1, ssim_fn):
    """train.py:140-211 (the live lines), one view per iteration, deterministic view order."""
    losses = []
    opt = types.SimpleNamespace(lambda_dssim=0.2, iterations=FIRST_ITER + N_IT + 5)
    for k in range(N_IT):
        iteration = FIRST_ITER + k
        model.update_learning_rate(iteration)
        if iteration % 1000 == 0:
            model.oneupSHdegree()
        cam = cams[views[k]]
        pose = model.get_RT(cam.uid)
        pkg = render(cam, model, pipe, bg, camera_pose=pose)
        image = pkg["render"]
        gt = gts[views[k]]
        Ll1 = l1(image, gt)
        ssim_value = ssim_fn(image.unsqueeze(0), gt.unsqueeze(0))
        loss = (1.0 - opt.lambda_dssim) * Ll1 + opt.lambda_dssim * (1.0 - ssim_value)
        loss.backward()
        losses.append(loss.item())
        assert pkg["viewspace_points"].grad is not None and pkg["visibility_filter"].dtype == torch.bool
        if iteration < opt.iterations:
            model.optimizer.step()
            model.optimizer.zero_grad(set_to_none=True)
    return losses


def pcd():
    """The point cloud both create_from_pcd implementations initialise from."""
    pts = np.random.default_rng(0).normal(size=(200, 3)).astype(np.float32)
    cols = np.random.default_rng(1).uniform(size=(200, 3)).astype(np.float32)
    return pts, cols


def main():
    z = np.load(GOLDEN)
    assert int(z["n_it"]) == N_IT and list(z["views"]) == views
    L_ref = [float(x) for x in z["losses"]]
    ref_xyz, ref_P = torch.from_numpy(z["xyz"]), torch.from_numpy(z["poses"])

    # ---- arm 1: the mirror (reference-shaped render body, stand-in rasterizer, CPU PerPointAdam)
    from per_point_adam_cpu import PerPointAdam
    RD.FUSED = False
    RD._RASTERIZER = (dgr.GaussianRasterizationSettings, dgr.GaussianRasterizer)
    M.PerPointAdam = PerPointAdam
    mir = M.GaussianModel(3, device="cpu")
    fill(mir)
    mir.per_point_lr = sc.per_point_lr.clone()
    mir.training_setup_pp(opt_args)
    L_mir = loop(mir, RD.render, lambda a, b: (a - b).abs().mean(), fused_ssim)

    # ---- arm 2: the oracle end to end
    prm = {k: v.clone().requires_grad_(True) for k, v in sc.params.items()}
    poses = sc.poses.clone().requires_grad_(True)
    state = {k: (torch.zeros_like(v), torch.zeros_like(v)) for k, v in prm.items()}
    pstate = (torch.zeros_like(poses), torch.zeros_like(poses))
    from instantsplat_b200.trainer import get_expon_lr_func
    xyz_s = get_expon_lr_func(1.6e-4, 1.6e-6, lr_delay_mult=0.01, max_steps=30000)
    cam_s = get_expon_lr_func(1e-4, 1e-6, lr_delay_mult=0.01, max_steps=1000)
    L_or, deg = [], START_SH
    for k in range(N_IT):
        iteration = FIRST_ITER + k
        if iteration % 1000 == 0:
            deg = min(3, deg + 1)
        cam = O.Camera.instantsplat(sc.width, sc.height, sc.fovx, sc.fovy, sh_degree=deg)
        v = views[k]
        img, _ = O.render_instantsplat(prm["xyz"], prm["rotation"], prm["scaling"], prm["opacity"], prm["f_dc"],
                                       prm["f_rest"], poses[v], cam)
        loss = O.training_loss(img, gts[v])
        loss.backward()
        L_or.append(loss.item())
        lrs = dict(xyz=xyz_s(iteration), f_dc=0.025, f_rest=0.00125, opacity=0.05, scaling=0.05, rotation=0.01)
        with torch.no_grad():
            for name, p in prm.items():
                m_, v_ = state[name]
                O.per_point_adam_step(p, p.grad, m_, v_, k + 1, lrs[name],
                                      per_point_lr=sc.per_point_lr.reshape(-1, 1) if name == "xyz" else None)
                p.grad = None
            O.per_point_adam_step(poses, poses.grad, pstate[0], pstate[1], k + 1, cam_s(iteration))
            poses.grad = None

    d_mir = max(abs(a - b) for a, b in zip(L_ref, L_mir))
    d_or = max(abs(a - b) for a, b in zip(L_ref, L_or))
    dp_mir = float((ref_xyz - mir._xyz).abs().max()), float((ref_P - mir.P).abs().max())
    dp_or = float((ref_xyz - prm["xyz"]).abs().max()), float((ref_P - poses).abs().max())
    print("losses ref   ", [round(x, 7) for x in L_ref])
    print("max |loss ref - mirror|", d_mir, " |loss ref - oracle|", d_or)
    print("max |xyz,P ref - mirror|", dp_mir, " ref - oracle", dp_or)
    assert int(z["sh_degree"]) == START_SH + 1 == mir.active_sh_degree, "oneupSHdegree did not fire"
    assert d_mir < 1e-6 and d_or < 2e-6, (d_mir, d_or)
    assert max(dp_mir) < 1e-6 and max(dp_or) < 5e-6, (dp_mir, dp_or)

    # ---- pose conversion: the reference's get_tensor_from_camera vs the mirror's w2c_to_pose (same rotation, same t)
    for v in range(3):
        a = torch.from_numpy(z["tensor_from_camera"][v])
        b = M.w2c_to_pose(O.pose_to_w2c(sc.poses[v]))
        Ra, Rb = O.quad2rotation(a[:4].float()), O.quad2rotation(b[:4])
        assert float((Ra - Rb).abs().max()) < 1e-5 and float((a[4:].float() - b[4:]).abs().max()) < 1e-6

    # ---- create_from_pcd: the reference's (with the stand-in distCUDA2) vs the mirror's
    pts, cols = pcd()
    m2 = M.GaussianModel(3, device="cpu")
    m2.create_from_pcd(pts, cols, 1.5)
    for attr in PCD_ATTRS:
        a, b = torch.from_numpy(z["pcd" + attr]), getattr(m2, attr)
        assert a.shape == b.shape and float((a - b).abs().max()) < 1e-6, attr
    print("REF_LOOP_OK")


if __name__ == "__main__":
    main()
