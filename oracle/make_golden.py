"""Generate tests/golden/*.npz by importing the REFERENCE's own Python modules.

Needs an InstantSplat checkout.  The vectors it writes are committed; tests/test_oracle_golden.py checks the oracle
(oracle/gs_oracle.py) against them on CPU, and the `-m gpu` tests check the CUDA kernels
against the same vectors.

    python oracle/make_golden.py <path to the InstantSplat checkout>

Reference modules used (imported by file path because `scene/__init__.py` pulls in plyfile):
    utils/sh_utils.py        eval_sh
    utils/loss_utils.py      ssim, l1_loss
    utils/pose_utils.py      get_camera_from_tensor, quadmultiply
    utils/graphics_utils.py  getProjectionMatrix
    scene/per_point_adam.py  PerPointAdam
The rasterizer itself (diff-gaussian-rasterization) is an empty submodule: no vectors can be
generated for it from the reference ("parity unpinned"); `raster_tiny.npz` holds the ORACLE's
own fp64 outputs as a regression pin and is labelled as such.
"""
import importlib.util
import os
import sys

import numpy as np
import torch

REF = None                                       # the InstantSplat checkout (command line)
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, ROOT)


def _load(name, rel):
    spec = importlib.util.spec_from_file_location(name, os.path.join(REF, rel))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    os.makedirs(OUT, exist_ok=True)
    sys.path.insert(0, REF)                      # pose_utils imports utils.stepfun
    sh_utils = _load("ref_sh_utils", "utils/sh_utils.py")
    loss_utils = _load("ref_loss_utils", "utils/loss_utils.py")
    pose_utils = _load("ref_pose_utils", "utils/pose_utils.py")
    graphics = _load("ref_graphics_utils", "utils/graphics_utils.py")
    ppa = _load("ref_per_point_adam", "scene/per_point_adam.py")

    g = torch.Generator().manual_seed(1234)

    # ---- eval_sh ------------------------------------------------------------------------
    sh = torch.randn(64, 16, 3, generator=g)
    dirs = torch.randn(64, 3, generator=g)
    dirs = dirs / dirs.norm(dim=1, keepdim=True)
    out = {f"deg{d}": sh_utils.eval_sh(d, sh.transpose(1, 2), dirs).numpy() for d in range(4)}
    np.savez(os.path.join(OUT, "eval_sh.npz"), sh=sh.numpy(), dirs=dirs.numpy(), **out)

    # ---- loss: ssim / l1 (+ autograd grads w.r.t. img1) ---------------------------------
    img1 = torch.rand(3, 40, 56, generator=g).requires_grad_(True)
    img2 = (img1.detach() + 0.1 * torch.randn(3, 40, 56, generator=g)).clamp(0, 1)
    s = loss_utils.ssim(img1, img2)
    (gs,) = torch.autograd.grad(s, img1)
    l1 = loss_utils.l1_loss(img1, img2)
    (gl,) = torch.autograd.grad(l1, img1)
    total = 0.8 * loss_utils.l1_loss(img1, img2) + 0.2 * (1.0 - loss_utils.ssim(img1, img2))
    (gt_,) = torch.autograd.grad(total, img1)
    np.savez(os.path.join(OUT, "loss.npz"), img1=img1.detach().numpy(), img2=img2.numpy(),
             ssim=s.item(), ssim_grad=gs.numpy(), l1=l1.item(), l1_grad=gl.numpy(),
             total=total.item(), total_grad=gt_.numpy())

    # ---- pose helpers ------------------------------------------------------------------
    poses = torch.randn(5, 7, generator=g)
    w2c = torch.stack([pose_utils.get_camera_from_tensor(p) for p in poses])
    q2 = torch.randn(32, 4, generator=g)
    qm = pose_utils.quadmultiply(poses[0, :4], q2)
    xyz = torch.randn(32, 3, generator=g)
    # the 4 lines of gaussian_renderer/__init__.py:83-88 driven by the
    # reference's own get_camera_from_tensor
    homo = torch.cat((xyz, torch.ones(32, 1)), dim=1)
    trans = (w2c[0] @ homo.T).T[:, :3]
    np.savez(os.path.join(OUT, "pose.npz"), poses=poses.numpy(), w2c=w2c.numpy(), q2=q2.numpy(),
             qmul=qm.numpy(), xyz=xyz.numpy(), xyz_trans=trans.numpy())

    # ---- projection matrix -------------------------------------------------------------
    Pm = graphics.getProjectionMatrix(0.01, 100.0, 1.0471975512, 0.6)
    np.savez(os.path.join(OUT, "proj.npz"), P=Pm.numpy(), znear=0.01, zfar=100.0,
             fovx=1.0471975512, fovy=0.6)

    # ---- PerPointAdam: 6 steps, step 4 has an all-zero gradient (whole-tensor gate) -----
    p_pp = torch.randn(50, 3, generator=g)
    p_pl = torch.randn(50, 1, 3, generator=g)
    lr_pp = 1.0 + 99.0 * torch.rand(50, 1, generator=g)
    a = torch.nn.Parameter(p_pp.clone())
    b = torch.nn.Parameter(p_pl.clone())
    opt = ppa.PerPointAdam([{"params": [a], "lr": 1.6e-4, "per_point_lr": lr_pp, "name": "xyz"},
                            {"params": [b], "lr": 2.5e-2, "name": "f_dc"}],
                           lr=0.0, betas=(0.9, 0.999), eps=1e-15, weight_decay=0.0)
    rec = dict(p_pp=p_pp.numpy(), p_pl=p_pl.numpy(), lr_pp=lr_pp.numpy())
    for it in range(6):
        ga = torch.randn(50, 3, generator=g) * 1e-3
        gb = torch.randn(50, 1, 3, generator=g) * 1e-3
        if it == 3:
            ga.zero_()
            gb.zero_()
        a.grad, b.grad = ga.clone(), gb.clone()
        opt.step()
        rec[f"ga{it}"], rec[f"gb{it}"] = ga.numpy(), gb.numpy()
        rec[f"a{it}"], rec[f"b{it}"] = a.detach().numpy().copy(), b.detach().numpy().copy()
        rec[f"am{it}"] = opt.state[a]["exp_avg"].numpy().copy()
        rec[f"av{it}"] = opt.state[a]["exp_avg_sq"].numpy().copy()
        rec[f"bm{it}"] = opt.state[b]["exp_avg"].numpy().copy()
        rec[f"bv{it}"] = opt.state[b]["exp_avg_sq"].numpy().copy()
    np.savez(os.path.join(OUT, "per_point_adam.npz"), **rec)

    # ---- ORACLE regression pin for the rasterizer (NOT reference-derived) ---------------
    from oracle import gs_oracle as O
    from instantsplat_b200.scenes import random_scene
    sc = random_scene(400, 48, 40, seed=77)
    cam = O.Camera.instantsplat(sc.width, sc.height, sc.fovx, sc.fovy,
                                bg=torch.tensor([0.1, 0.2, 0.3]), sh_degree=3).to(torch.float64)
    P64 = {k: v.double().clone().requires_grad_(True) for k, v in sc.params.items()}
    pose = sc.poses[0].double().clone().requires_grad_(True)
    m2d = torch.zeros(sc.P, 3, dtype=torch.float64, requires_grad=True)
    img, radii, aux = O.render_instantsplat(P64["xyz"], P64["rotation"], P64["scaling"],
                                            P64["opacity"], P64["f_dc"], P64["f_rest"], pose, cam,
                                            means2D=m2d, return_aux=True)
    gt = torch.rand(3, sc.height, sc.width, generator=g).double()
    loss = O.training_loss(img, gt)
    loss.backward()
    rec = {"in_" + k: v.detach().float().numpy() for k, v in sc.params.items()}
    rec.update(pose=sc.poses[0].numpy(), gt=gt.float().numpy(), image=img.detach().numpy(),
               radii=radii.numpy(), loss=loss.item(), g_pose=pose.grad.numpy(),
               g_means2D=m2d.grad.numpy(), ambiguous=aux["ambiguous"].numpy(),
               width=sc.width, height=sc.height, fovx=sc.fovx, fovy=sc.fovy,
               bg=np.array([0.1, 0.2, 0.3], dtype=np.float32))
    for k in P64:
        rec["g_" + k] = P64[k].grad.numpy()
    np.savez_compressed(os.path.join(OUT, "raster_tiny.npz"), **rec)
    # ---- scene file formats (row f3): files written by instantsplat_b200.scene_io, parsed by the REFERENCE's
    # own COLMAP text readers (scene/colmap_loader.py:159-182,248-275)
    import tempfile
    from instantsplat_b200 import scene_io
    from instantsplat_b200.scenes import surface_scene
    cl = _load("ref_colmap_loader", "scene/colmap_loader.py")
    sc3 = surface_scene(300, 3, 64, 48, seed=21)
    with tempfile.TemporaryDirectory() as td:
        folder = scene_io.write_synthetic_source(td, sc3)
        cams = cl.read_intrinsics_text(os.path.join(folder, "cameras.txt"))
        imgs = cl.read_extrinsics_text(os.path.join(folder, "images.txt"))
    ids = sorted(imgs)
    np.savez(os.path.join(OUT, "scene_io.npz"),
             cam_ids=np.array(sorted(cams)), cam_wh=np.array([[cams[i].width, cams[i].height] for i in sorted(cams)]),
             cam_params=np.stack([cams[i].params for i in sorted(cams)]),
             img_ids=np.array(ids), qvec=np.stack([imgs[i].qvec for i in ids]), tvec=np.stack([imgs[i].tvec for i in ids]),
             img_cam=np.array([imgs[i].camera_id for i in ids]), names=np.array([imgs[i].name for i in ids]),
             rot=np.stack([cl.qvec2rotmat(imgs[i].qvec) for i in ids]))
    print("wrote", sorted(os.listdir(OUT)))


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    REF = sys.argv[1]
    main()
