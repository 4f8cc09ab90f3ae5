"""Mip-Splatting filters on the CPU (DESIGN.md section 4.7): the fp64 restatement in tests/_mip.py against central
differences, its off path against the oracle, the settings keyword and the PLY property."""
import math

import numpy as np
import torch

from oracle import gs_oracle as O

import _mip as MIP
from test_oracle_fd import _scene

TOL = 2e-5


def _filtered_scene():
    prm, pose, cam, w = _scene(seed=5)
    P = prm["xyz"].shape[0]
    g = torch.Generator().manual_seed(9)
    # f between 0.3x and 3x the median scale: some Gaussians have every s_k < f, others every s_k > f
    f3d = 0.12 * torch.exp(torch.empty(P, dtype=torch.float64).uniform_(math.log(0.3), math.log(3.0), generator=g))
    return prm, pose, cam, w, f3d


def _loss(prm, pose, cam, w, f3d, kappa=0.1):
    img, _ = MIP.render_mip(prm["xyz"], prm["rotation"], prm["scaling"], prm["opacity"], prm["f_dc"], prm["f_rest"],
                            pose, cam, kernel_size=kappa, filter3D=f3d, alpha_min=0.0, t_eps=0.0)
    return (img * w).sum()


def test_restatement_off_path_is_the_oracle():
    prm, pose, cam, _ = _scene()
    means, rots = O.pose_pretransform(prm["xyz"], prm["rotation"], pose)
    shs = torch.cat([prm["f_dc"], prm["f_rest"]], 1)
    a = O.project(means, torch.exp(prm["scaling"]), rots, torch.sigmoid(prm["opacity"]), shs, cam)
    b = MIP.project_mip(means, torch.exp(prm["scaling"]), rots, torch.sigmoid(prm["opacity"]), shs, cam, None)
    for k in ("xy", "conic", "opacity", "radii", "rect"):
        assert torch.equal(a[k], b[k]), k
    # the 2D filter with kernel_size 0.3 keeps conic and radius of the 0.3 dilation, and only scales the opacity
    c = MIP.project_mip(means, torch.exp(prm["scaling"]), rots, torch.sigmoid(prm["opacity"]), shs, cam, 0.3)
    assert torch.allclose(c["conic"], a["conic"], rtol=1e-12, atol=0) and torch.equal(c["radii"], a["radii"])
    assert bool((c["opacity"] < a["opacity"]).all())


def test_filtered_gradients_match_fp64_central_differences():
    prm, pose, cam, w, f3d = _filtered_scene()
    s = torch.exp(prm["scaling"])
    assert bool((s < f3d[:, None]).all(1).any()) and bool((s > f3d[:, None]).all(1).any())
    with torch.no_grad():
        means, rots = O.pose_pretransform(prm["xyz"], prm["rotation"], pose)
        sf, of = MIP.apply_filter3d(s, torch.sigmoid(prm["opacity"]), f3d)
        pr = MIP.project_mip(means, sf, rots, of, torch.cat([prm["f_dc"], prm["f_rest"]], 1), cam, 0.1)
        assert bool(pr["visible"].all()) and not bool(pr["h2_clamp"].any())
        assert float(pr["h2"].min()) < 0.99                 # the 2D filter does something
        a, b, c = pr["cov2d"].unbind(-1)
        assert float((a * c - b * b).min()) > 0.25
    leaves = {k: v.clone().requires_grad_(True) for k, v in prm.items()}
    pose_l = pose.clone().requires_grad_(True)
    _loss(leaves, pose_l, cam, w, f3d).backward()
    grads = {k: v.grad.clone() for k, v in leaves.items()}
    grads["pose"] = pose_l.grad.clone()
    g = torch.Generator().manual_seed(0)
    eps = 1e-6

    def fd(name, d):
        vals = []
        for sgn in (1.0, -1.0):
            p2 = {k: v.clone() for k, v in prm.items()}
            po = pose.clone()
            if name == "pose":
                po = po + sgn * eps * d
            else:
                p2[name] = p2[name] + sgn * eps * d
            with torch.no_grad():
                vals.append(float(_loss(p2, po, cam, w, f3d)))
        return (vals[0] - vals[1]) / (2 * eps)

    worst = {}
    for name, gr in grads.items():
        scale = float(gr.abs().max())
        assert scale > 0, name
        coords = list(range(7)) if name == "pose" else \
            torch.randperm(gr.numel(), generator=g)[:15].tolist() + [int(gr.abs().reshape(-1).argmax())]
        errs = []
        for ci in coords:
            d = torch.zeros(gr.numel(), dtype=torch.float64)
            d[ci] = 1.0
            d = d.reshape(gr.shape)
            errs.append(abs(fd(name, d) - float((gr * d).sum())) / scale)
        for _ in range(4):
            d = torch.randn(gr.shape, generator=g, dtype=torch.float64)
            d = d / d.norm()
            ref = float((gr * d).sum())
            errs.append(abs(fd(name, d) - ref) / max(abs(ref), scale))
        worst[name] = max(errs)
    assert not {k: v for k, v in worst.items() if not v < TOL}, worst


def test_filter3d_restatement_rules():
    W, H, t = 64, 48, 0.5
    xyz = torch.tensor([[0.0, 0.0, 2.0], [0.0, 0.0, 0.1], [0.0, 0.0, -3.0], [1.1 * t * 2.0, 0.0, 2.0],
                        [1.35 * t * 2.0, 0.0, 2.0]], dtype=torch.float64)
    poses = torch.tensor([[1.0, 0, 0, 0, 0, 0, 0], [1.0, 0, 0, 0, 0, 0, 1.0]], dtype=torch.float64)
    f = MIP.filter3d_ref(xyz, poses, W, H, t, t)
    fx = W / (2 * t)
    # 0: seen by both views, nearest 2.0; 1: seen only by view 1 (1.1); 2: behind both -> max d (3.0);
    # 3: u = 1.1 W, inside the 15 % margin; 4: u = 1.35 W, outside in view 0, and at 1.175 W in view 1 -> unseen
    expect = torch.tensor([2.0, 1.1, 3.0, 2.0, 3.0], dtype=torch.float64) / fx * math.sqrt(0.2)
    assert torch.allclose(f, expect, rtol=1e-12)


def test_settings_keyword_and_positional():
    import instantsplat_b200 as I
    kw = dict(image_height=4, image_width=5, tanfovx=0.5, tanfovy=0.4, bg=torch.zeros(3), scale_modifier=1.0,
              viewmatrix=torch.eye(4), projmatrix=torch.eye(4), sh_degree=0, campos=torch.zeros(3),
              prefiltered=False, debug=False)
    a = I.GaussianRasterizationSettings(**kw)
    assert a.kernel_size is None and len(tuple(a)) == 12
    b = I.GaussianRasterizationSettings(**kw, kernel_size=0.1)
    assert b.kernel_size == 0.1 and tuple(b)[:2] == (4, 5)
    c = I.GaussianRasterizationSettings(*kw.values(), kernel_size=0.3)
    assert c.image_width == 5 and c.kernel_size == 0.3


def test_ply_filter3d_round_trip(tmp_path):
    from instantsplat_b200 import scene_io as S
    rng = np.random.default_rng(0)
    P = 7
    t = dict(xyz=rng.normal(size=(P, 3)), f_dc=rng.normal(size=(P, 1, 3)), f_rest=rng.normal(size=(P, 15, 3)),
             opacity=rng.normal(size=(P, 1)), scaling=rng.normal(size=(P, 3)), rotation=rng.normal(size=(P, 4)))
    S.save_gaussians_ply(str(tmp_path / "a.ply"), **t)
    a = S.load_gaussians_ply(str(tmp_path / "a.ply"))
    assert "filter_3D" not in a
    f3d = rng.uniform(0.01, 0.1, size=(P, 1))
    S.save_gaussians_ply(str(tmp_path / "b.ply"), **t, filter_3D=f3d)
    b = S.load_gaussians_ply(str(tmp_path / "b.ply"))
    assert np.array_equal(b["filter_3D"], f3d.astype(np.float32))
    for k, v in t.items():
        assert np.array_equal(a[k], v.astype(np.float32)) and np.array_equal(b[k], a[k]), k
    # Mip-Splatting's layout: the property follows rot_3
    hdr = open(tmp_path / "b.ply", "rb").read(4000).split(b"end_header")[0].decode()
    assert hdr.index("property float rot_3") < hdr.index("property float filter_3D")


# ---- the kernels' own arithmetic, compiled for the host -------------------------------------------------------------
def _host_lib(tmp_path_factory):
    import ctypes
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = str(tmp_path_factory.mktemp("hmip") / "libhostmip.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-x", "c++", "-ffp-contract=off",
                           os.path.join(root, "tests", "host_mip.cpp"), "-o", out])
    return ctypes.CDLL(out)


def test_host_compiled_mip_math_matches_restatement(tmp_path_factory):
    import ctypes
    from test_host_math import _cam, _fp
    from instantsplat_b200.scenes import random_scene
    L = _host_lib(tmp_path_factory)
    sc = random_scene(1500, 96, 80, seed=17, sh_degree=3)
    g = torch.Generator().manual_seed(4)
    sc.params["scaling"] = math.log(0.006) + 0.9 * torch.randn(sc.P, 3, generator=g)
    sc.params["scaling"][:60] = math.log(2e-4)                          # h2 at its floor without the 3D filter
    cam = O.Camera.instantsplat(sc.width, sc.height, sc.fovx, sc.fovy, sh_degree=3)
    f3d_all = MIP.filter3d_ref(sc.params["xyz"], sc.poses, sc.width, sc.height, cam.tanfovx, cam.tanfovy).float()
    h = _cam(sc, 3, cam)
    P = sc.P
    np_in = {k: np.ascontiguousarray(v.numpy()) for k, v in sc.params.items()}
    for kappa, f3d in ((0.1, f3d_all), (0.3, None), (None, f3d_all)):
        prm = {k: v.double().clone().requires_grad_(True) for k, v in sc.params.items()}
        pose = sc.poses[0].double().clone().requires_grad_(True)
        means, rots = O.pose_pretransform(prm["xyz"], prm["rotation"], pose)
        s, o = torch.exp(prm["scaling"]), torch.sigmoid(prm["opacity"]).reshape(-1)
        if f3d is not None:
            s, o = MIP.apply_filter3d(s, o, f3d.double())
        pr = MIP.project_mip(means, s, rots, o, torch.cat([prm["f_dc"], prm["f_rest"]], 1), cam.to(torch.float64),
                             kappa)
        geom = np.zeros((P, 12), np.float32)
        h2 = np.zeros((P, 2), np.float32)
        fa = None if f3d is None else np.ascontiguousarray(f3d.numpy())
        args = (ctypes.byref(h), P, _fp(np_in["xyz"]), _fp(np_in["scaling"]), _fp(np_in["rotation"]),
                _fp(np_in["opacity"]), _fp(np_in["f_dc"]), _fp(np_in["f_rest"]), int(kappa is not None),
                ctypes.c_float(kappa or 0.0), None if fa is None else _fp(fa))
        L.host_project_mip(*args, _fp(geom), _fp(h2))
        vis = pr["visible"].numpy() & (geom[:, 11] > 0)
        assert vis.sum() > 300
        ref = torch.cat([pr["xy"], pr["conic"], pr["opacity"][:, None]], 1).detach().numpy()
        rel = np.abs(geom[vis, :6] - ref[vis]) / (np.abs(ref[vis]) + 1e-3 * np.abs(ref[vis]).max(0))
        # h2 comes from det(Sigma2) = a0 c0 - b^2, which fp32 resolves to (a0 c0 + b^2) / det * 6e-8 relative: the
        # opacity is bounded on that scale (needles far below a pixel are the ill-conditioned ones)
        a_, b_, c_ = (t.detach().numpy() for t in pr["cov2d"].unbind(-1))
        k_ = kappa or 0.0
        det0 = (a_ - k_) * (c_ - k_) - b_ * b_
        cond = np.abs((a_ - k_) * (c_ - k_) + b_ * b_) / np.maximum(np.abs(det0), 1e-300)
        rel[:, 5] /= 1.0 + (1e-7 * cond[vis] / 2e-4 if kappa is not None else 0.0)
        assert rel.max() < 2e-4, (kappa, f3d is not None, rel.max(0))
        if kappa is not None:
            clamp = pr["h2_clamp"].numpy()
            assert ((h2[vis, 1] > 0) == clamp[vis]).mean() > 0.999
            if f3d is None:
                assert clamp[vis].sum() > 10          # the floor is reached (and then carries no gradient)
        ds = torch.randn(P, 9, generator=g, dtype=torch.float64) * torch.as_tensor(vis)[:, None]
        Lo = (ds[:, 0:2] * pr["xy"]).sum() + (ds[:, 2:5] * pr["conic"]).sum() + (ds[:, 5] * pr["opacity"]).sum() \
            + (ds[:, 6:9] * pr["rgb"]).sum()
        Lo.backward()
        out = [np.zeros(sh, np.float32) for sh in ((P, 3), (P, 3), (P, 4), (P,), (7,))]
        L.host_project_bwd_mip(*args, _fp(np.ascontiguousarray(ds.float().numpy())), *(_fp(a) for a in out))
        for mine, ref_t, name in zip(out, (prm["xyz"].grad, prm["scaling"].grad, prm["rotation"].grad,
                                           prm["opacity"].grad, pose.grad), ("xyz", "scaling", "rotation", "opacity",
                                                                             "pose")):
            r = ref_t.detach().numpy().reshape(mine.shape)
            sel = vis if mine.shape[0] == P else slice(None)
            err = np.abs(mine[sel] - r[sel]).max() / (np.abs(r[sel]).max() + 1e-12)
            assert err < 2e-3, (kappa, f3d is not None, name, err)
    # the per-view rule of the filter size
    dep = np.zeros(P, np.float32)
    fx, fy = sc.width / (2 * cam.tanfovx), sc.height / (2 * cam.tanfovy)
    poses = np.ascontiguousarray(sc.poses.numpy())
    L.host_mip_depth(P, _fp(np_in["xyz"]), poses.shape[0], _fp(poses), ctypes.c_float(fx), ctypes.c_float(fy),
                     sc.width, sc.height, _fp(dep))
    seen = dep >= 0
    fmax = dep[seen].max()
    f_host = np.where(seen, dep, fmax) / fx * math.sqrt(0.2)
    np.testing.assert_allclose(f_host, f3d_all.numpy(), rtol=1e-5)


# ---- the model mirror's getters and the unfused render body, on a CPU rasterizer built from tests/_mip.py ----------
class _CpuRasterizer:
    def __init__(self, raster_settings):
        self.rs = raster_settings

    def __call__(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                 cov3D_precomp=None):
        rs = self.rs
        cam = O.Camera(rs.image_width, rs.image_height, rs.tanfovx, rs.tanfovy, rs.viewmatrix, rs.projmatrix,
                       rs.campos, rs.bg, rs.sh_degree, rs.scale_modifier)
        proj = MIP.project_mip(means3D, scales, rotations, opacities.reshape(-1), shs, cam, rs.kernel_size)
        return O.blend(proj, cam), proj["radii"]


def test_model_getters_and_unfused_render_match_restatement():
    import instantsplat_b200.renderer as RD
    from instantsplat_b200.camera import SimpleCamera
    from instantsplat_b200.model import GaussianModel
    from instantsplat_b200.rasterizer import GaussianRasterizationSettings
    from instantsplat_b200.scenes import random_scene
    sc = random_scene(400, 64, 48, seed=23, sh_degree=3)
    m = GaussianModel(3, device="cpu")
    m._set_params(sc.params)
    m.active_sh_degree = 3
    m.init_RT_seq(sc.poses)
    f3d = MIP.filter3d_ref(sc.params["xyz"], sc.poses, sc.width, sc.height, math.tan(sc.fovx / 2),
                           math.tan(sc.fovy / 2)).float()
    m.filter_3D = f3d[:, None]
    s_ref, o_ref = MIP.apply_filter3d(torch.exp(sc.params["scaling"]), torch.sigmoid(sc.params["opacity"]), f3d)
    assert torch.allclose(m.get_scaling_with_3D_filter, s_ref, rtol=1e-6)
    assert torch.allclose(m.get_opacity_with_3D_filter.reshape(-1), o_ref, rtol=1e-6)
    camv = SimpleCamera(sc.width, sc.height, sc.fovx, sc.fovy, device="cpu")
    bg = torch.tensor([0.1, 0.2, 0.3])
    saved = RD._RASTERIZER, RD.FUSED
    RD._RASTERIZER, RD.FUSED = (GaussianRasterizationSettings, _CpuRasterizer), False
    try:
        out = RD.render(camv, m, None, bg, camera_pose=m.get_RT(0), kernel_size=0.1)
    finally:
        RD._RASTERIZER, RD.FUSED = saved
    cam = O.Camera.instantsplat(sc.width, sc.height, sc.fovx, sc.fovy, bg=bg, sh_degree=3)
    ref, radii = MIP.render_mip(sc.params["xyz"], sc.params["rotation"], sc.params["scaling"], sc.params["opacity"],
                                sc.params["f_dc"], sc.params["f_rest"], sc.poses[0], cam, 0.1, f3d)
    assert float((out["render"].detach() - ref.detach()).abs().max()) < 1e-5
    assert torch.equal(out["radii"], radii) and int((radii > 0).sum()) > 100
    # gradients reach the model's raw tensors through the getters
    out["render"].sum().backward()
    assert float(m._scaling.grad.abs().max()) > 0 and float(m._opacity.grad.abs().max()) > 0


def test_settings_kernel_size_survives_replace_copy_and_pickle():
    import copy
    import pickle
    import instantsplat_b200 as I
    a = I.GaussianRasterizationSettings(4, 5, 0.5, 0.4, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0,
                                        torch.zeros(3), False, False, kernel_size=0.1)
    for b in (a._replace(debug=True), copy.copy(a), copy.deepcopy(a), pickle.loads(pickle.dumps(a)),
              I.GaussianRasterizationSettings._make(tuple(a), kernel_size=0.1)):
        assert b.kernel_size == 0.1 and tuple(b)[:2] == (4, 5)
    assert a._replace(kernel_size=None).kernel_size is None
