"""JointTrainer at SH degrees 0, 1 and 2 on the GPU (-m gpu, DESIGN.md section 4.16).

The main oracle is padding equivalence: a trainer on a degree-D scene (f_rest [P, (D+1)^2 - 1, 3]) against a trainer
on the same scene padded to degree 3 with zero rows and max_sh_degree = D.  Every value both hold must be bit-equal
(images, loss sums, the pose table, every shared parameter row and Adam moment), and the padded rows must stay 0, through
step() eager and replayed, step_batch, densification (clone + split) and Mip-Splatting.  Then: checkpoint shapes and
20 iterations against train.py's loop on the drop-in render() and the mirror GaussianModel(D), checkpoint resume and
refusals, the ply at the degree, and render.py / metrics.py on a degree-1 model."""
import json
import os
import sys

import numpy as np
import pytest
import torch

import instantsplat_b200 as I
from instantsplat_b200 import freeview as F
from instantsplat_b200 import metrics as M
from instantsplat_b200 import render_views as R
from instantsplat_b200 import scene_io as S
from instantsplat_b200 import train as T
from instantsplat_b200.model import GaussianModel
from instantsplat_b200.scenes import Scene, surface_scene
from instantsplat_b200.tracking import PoseTracker

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROWS = {0: 0, 1: 3, 2: 8, 3: 15}


def _at_degree(sc: Scene, D: int, pad: bool) -> Scene:
    """sc with f_rest cut to degree D ([P, (D+1)^2 - 1, 3]), or with rows (D+1)^2 - 1 .. 14 zeroed (pad)."""
    p = {k: v.clone() for k, v in sc.params.items()}
    if pad:
        p["f_rest"][:, ROWS[D]:] = 0
    else:
        p["f_rest"] = p["f_rest"][:, :ROWS[D]].contiguous()
    return Scene(p, sc.poses.clone(), sc.width, sc.height, sc.fovx, sc.fovy, sc.sh_degree, sc.bg.clone(),
                 None if sc.per_point_lr is None else sc.per_point_lr.clone(), sc.name)


def _cfg(D, **over):
    c = I.OptimConfig()
    c.iterations = 1000
    c.max_sh_degree = D
    c.sh_increase_interval = 8          # degree steps at iterations 8, 16 and 24
    for k, v in over.items():
        setattr(c, k, v)
    return c


def _grad_threshold(sc, gts, D):
    """A densify threshold that selects about 10 % of the seen Gaussians after a few iterations."""
    tr = I.JointTrainer(_at_degree(sc, D, False), DEV, gt_images=gts,
                        cfg=_cfg(D, densify=True, densify_from_iter=10 ** 9, densify_until_iter=10 ** 9))
    for k in range(5):
        tr.step(k % sc.n_views)
    g = (tr.xyz_gradient_accum / tr.denom)[tr.denom > 0]
    return float(torch.quantile(g, 0.9))


MODES = {   # name: (use_graph, views per step, config overrides)
    "eager": (False, 1, {}),
    "graph": (True, 1, {}),
    "batch3_graph": (True, 3, {}),
    "densify": (False, 1, dict(densify=True, densify_clone_split=True, densify_from_iter=5, densification_interval=5,
                               opacity_reset_interval=20, densify_until_iter=28)),
    "densify_batch3": (False, 3, dict(densify=True, densify_batches=True, densify_clone_split=True, densify_from_iter=5,
                                      densification_interval=5, opacity_reset_interval=20, densify_until_iter=28)),
    "mip_graph": (True, 1, dict(mip_kernel_size=0.1, mip_filter3d_interval=10)),
    "mip_batch3": (False, 3, dict(mip_kernel_size=0.1, mip_filter3d_interval=10)),
}


def _rest(tr, buf):
    return tr.view(buf, "f_rest").reshape(tr.P, tr.sh_coeffs - 1, 3)


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("D", [0, 1, 2])
def test_padding_equivalence(D, mode):
    use_graph, V, over = MODES[mode]
    sc = surface_scene(5000, 3, 96, 72, seed=61 + D, sh_degree=0, sh_rest_std=0.2)
    g = torch.Generator().manual_seed(7)
    gts = torch.rand(3, 3, sc.height, sc.width, generator=g).to(DEV)
    if over.get("densify"):
        over = dict(over, densify_grad_threshold=_grad_threshold(sc, gts, D))
    A = I.JointTrainer(_at_degree(sc, D, False), DEV, gt_images=gts, cfg=_cfg(D, **over), use_graph=use_graph)
    B = I.JointTrainer(_at_degree(sc, D, True), DEV, gt_images=gts, cfg=_cfg(D, **over), use_graph=use_graph)
    assert (A.sh_coeffs, B.sh_coeffs) == ((D + 1) ** 2, 16)
    assert A.total < B.total
    for k in range(30 // V):
        views = [(k * V + j) % 3 for j in range(V)] if V > 1 else [k % 3]
        events = len(A.densified_at) + len(A.reset_at)
        for tr in (A, B):
            tr.step_batch(views) if V > 1 else tr.step(views[0])
        assert torch.equal(A._batch_sums, B._batch_sums) if V > 1 else torch.equal(A.sums, B.sums), k
        if len(A.densified_at) + len(A.reset_at) == events:      # a densify or reset rebuilds the frames: no image
            assert torch.equal(A._batch.frame.color if V > 1 else A.color,
                               B._batch.frame.color if V > 1 else B.color), k
    torch.cuda.synchronize()
    assert A.active_sh_degree == B.active_sh_degree == D
    assert A.iteration == B.iteration and A.opt_step == B.opt_step and A.P == B.P
    if over.get("densify"):
        assert A.densified_at == B.densified_at and A.densified_at and A.P != sc.P
    if over.get("mip_kernel_size"):
        assert A.mip_recomputed_at == B.mip_recomputed_at and A.mip_recomputed_at
        assert torch.equal(A.filter_3D, B.filter_3D)
    for t in ("poses", "pose_m", "pose_v"):
        assert torch.equal(getattr(A, t), getattr(B, t)), t
    for buf in ("params", "exp_avg", "exp_avg_sq"):
        for name, _ in A.widths:
            assert A.step_count(name) == B.step_count(name), name
            if name == "f_rest":
                a, b = _rest(A, getattr(A, buf)), _rest(B, getattr(B, buf))
                assert torch.equal(a, b[:, :ROWS[D]]), buf
                assert not bool(b[:, ROWS[D]:].any()), buf               # the padded rows stay exactly 0
            else:
                assert torch.equal(A.view(getattr(A, buf), name), B.view(getattr(B, buf), name)), (buf, name)


# ---- the reference's shapes and the drop-in loop ---------------------------------------------------------------------
def _source(root, P=20_000, W=160, H=112, seed=43):
    sc = surface_scene(P, 3, W, H, seed=seed, sh_degree=3)
    p = sc.params
    truth = PoseTracker(p["xyz"], p["rotation"], p["scaling"], p["opacity"], p["f_dc"], p["f_rest"], W, H, sc.fovx,
                        sc.fovy, sh_degree=3, device=DEV)
    imgs = F.quantise(truth.render_batch(sc.poses).contiguous()).cpu().numpy()
    S.write_synthetic_source(root, sc, imgs)
    return root


def _shapes(cap):
    """(shape, dtype) of every tensor of a capture() tuple, the optimizer's per-group state by group name."""
    out = [(tuple(t.shape), t.dtype) for t in cap[1:10]] + [(tuple(cap[12].shape), cap[12].dtype)]
    sd = cap[10]
    names = {g["params"][0]: g["name"] for g in sd["param_groups"]}
    st = {names[i]: tuple((tuple(s[k].shape), s[k].dtype) for k in ("exp_avg", "exp_avg_sq"))
          for i, s in sd["state"].items()}
    return out, st


@pytest.mark.parametrize("D", [0, 1, 2])
def test_agrees_with_the_reference_loop_and_its_shapes(tmp_path, D):
    """20 iterations against train.py:140-211 on the drop-in render() and the mirror GaussianModel(D) with PerPointAdam
    (tests/test_reference_loop.py), at test_train_cli_gpu.py's 5e-5; then capture() against the mirror's."""
    sys.path.insert(0, os.path.join(ROOT, "shims"))
    from instantsplat_b200.camera import SimpleCamera
    from test_reference_loop import reference_loop
    src = _source(str(tmp_path / "src"))
    n = 20
    ts = T.load_training_scene(src, 3, 1, sh_degree=D)
    assert tuple(ts.scene.params["f_rest"].shape) == (ts.scene.P, ROWS[D], 3)
    args = T.parse_args(["-s", src, "-m", str(tmp_path / "m"), "-r", "1", "--n_views", "3", "--iterations", str(n),
                         "--pp_optimizer", "--optim_pose", "--sh_degree", str(D)])
    tr = I.JointTrainer(ts.scene, DEV, gt_images=ts.targets, cfg=T.optim_config(args, ts.host.extent), use_graph=True)
    assert tr._shapes()["f_rest"] == (ts.scene.P, ROWS[D], 3)
    rows = T.view_schedule(3, n)[1]
    losses = []
    for row in rows:
        tr.step(row)
        losses.append(float(tr.loss_value()))
    gm = GaussianModel(D, DEV)
    gm.create_from_pcd(ts.host.points, ts.host.colors, ts.host.extent)
    gm.init_RT_seq(ts.host.poses)
    gm.training_setup_pp(I.optimization_defaults(iterations=n), ts.host.per_point_lr.to(DEV))
    cams = []
    for v in range(3):
        c = SimpleCamera(ts.scene.width, ts.scene.height, ts.scene.fovx, ts.scene.fovy, device=DEV)
        c.uid = v
        cams.append(c)
    ref = reference_loop(gm, I.render, rows, ts.targets, cams, n, iterations=n)
    assert ref[-1] < ref[0]
    d = max(abs(a - b) for a, b in zip(ref, losses))
    assert d < 5e-5, (d, ref, losses)
    mine, theirs = _shapes(tr.capture()), _shapes(gm.capture())
    assert mine == theirs
    assert mine[1]["f_rest"][0][0] == (ts.scene.P, ROWS[D], 3)


# ---- files at the degree ---------------------------------------------------------------------------------------------
def _small(D, seed=81):
    sc = surface_scene(3000, 3, 80, 56, seed=seed, sh_degree=0, sh_rest_std=0.2)
    g = torch.Generator().manual_seed(seed)
    return _at_degree(sc, D, False), torch.rand(3, 3, sc.height, sc.width, generator=g).to(DEV)


def test_checkpoint_resume_at_degree_1(tmp_path):
    sc, gts = _small(1)
    cfg = lambda: _cfg(1, densify=True, densify_clone_split=True, densify_from_iter=3, densification_interval=4,
                       densify_until_iter=20, densify_grad_threshold=1e-5)
    a = I.JointTrainer(sc, DEV, gt_images=gts, cfg=cfg(), use_graph=True)
    path = str(tmp_path / "chkpnt6.pth")
    for k in range(14):
        a.step(k % 3)
        if k == 5:
            a.save_checkpoint(path)
    model_args, it = torch.load(path)
    assert it == 6 and tuple(model_args[3].shape) == (model_args[1].shape[0], 3, 3)
    b = I.JointTrainer.from_checkpoint(path, sc, gt_images=gts, use_graph=True)
    assert b.sh_coeffs == 4 and b.iteration == 6
    for k in range(6, 14):
        b.step(k % 3)
    torch.cuda.synchronize()
    assert a.densified_at and a.densified_at == b.densified_at
    for buf in ("params", "exp_avg", "exp_avg_sq"):
        assert torch.equal(getattr(a, buf), getattr(b, buf)), buf
    for t in ("poses", "pose_m", "pose_v"):
        assert torch.equal(getattr(a, t), getattr(b, t)), t
    assert (a.opt_step, a._lag, a.active_sh_degree) == (b.opt_step, b._lag, b.active_sh_degree)


def test_checkpoint_of_another_degree_is_refused(tmp_path):
    s1, gts = _small(1)
    s3, _ = _small(3)
    cases = ((s3, 3, s1, 1, r"needs \[P,3,3\] \(the checkpoint holds SH degree 3, the trainer's scene SH degree 1"),
             (s1, 1, s3, 3, r"f_rest is \(3000, 3, 3\), the trainer's SH layout needs \[P,15,3\]$"))
    for src, d_src, dst, d_dst, match in cases:
        tr = I.JointTrainer(src, DEV, gt_images=gts, cfg=_cfg(d_src))
        tr.step(0)
        path = str(tmp_path / "c.pth")
        tr.save_checkpoint(path)
        with pytest.raises(I.GsbError, match=match):
            I.JointTrainer.from_checkpoint(path, dst, gt_images=gts, cfg=_cfg(d_dst))


@pytest.mark.parametrize("D", [0, 1, 2])
def test_ply_at_the_degree(tmp_path, D):
    sc, gts = _small(D)
    tr = I.JointTrainer(sc, DEV, gt_images=gts, cfg=_cfg(D, sh_increase_interval=2))
    for k in range(8):
        tr.step(k % 3)
    assert tr.active_sh_degree == D
    ply = str(tmp_path / "point_cloud.ply")
    tr.save_ply(ply)
    assert list(S._read_ply(ply).dtype.names) == S.gaussian_ply_fields(3 * ROWS[D])
    g = S.load_gaussians_ply(ply)
    assert np.array_equal(g["f_rest"], _rest(tr, tr.params).cpu().numpy())
    tk = F.load_tracker(ply, sc.width, sc.height, sc.fovx, sc.fovy)
    assert tk.sh_degree == D and tuple(tk.f_rest.shape) == (sc.P, ROWS[D], 3)
    torch.testing.assert_close(tk.render(tr.poses[1]), tr.render(1), rtol=0, atol=1e-5)


# ---- render.py and metrics.py on a degree-1 model --------------------------------------------------------------------
def test_degree_1_end_to_end(tmp_path):
    from test_render_views_gpu import _read, _source_and_model
    src, _, _ = _source_and_model(str(tmp_path))
    ts = T.load_training_scene(src, 3, 1, sh_degree=1)
    assert tuple(ts.scene.params["f_rest"].shape) == (ts.scene.P, 3, 3)
    cfg = _cfg(1, sh_increase_interval=10, iterations=40, pp_optimizer=True, optim_pose=True)
    cfg.spatial_lr_scale = float(ts.host.extent)
    tr = I.JointTrainer(ts.scene, DEV, gt_images=ts.targets, cfg=cfg, use_graph=True)
    rows = T.view_schedule(3, 40)[1]
    losses = []
    for row in rows:
        tr.step(row)
        losses.append(float(tr.loss_value()))
    assert tr.active_sh_degree == 1 and np.mean(losses[-10:]) < np.mean(losses[:10])
    model, it = str(tmp_path / "trained"), 40
    tr.save_ply(os.path.join(model, "point_cloud", f"iteration_{it}", "point_cloud.ply"))
    tr.save_poses(os.path.join(model, "pose", f"ours_{it}", "pose_optimized.npy"), ts.host.colmap_ids)
    base = ["-s", src, "-m", model, "--n_views", "3", "--iterations", "-1", "-r", "1", "--workers", "2"]
    assert R.main(base) == 0
    views = S.load_views(src, 3, 0)
    tk = R.tracker_for(model, it, views)
    assert tk.sh_degree == 1
    poses = F.poses_from_w2c(np.load(os.path.join(model, "pose", f"ours_{it}", "pose_optimized.npy")))
    idx = [f"{i:05d}.png" for i in range(3)]
    want = F.quantise(tk.render_batch(poses.to(DEV)).contiguous()).cpu().numpy()
    assert np.array_equal(_read(os.path.join(model, "train", f"ours_{it}", "renders"), idx), want)
    assert R.main(base + ["--eval", "--optim_test_pose_iter", "10"]) == 0
    assert M.main(["-s", src, "-m", model, "--n_views", "3"]) == 0
    res = json.loads(open(os.path.join(model, "results.json")).read())[f"ours_{it}"]
    assert np.isfinite(res["PSNR"]) and np.isfinite(res["SSIM"])
