"""Densify with batched training (-m gpu, DESIGN.md sections 4.8 and 4.10): the statistics of gsb_backward_batch_stats
against single-view backwards with statistics made in view order, an overflowed batch counted once, step_batch with
densify against a restatement from the trainer's public pieces, step_batch([v]) against step(v), interleaving with
step() under graph replay, and checkpoints around a batched event -- all bit for bit (torch.equal)."""
import math

import pytest
import torch

import instantsplat_b200 as I
from instantsplat_b200 import GsbError
from instantsplat_b200._lib import GsbGrads
from instantsplat_b200.frame import densify_stats, gaussians
from instantsplat_b200.scenes import surface_scene
from instantsplat_b200.trainer import SEGMENTS
from test_densify_gpu import _quat_R, grad_threshold, inputs
from test_train_batch import _with_big_gaussian

pytestmark = pytest.mark.gpu
DEV = "cuda"
KEYS = tuple(name for name, _ in SEGMENTS)


def _cfg(**over):
    c = I.OptimConfig()
    c.iterations = 1000
    c.densify = True
    c.densify_batches = True
    c.densify_from_iter = c.densify_until_iter = 10 ** 9      # statistics only, unless overridden
    for k, v in over.items():
        setattr(c, k, v)
    return c


# ---- 1. statistics of the batched backward --------------------------------------------------------------------------
def _stats_scene(big, behind_view):
    """215x167 frames; 200 Gaussians below the 1/255 opacity cutoff, 200 behind the camera of view `behind_view`."""
    sc = surface_scene(6000, 5, 215, 167, seed=71, sh_degree=3)
    sc.params["opacity"][:200] = torch.logit(torch.tensor(0.002))
    R, t = _quat_R(sc.poses[behind_view, :4]), sc.poses[behind_view, 4:]
    behind = torch.stack([torch.tensor([0.1 * (k % 20 - 10), 0.1 * (k // 20 - 5), -1.0]) for k in range(200)])
    sc.params["xyz"][200:400] = (behind - t) @ R
    if big:
        sc = _with_big_gaussian(sc)
    return sc


STATS_CASES = [  # (V, SH degree, mip, blind view position, big Gaussian, n_stats)
    (1, 3, False, None, False, 1),
    (2, 3, False, None, True, 2),
    (3, 3, False, 1, True, 3),
    (5, 3, False, 4, True, 2),
    (3, 0, False, None, True, 3),
    (3, 3, True, 0, True, 1),
    (5, 0, True, 2, False, 5),
    (3, 3, False, None, True, 0),
]


@pytest.mark.parametrize("V,deg,mip,blind,big,n_stats", STATS_CASES)
def test_batched_statistics_equal_single_views(V, deg, mip, blind, big, n_stats):
    views = [4, 1, 3, 0, 2][:V]                                     # not in index order
    sc = _stats_scene(big, views[0])
    gts = torch.rand(5, 3, sc.height, sc.width, generator=torch.Generator().manual_seed(V)).to(DEV)
    tr = I.JointTrainer(sc, DEV, gt_images=gts, cfg=_cfg(mip_kernel_size=0.1 if mip else None))
    tr.active_sh_degree = deg
    if blind is not None:
        tr.poses[views[blind], 4:] = torch.tensor([0.0, 0.0, -100.0], device=DEV)   # sees nothing
    g = torch.Generator(device=DEV).manual_seed(5)
    s0 = torch.stack([torch.rand(tr.P, device=DEV, generator=g) * 1e-3, torch.randint(0, 3, (tr.P,), device=DEV,
                      generator=g).float(), torch.rand(tr.P, device=DEV, generator=g) * 30])
    # V single views in view order, the first n_stats with statistics
    tr._stats.copy_(s0)
    acc = None
    for k, v in enumerate(views):
        tr.render(v)
        if k == 0:
            assert int((tr.frame.radii[200:400] == 0).sum()) == 200            # behind view 0's camera
        tr.loss_and_backward(v, tr.gt[v], stats=k < n_stats)
        acc = tr.grads.clone() if acc is None else acc + tr.grads
    single = tr._stats.clone()
    # one batched forward and backward, with and without statistics
    b = tr._batch_scratch(V)
    b.sel.copy_(torch.tensor([views, views]))
    out = {}
    for n in (n_stats, 0):
        tr._stats.copy_(s0)
        tr._settled(lambda: tr._enqueue_batch(b, tr.gt, False, n), batch=b)
        out[n] = (tr.grads.clone(), tr._stats.clone())
    for k in range(3):
        assert torch.equal(out[n_stats][1][k], single[k]), k
    assert torch.equal(out[0][1], s0)
    assert torch.equal(out[n_stats][0], out[0][0]) and torch.equal(out[0][0], acc)
    radii = b.frame.radii[:n_stats]
    assert int((single[1] - s0[1]).sum()) == int((radii > 0).sum())
    if bool((radii > 0).any()):
        seen_low = (radii[:, :200] > 0).any(0)
        assert bool(seen_low.any()) and torch.equal(single[0][:200][seen_low], s0[0][:200][seen_low])  # no tile, |g| = 0
        assert bool((single[0] > s0[0]).any())
    else:                                                           # only blind views counted
        assert torch.equal(single, s0)
    if big:
        assert int(b.frame.radii[:, -1].max()) > 215


# ---- 2. overflow -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("use_graph", [False, True])
def test_overflowed_batch_counts_once(use_graph):
    sc, gts, _ = inputs(P=30_000, n_views=4, W=256, H=160, seed=73)
    batches = [[0, 1, 2], [3, 0, 1], [2, 3, 0], [1, 2, 3], [0, 3, 1]]

    def run(sabotage_at=None):
        tr = I.JointTrainer(sc, DEV, gt_images=gts, cfg=_cfg(), use_graph=use_graph)
        for k, views in enumerate(batches):
            if k == sabotage_at:
                tr._batch.frame.alloc_binning(2000)
            tr.step_batch(views)
        torch.cuda.synchronize()
        return tr

    ref, ovf = run(), run(sabotage_at=3)
    assert ovf.overflows == 1 and ref.overflows == 0
    assert int(ref.denom.max()) > 3
    assert torch.equal(ref._stats, ovf._stats) and torch.equal(ref.params, ovf.params)


# ---- 3. training steps against a restatement -------------------------------------------------------------------------
def snapshot(tr):
    s = {f"{b}_{k}": tr.view(getattr(tr, b), k).clone() for b in ("params", "exp_avg", "exp_avg_sq") for k in KEYS}
    s.update(poses=tr.poses.clone(), pose_m=tr.pose_m.clone(), pose_v=tr.pose_v.clone(), stats=tr._stats.clone(),
             P=tr.P, opt_step=tr.opt_step, iteration=tr.iteration, steps={n: tr.step_count(n) for n in KEYS + ("pose",)},
             densified_at=list(tr.densified_at), reset_at=list(tr.reset_at), active_sh_degree=tr.active_sh_degree,
             filter_3D=None if tr.filter_3D is None else tr.filter_3D.clone(), mip=list(tr.mip_recomputed_at))
    return s


def assert_same(a, b, where=""):
    assert a.keys() == b.keys()
    for k in a:
        if torch.is_tensor(a[k]):
            assert torch.equal(a[k], b[k]), (where, k)
        else:
            assert a[k] == b[k], (where, k, a[k], b[k])


def restated_step(tr, views):
    """One step over `views` from the trainer's public pieces and step()'s per-iteration rules: view k stands for
    iteration before+1+k and counts its statistics while that is below densify_until_iter; the densify / reset points
    the step covers fire once, recorded at the iteration after the step; optimizer_step(grad_scale=1/V) without the
    replaced tensors."""
    c, V = tr.cfg, len(views)
    before = tr.iteration
    its = list(range(before + 1, before + V + 1))
    tr.iteration += V
    if tr.iteration // c.sh_increase_interval > before // c.sh_increase_interval:
        tr.active_sh_degree = min(tr.active_sh_degree + 1, c.max_sh_degree)
    dens = [j for j in its if c.densify_from_iter < j < c.densify_until_iter and j % c.densification_interval == 0]
    reset = any(j < c.densify_until_iter and (j % c.opacity_reset_interval == 0 or
                                              (tr.white_background and j == c.densify_from_iter)) for j in its)
    acc, pg, losses = None, None, []
    for j, v in zip(its, views):
        tr.render(v)
        tr.loss_and_backward(v, tr.gt[v], stats=j < c.densify_until_iter)
        acc = tr.grads.clone() if acc is None else acc + tr.grads
        pg = tr.pose_grad.clone() if pg is None else pg + tr.pose_grad
        losses.append(tr.loss_value().clone())
    tr.grads.copy_(acc)
    tr.pose_grad.copy_(pg)
    skip = set()
    if dens:
        size = c.size_threshold if dens[-1] > c.opacity_reset_interval else None
        tr.densify_and_prune(c.densify_grad_threshold, c.min_opacity, tr.scene_extent, size, c.densify_clone_split,
                             tr.densify_generator)
        tr.densified_at.append(tr.iteration)
        skip.update(KEYS)
    if reset:
        tr.reset_opacity()
        tr.reset_at.append(tr.iteration)
        skip.add("opacity")
    if tr.iteration < c.iterations:
        tr.optimizer_step(grad_scale=1.0 / V, skip=[n for n in KEYS if n in skip])
    if tr.filt is not None and tr.iteration // c.mip_filter3d_interval > before // c.mip_filter3d_interval and \
            tr.iteration < c.iterations - 100:
        tr.compute_filter_3D()
        tr.mip_recomputed_at.append(tr.iteration)
    return torch.stack(losses)


LOOP = dict(densify_from_iter=5, densification_interval=5, opacity_reset_interval=20, densify_until_iter=35)
TRAIN_CASES = {   # name: (V, clone + split, Mip, white background, schedule overrides)
    "prune_only_v3": (3, False, False, False, {}),
    "clone_split_mip_white_v3": (3, True, True, True, {}),
    "v4_interval_5": (4, True, False, False, {}),
    "v5_two_points_per_step": (5, True, False, False, dict(densification_interval=2, densify_until_iter=27)),
}


def _loop_scene(white=False, seed=75):
    sc, gts, _ = inputs(P=12_000, n_views=5, W=160, H=96, seed=seed, white=white)
    return sc, gts


@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("case", sorted(TRAIN_CASES))
def test_step_batch_with_densify_equals_restatement(case, use_graph):
    V, cs, mip, white, over = TRAIN_CASES[case]
    sc, gts = _loop_scene(white)
    kw = dict(LOOP, **over)
    thr = grad_threshold(sc, gts)
    cfg = lambda: _cfg(densify_clone_split=cs, densify_grad_threshold=thr,
                       mip_kernel_size=0.1 if mip else None, sh_increase_interval=7, mip_filter3d_interval=9, **kw)
    a = I.JointTrainer(sc, DEV, gt_images=gts, cfg=cfg(), use_graph=use_graph)
    b = I.JointTrainer(sc, DEV, gt_images=gts, cfg=cfg())
    a.active_sh_degree = b.active_sh_degree = 0
    n_steps = -(-40 // V)
    crossed_until = False
    for k in range(n_steps):
        views = [(k * V + j) % 5 for j in range(V)]
        before = a.iteration
        crossed_until |= before + 1 < kw["densify_until_iter"] <= before + V
        a.step_batch(views)
        losses = restated_step(b, views)
        assert_same(snapshot(a), snapshot(b), (k, views))
        assert torch.equal(a.batch_loss_values(), losses), k
    assert crossed_until
    assert len(a.densified_at) >= 3 and len(a.reset_at) >= 1 and len(set(snapshot(a)["steps"].values())) > 1
    if use_graph:
        assert len(a._graphs) > 0


# ---- 4. consistency --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("use_graph", [False, True])
def test_step_batch_of_one_view_equals_step_with_densify(use_graph):
    sc, gts = _loop_scene(white=True, seed=77)
    thr = grad_threshold(sc, gts)
    cfg = lambda: _cfg(densify_clone_split=True, densify_grad_threshold=thr, **LOOP)
    a = I.JointTrainer(sc, DEV, gt_images=gts, cfg=cfg(), use_graph=use_graph)
    b = I.JointTrainer(sc, DEV, gt_images=gts, cfg=cfg(), use_graph=use_graph)
    for k in range(40):
        v = (3 * k) % 5
        a.step_batch([v])
        b.step(v)
        assert_same(snapshot(a), snapshot(b), k)
        assert torch.equal(a.batch_loss_values()[0], b.loss_value()), k
    assert a.densified_at == [10, 15, 20, 25, 30] and a.reset_at == [5, 20]


# batches of three views (one scratch, replayed between events) and single views; densify points 10, 15, 20 and 25
# fall inside batches, 30 on a step() call, and the last batch has two views
CALLS = [0, [1, 2, 3], 4, [0, 1, 2], [3, 4, 0], 1, [2, 3, 4], 0, [1, 2, 4], [0, 3, 4], 2, [3, 1, 0], [2, 4, 1], 0,
         [1, 3, 4], 2, [0, 2, 1], 4, [3, 0]]


def test_step_and_step_batch_interleaved_with_densify():
    """step() and step_batch() interleaved on one replaying trainer give the results of the same calls run eagerly,
    with densify, reset and statistics in both kinds of call."""
    sc, gts = _loop_scene(seed=79)
    thr = grad_threshold(sc, gts)
    cfg = lambda: _cfg(densify_clone_split=True, densify_grad_threshold=thr, **LOOP)
    a = I.JointTrainer(sc, DEV, gt_images=gts, cfg=cfg(), use_graph=True)
    b = I.JointTrainer(sc, DEV, gt_images=gts, cfg=cfg())
    replayed = set()
    for k, call in enumerate(CALLS):
        for tr in (a, b):
            if isinstance(call, list):
                tr.step_batch(call)
            else:
                tr.step(call)
        assert_same(snapshot(a), snapshot(b), (k, call))
        assert a.overflows == b.overflows
        replayed.update(key[0] == "batch" for key in a._graphs)
    assert a.densified_at == [11, 15, 22, 26, 30] and a.reset_at == [22] and a.iteration == 40
    assert replayed == {True, False}


@pytest.mark.parametrize("k_save", [3, 4])
def test_checkpoint_around_a_batched_densify_event(tmp_path, k_save):
    """V = 3 from iteration 0: step 4 covers 10..12 and densifies.  A checkpoint after step 3 (just before the event)
    and after step 4 (just after it) resumes bit-identically."""
    sc, gts = _loop_scene(seed=81)
    thr = grad_threshold(sc, gts)
    cfg = lambda: _cfg(densify_clone_split=True, densify_grad_threshold=thr, **LOOP)
    batches = [[(3 * k + j) % 5 for j in range(3)] for k in range(9)]
    full = I.JointTrainer(sc, DEV, gt_images=gts, cfg=cfg())
    snaps = []
    for views in batches:
        full.step_batch(views)
        snaps.append(snapshot(full))
    assert full.densified_at[0] == 12
    a = I.JointTrainer(sc, DEV, gt_images=gts, cfg=cfg())
    for views in batches[:k_save]:
        a.step_batch(views)
    path = str(tmp_path / "chkpnt.pth")
    a.save_checkpoint(path)
    c = I.JointTrainer.from_checkpoint(path, sc, gt_images=gts, device=DEV)
    assert c.cfg.densify_batches and c.iteration == 3 * k_save
    with pytest.raises(GsbError):
        c.batch_loss_values()
    for k, views in enumerate(batches[k_save:], k_save):
        c.step_batch(views)
        assert_same(snaps[k], snapshot(c), k)


def test_refusals_with_densify():
    sc, gts = _loop_scene(seed=83)
    off = I.JointTrainer(sc, DEV, gt_images=gts, cfg=_cfg(densify_batches=False))
    with pytest.raises(GsbError, match="densify_batches"):
        off.step_batch([0, 1])
    assert off.iteration == 0 and off.opt_step == 0
    # the C entry point refuses n_stats outside 0..V and missing statistics buffers
    tr = I.JointTrainer(sc, DEV, gt_images=gts, cfg=_cfg())
    tr.step_batch([0, 1])
    b = tr._batch
    cam = tr.ident.camera(tr.active_sh_degree, 16)
    g = gaussians(tr.P, *(tr.view(tr.params, n) for n in ("xyz", "rotation", "scaling", "opacity", "f_dc",
                                                                   "f_rest")), b.poses)
    gr = GsbGrads()
    gr.dL_dmeans3D = tr.view(tr.grads, "xyz").data_ptr()
    ok = densify_stats(b.frame.radii, tr._stats[0], tr._stats[1], tr._stats[2])
    null = densify_stats(b.frame.radii, tr._stats[0], None, tr._stats[2])
    for st, n in ((ok, -1), (ok, 3), (None, 1), (null, 2)):
        with pytest.raises(GsbError):
            b.frame.backward_batch(cam, g, b.poses, b.dL, gr, b.dpose, None, st, n)
    assert math.isfinite(float(tr.batch_loss_values().sum()))
