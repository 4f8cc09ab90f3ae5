"""JointTrainer with train.py's random background on the GPU (-m gpu, DESIGN.md section 4.17).

train.py:164 renders every iteration over bg = torch.rand((3), device="cuda"), a stream seeded by safe_state's
torch.manual_seed(0).  The trainer draws the same colours from its own CUDA generator, one torch.rand(3) per iteration,
into fixed device rows that step()'s camera and step_batch's per-view background table point at.  Checked here: the
sequence itself, agreement with train.py's loop on the drop-ins, equality with a fixed background holding the same
colour, eager against graph replay, the repeat after a binning overflow, the view-batched kernels against single views,
checkpoint resume and the refusal of blend version 1."""
import dataclasses
import os
import subprocess
import sys

import pytest
import torch

import instantsplat_b200 as I
from instantsplat_b200 import _lib
from instantsplat_b200.scenes import surface_scene

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")


def _cfg(**over):
    c = I.OptimConfig()
    c.iterations = 1000
    c.random_background = True
    for k, v in over.items():
        setattr(c, k, v)
    return c


def _scene(P=5000, W=96, H=72, seed=71, sh_degree=3):
    sc = surface_scene(P, 3, W, H, seed=seed, sh_degree=sh_degree)
    gts = torch.rand(3, 3, H, W, generator=torch.Generator().manual_seed(seed)).to(DEV)
    return sc, gts


def _state(tr):
    """Everything a step changes, as one dict of device tensors."""
    s = {f"{b}_{k}": tr.view(getattr(tr, b), k) for b in ("params", "exp_avg", "exp_avg_sq") for k, w in tr.widths}
    s.update(poses=tr.poses, pose_m=tr.pose_m, pose_v=tr.pose_v)
    return s


def _assert_equal(a, b, where=""):
    sa, sb = _state(a), _state(b)
    for k in sa:
        assert torch.equal(sa[k], sb[k]), (where, k)
    assert (a.iteration, a.opt_step, a.active_sh_degree) == (b.iteration, b.opt_step, b.active_sh_degree), where


def _draws(n, seed=0):
    """n consecutive torch.rand(3) draws of a fresh CUDA generator seeded with `seed`."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.stack([torch.rand(3, generator=g, device=DEV) for _ in range(n)])


# ---- 1. the sequence ----------------------------------------------------------------------------------------------
def test_colours_are_train_py_sequence():
    """50 iterations of step(), read from the trainer's slot, against torch.manual_seed(0) followed by 50 calls of
    torch.rand((3), device="cuda") in a fresh process; then step_batch calls of V = 1, 3 and 2 take them in order."""
    code = ("import torch\ntorch.manual_seed(0)\n"
            "x = torch.stack([torch.rand((3), device='cuda') for _ in range(50)])\n"
            "print(x.cpu().numpy().tobytes().hex())\n")
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, check=True)
    import numpy as np
    want = torch.from_numpy(np.frombuffer(bytes.fromhex(out.stdout.strip()), dtype=np.float32).reshape(50, 3).copy())
    sc, gts = _scene(P=2000, W=64, H=48)
    tr = I.JointTrainer(sc, DEV, gt_images=gts, cfg=_cfg(), use_graph=True)
    got = []
    for k in range(50):
        tr.step(k % 3)
        got.append(tr._single.bg.clone())
    assert torch.equal(torch.stack(got).cpu(), want)
    tb = I.JointTrainer(sc, DEV, gt_images=gts, cfg=_cfg(), use_graph=True)
    rows = []
    for views in ([1], [0, 1, 2], [2, 0]):
        tb.step_batch(views)
        rows.append(tb._batch.bg.clone())
    assert tb.iteration == 6
    assert torch.equal(torch.cat(rows).cpu(), want[:6])


# ---- 2. train.py's loop ---------------------------------------------------------------------------------------------
def random_bg_loop(model, render, views, gts, cams, n_iters, iterations=1000, lambda_dssim=0.2):
    """tests/test_reference_loop.py's reference_loop with train.py:164's random background: after safe_state's
    torch.manual_seed(0), bg = torch.rand((3), device="cuda") at the top of every iteration."""
    from fused_ssim import fused_ssim
    pipe = type("Pipe", (), dict(convert_SHs_python=False, compute_cov3D_python=False, debug=False))()
    losses = []
    with torch.random.fork_rng(devices=[torch.cuda.current_device()]):
        torch.manual_seed(0)
        for k in range(n_iters):
            iteration = 1 + k
            model.update_learning_rate(iteration)
            if iteration % 1000 == 0:
                model.oneupSHdegree()
            bg = torch.rand((3), device="cuda")
            cam = cams[views[k]]
            pkg = render(cam, model, pipe, bg, camera_pose=model.get_RT(cam.uid))
            image = pkg["render"]
            Ll1 = torch.abs(image - gts[views[k]]).mean()
            ssim_value = fused_ssim(image.unsqueeze(0), gts[views[k]].unsqueeze(0))
            loss = (1.0 - lambda_dssim) * Ll1 + lambda_dssim * (1.0 - ssim_value)
            loss.backward()
            losses.append(loss.item())
            if iteration < iterations:
                model.optimizer.step()
                model.optimizer.zero_grad(set_to_none=True)
    return losses


def test_agrees_with_train_py_loop():
    """20 iterations against train.py's loop body with the random background, the drop-in render(), the mirror
    GaussianModel and PerPointAdam: losses and the pose table within 5e-5 (as sections 4.14 / 4.16).  Parameters and
    Adam moments are compared by their norm-wise relative error: the two paths' loss gradients differ in the last bits,
    and Adam turns such a difference on a near-zero gradient into a whole step of either sign, so single elements drift
    apart by up to a few learning rates, with the fixed background as well (DESIGN.md section 4.17 has both pairs'
    values; the bounds are five times the largest measured)."""
    sys.path.insert(0, os.path.join(ROOT, "shims"))
    from test_reference_loop import make_inputs
    sc, gts, cams = make_inputs(P=20_000, W=160, H=112, seed=57)
    n = 20
    views = [k % sc.n_views for k in range(n)]
    gm = I.GaussianModel.from_scene(sc, DEV)
    gm.training_setup_pp(I.optimization_defaults(iterations=1000))
    ref = random_bg_loop(gm, I.render, views, gts, cams, n)
    tr = I.JointTrainer(sc, DEV, gt_images=gts, cfg=_cfg(), use_graph=True)
    losses = []
    for v in views:
        tr.step(v)
        losses.append(float(tr.loss_value()))
    assert ref[-1] < ref[0]
    d_loss = max(abs(a - b) for a, b in zip(ref, losses))
    d_pose = float((tr.poses - gm.P.detach()).abs().max())
    assert d_loss < 5e-5 and d_pose < 5e-5, (d_loss, d_pose, ref, losses)
    nrel = lambda a, b: float(torch.linalg.vector_norm((a.reshape(-1) - b.reshape(-1)).double()) /
                              torch.linalg.vector_norm(b.reshape(-1).double()))
    st = gm.optimizer.state
    params, moments = {}, {}
    for k in KEYS:
        p = getattr(gm, gm._ATTR[k])
        params[k] = nrel(tr.view(tr.params, k), p.detach())
        moments[k + "_m"] = nrel(tr.view(tr.exp_avg, k), st[p]["exp_avg"])
        moments[k + "_v"] = nrel(tr.view(tr.exp_avg_sq, k), st[p]["exp_avg_sq"])
    moments["pose_m"] = nrel(tr.pose_m, st[gm.P]["exp_avg"])
    moments["pose_v"] = nrel(tr.pose_v, st[gm.P]["exp_avg_sq"])
    assert max(params.values()) < 5e-3, params          # measured <= 9.4e-4 (fixed background: 4.0e-4)
    assert max(moments.values()) < 0.25, moments         # measured <= 0.049 (fixed background: 0.022)


# ---- 3. a random background is a fixed background per iteration -------------------------------------------------------
def test_one_step_equals_fixed_background_of_first_draw():
    sc, gts = _scene()
    a = I.JointTrainer(sc, DEV, gt_images=gts, cfg=_cfg())
    first = _draws(1)[0].cpu()
    b = I.JointTrainer(dataclasses.replace(sc, bg=first), DEV, gt_images=gts, cfg=_cfg(random_background=False))
    a.step(1)
    b.step(1)
    torch.cuda.synchronize()
    assert torch.equal(a._single.bg.cpu(), first)
    assert torch.equal(a.color, b.color) and torch.equal(a.sums, b.sums)
    _assert_equal(a, b)
    # and the scene's own background stays what render() and evaluate() use
    assert torch.equal(a.ident.bg.cpu(), sc.bg)


# ---- 4. eager against graph replay ------------------------------------------------------------------------------------
@pytest.mark.parametrize("V", [1, 3])
def test_eager_equals_replay_across_sh_degree_step(V):
    sc, gts = _scene(sh_degree=0)
    cfg = lambda: _cfg(sh_increase_interval=8)       # degree steps at iterations 8, 16 and 24
    a = I.JointTrainer(sc, DEV, gt_images=gts, cfg=cfg(), use_graph=False)
    b = I.JointTrainer(sc, DEV, gt_images=gts, cfg=cfg(), use_graph=True)
    for k in range(30 // V):
        for tr in (a, b):
            tr.step_batch([0, 1, 2]) if V > 1 else tr.step(k % 3)
        if V > 1:
            assert torch.equal(a._batch.frame.color, b._batch.frame.color) and torch.equal(a._batch_sums, b._batch_sums)
        else:
            assert torch.equal(a.color, b.color) and torch.equal(a.sums, b.sums), k
    torch.cuda.synchronize()
    assert b._graphs and a.active_sh_degree == 3
    _assert_equal(a, b)
    assert torch.equal(a.background_generator.get_state(), b.background_generator.get_state())


# ---- 5. the repeat after a binning overflow --------------------------------------------------------------------------
@pytest.mark.parametrize("use_graph", [False, True])
def test_overflow_repeat_keeps_its_colour(use_graph):
    sc, gts = _scene(P=20_000, W=160, H=112)
    n = 12

    def run(sabotage_at=None):
        tr = I.JointTrainer(sc, DEV, gt_images=gts, cfg=_cfg(), use_graph=use_graph)
        colours = []
        for k in range(n):
            if k == sabotage_at:
                tr.frame.alloc_binning(2000)
            tr.step(k % 3)
            colours.append(tr._single.bg.clone())
        torch.cuda.synchronize()
        return tr, torch.stack(colours)

    (ref, c_ref), (ovf, c_ovf) = run(), run(sabotage_at=7)
    assert ovf.overflows == 1 and ref.overflows == 0
    assert torch.equal(c_ovf, c_ref) and torch.equal(c_ref, _draws(n))
    _assert_equal(ref, ovf)
    fresh = torch.Generator(device=DEV).manual_seed(0)
    for _ in range(n):
        torch.rand(3, generator=fresh, device=DEV)
    assert torch.equal(ovf.background_generator.get_state(), fresh.get_state())   # one draw per iteration


# ---- 6. the view-batched kernels -------------------------------------------------------------------------------------
BATCH_MODES = {
    "plain": {},
    "densify_batches": dict(densify=True, densify_batches=True, densify_from_iter=10 ** 6, densify_until_iter=10 ** 6),
    "mip": dict(mip_kernel_size=0.1),
}


@pytest.mark.parametrize("mode", list(BATCH_MODES))
def test_step_batch_of_one_equals_step(mode):
    sc, gts = _scene()
    a = I.JointTrainer(sc, DEV, gt_images=gts, cfg=_cfg(**BATCH_MODES[mode]), use_graph=True)
    b = I.JointTrainer(sc, DEV, gt_images=gts, cfg=_cfg(**BATCH_MODES[mode]), use_graph=True)
    for k in range(6):
        a.step(k % 3)
        b.step_batch([k % 3])
        assert torch.equal(a.color, b._batch.frame.color[0]) and torch.equal(a.sums, b._batch_sums[0]), k
    torch.cuda.synchronize()
    _assert_equal(a, b)
    if a._stats is not None:
        assert torch.equal(a._stats, b._stats)


@pytest.mark.parametrize("mode", list(BATCH_MODES))
def test_batched_views_with_three_colours_equal_single_views(mode):
    """V = 3 views over three different colours: view k's image and loss equal a single-view forward over colour k;
    the view-summed gradients equal the single-view backwards added in view order, and each view's pose gradient
    (and, with densify_batches, the statistics) equal the single-view ones, bit for bit."""
    sc, gts = _scene()
    views = [2, 0, 1]
    a = I.JointTrainer(sc, DEV, gt_images=gts, cfg=_cfg(**BATCH_MODES[mode]))
    snap = {}
    a._after_backward = lambda: snap.update(grads=a.grads.clone(), pose_grad=a.pose_grad.clone())
    a.step_batch(views)
    colours = a._batch.bg.clone()
    assert len({tuple(c) for c in colours.tolist()}) == 3
    c = I.JointTrainer(sc, DEV, gt_images=gts, cfg=_cfg(**BATCH_MODES[mode], random_background=False))
    total, stats = None, c._stats is not None
    for k, v in enumerate(views):
        c.ident.bg.copy_(colours[k])
        c.render(v)
        assert torch.equal(c.color, a._batch.frame.color[k]), k
        c.loss_and_backward(v, gts[v], stats=stats)
        assert torch.equal(c.sums, a._batch_sums[k]), k
        assert torch.equal(c.pose_grad[v], snap["pose_grad"][v]), k
        total = c.grads.clone() if total is None else total + c.grads
    torch.cuda.synchronize()
    for name, _ in a._nonempty():
        assert torch.equal(a.view(snap["grads"], name), c.view(total, name)), name
    if stats:
        assert torch.equal(a._stats, c._stats) and int(c.denom.max()) == 3


# ---- 7. checkpoints --------------------------------------------------------------------------------------------------
def test_checkpoint_resume_continues_the_colours(tmp_path):
    sc, gts = _scene()
    a = I.JointTrainer(sc, DEV, gt_images=gts, cfg=_cfg(), use_graph=True)
    path = str(tmp_path / "chkpnt10.pth")
    for k in range(20):
        a.step(k % 3)
        if k == 9:
            a.save_checkpoint(path)
    model_args, it = torch.load(path, weights_only=True)
    extra = model_args[10][I.CHECKPOINT_KEY]
    assert it == 10 and extra["cfg"]["random_background"] is True
    assert torch.equal(extra["background_generator"], _gen_after(10).get_state())
    b = I.JointTrainer.from_checkpoint(path, sc, gt_images=gts, use_graph=True)
    assert b.cfg.random_background and b.iteration == 10
    for k in range(10, 20):
        b.step(k % 3)
    torch.cuda.synchronize()
    _assert_equal(a, b)
    assert torch.equal(a.background_generator.get_state(), b.background_generator.get_state())
    # a file without the generator state (any run without the option) starts the colours from the seed
    del extra["background_generator"]
    bare = str(tmp_path / "bare.pth")
    torch.save((model_args, it), bare)
    c = I.JointTrainer.from_checkpoint(bare, sc, gt_images=gts, cfg=_cfg(background_seed=5))
    assert torch.equal(c.background_generator.get_state(), torch.Generator(device=DEV).manual_seed(5).get_state())


def _gen_after(n, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    for _ in range(n):
        torch.rand(3, generator=g, device=DEV)
    return g


def test_checkpoint_without_the_option_has_no_generator(tmp_path):
    sc, gts = _scene()
    tr = I.JointTrainer(sc, DEV, gt_images=gts, cfg=_cfg(random_background=False))
    tr.step(0)
    path = str(tmp_path / "c.pth")
    tr.save_checkpoint(path)
    extra = torch.load(path, weights_only=True)[0][10][I.CHECKPOINT_KEY]
    assert "background_generator" not in extra and tr.background_generator is None


# ---- 8. refusals -----------------------------------------------------------------------------------------------------
def test_blend_version_1_refuses_a_background_table():
    sc, gts = _scene()
    tr = I.JointTrainer(sc, DEV, gt_images=gts, cfg=_cfg())
    L = _lib.lib()
    assert L.gsb_set_option(b"blend_version", 1) == 0
    try:
        with pytest.raises(I.GsbError, match="blend version 1 takes one shared background"):
            tr.step_batch([0, 1])
        tr.render(0)                            # a shared background still renders on version 1
    finally:
        assert L.gsb_set_option(b"blend_version", 2) == 0
    with pytest.raises(I.GsbError, match=r"contiguous float32 \[2, 3\] CUDA tensor"):
        tr._batch.frame.render_batch(tr._camera(), None, torch.zeros(3, device=DEV))
