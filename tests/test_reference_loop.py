"""GPU side of "the reference's loop on the drop-ins" (-m gpu).  The reference tree is not a dependency, so the loop body
of train.py:140-211 is transcribed here and driven through the repo's mirror of the reference's
`GaussianModel` (instantsplat_b200/model.py; tests/test_reference_shims_cpu.py shows on the CPU, with the REAL reference
modules, that mirror == reference).  Three ways of running the same 20 iterations must give the same losses:

  dropin_unchanged  reference-shaped render body (PyTorch pose pre-transform, activations, feature cat) ->
                    GaussianRasterizer shim; torch l1 + fused_ssim shim; PerPointAdam drop-in
  dropin_fused      same loop with the fused render() (the two-line edit / the import hook)
  JointTrainer      flat buffers, fused loss, one Adam launch
"""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
DEV = "cuda"


def reference_loop(model, render, views, gts, cams, n_iters, first_iter=1, iterations=1000, lambda_dssim=0.2):
    """train.py:140-211, live lines only; `views[k]` replaces the random camera pick."""
    from fused_ssim import fused_ssim          # the shim, as train.py:39-43 imports it
    bg = torch.zeros(3, device=DEV)
    pipe = type("Pipe", (), dict(convert_SHs_python=False, compute_cov3D_python=False, debug=False))()
    losses = []
    for k in range(n_iters):
        iteration = first_iter + k
        model.update_learning_rate(iteration)
        if iteration % 1000 == 0:
            model.oneupSHdegree()
        cam = cams[views[k]]
        pose = model.get_RT(cam.uid)
        pkg = render(cam, model, pipe, bg, camera_pose=pose)
        image = pkg["render"]
        gt_image = gts[views[k]]
        Ll1 = torch.abs(image - gt_image).mean()                               # utils/loss_utils.py:39-40
        ssim_value = fused_ssim(image.unsqueeze(0), gt_image.unsqueeze(0))
        loss = (1.0 - lambda_dssim) * Ll1 + lambda_dssim * (1.0 - ssim_value)
        loss.backward()
        losses.append(loss.item())
        if iteration < iterations:
            model.optimizer.step()
            model.optimizer.zero_grad(set_to_none=True)
    return losses


def make_inputs(P=40_000, n_views=3, W=320, H=192, seed=51):
    import instantsplat_b200 as I
    from instantsplat_b200.camera import SimpleCamera
    from instantsplat_b200.scenes import perturbed_copy, surface_scene
    sc = surface_scene(P, n_views, W, H, seed=seed, sh_degree=3)
    tgt = I.JointTrainer(sc, DEV)
    pp = perturbed_copy(sc, sigma=0.05)
    for k, kk in (("xyz", 3), ("f_dc", 3), ("opacity", 1), ("scaling", 3)):
        tgt.view(tgt.params, k).copy_(pp[k].reshape(sc.P, kk).to(DEV))
    gts = torch.stack([tgt.render(v).clone() for v in range(n_views)])
    cams = []
    for v in range(n_views):
        c = SimpleCamera(W, H, sc.fovx, sc.fovy, device=DEV)
        c.uid = v
        cams.append(c)
    return sc, gts, cams


def test_three_ways_of_running_the_loop_agree():
    sys.path.insert(0, os.path.join(ROOT, "shims"))
    import instantsplat_b200 as I
    import instantsplat_b200.renderer as RD
    sc, gts, cams = make_inputs()
    n = 20
    views = [k % sc.n_views for k in range(n)]
    args = I.optimization_defaults(iterations=1000)
    out = {}
    try:
        for name, fused in (("dropin_unchanged", False), ("dropin_fused", True)):
            RD.FUSED = fused
            gm = I.GaussianModel.from_scene(sc, DEV)
            gm.training_setup_pp(args)
            out[name] = reference_loop(gm, I.render, views, gts, cams, n)
    finally:
        RD.FUSED = True
    cfg = I.OptimConfig()
    cfg.iterations = 1000
    tr = I.JointTrainer(sc, DEV, gt_images=gts, cfg=cfg)
    lj = []
    for k in range(n):
        tr.step(views[k])
        lj.append(float(tr.loss_value()))
    out["JointTrainer"] = lj
    ref = out["dropin_unchanged"]
    assert ref[-1] < 0.97 * ref[0], "the loop is expected to learn"
    for name in ("dropin_fused", "JointTrainer"):
        d = max(abs(a - b) for a, b in zip(ref, out[name]))
        assert d < 1e-5, (name, d, ref, out[name])
    # the last iteration of a schedule takes no optimizer step (train.py:209-211)
    p_before = tr.params.clone()
    tr.iteration = cfg.iterations - 1
    tr.step(0)
    assert torch.equal(tr.params, p_before)


def test_sh_degree_schedule_matches_the_reference():
    """oneupSHdegree every 1000 iterations (train.py:146-147): JointTrainer.active_sh_degree follows the same schedule
    as the mirror model, and the renders with the raised degree agree."""
    import instantsplat_b200 as I
    sc, gts, cams = make_inputs(P=8000, W=160, H=96, seed=52)
    sc.sh_degree = 1
    tr = I.JointTrainer(sc, DEV, gt_images=gts)
    assert tr.active_sh_degree == 1
    tr.iteration = 998
    tr.step(0)
    assert tr.active_sh_degree == 1 and tr.iteration == 999
    tr.step(1)
    assert tr.active_sh_degree == 2 and tr.iteration == 1000
    tr.iteration = 2999
    tr.step(2)
    assert tr.active_sh_degree == 3
    tr.iteration = 3999
    tr.step(0)
    assert tr.active_sh_degree == 3          # capped at max_sh_degree


def test_densify_prune_reset_state_surgery_vs_reference_golden(golden_dir):
    """Row f4: the same script as oracle/make_golden_surgery.py (two Adam steps, prune, step, append, step, opacity
    reset, step -- run there on the REFERENCE's GaussianModel + PerPointAdam on CPU) replayed on (a) JointTrainer's
    flat buffers and (b) the mirror GaussianModel + PerPointAdam drop-in; parameters and both Adam moments must land on
    the reference's vectors after every stage."""
    import numpy as np
    import instantsplat_b200 as I
    from instantsplat_b200.scenes import surface_scene
    z = np.load(os.path.join(golden_dir, "surgery.npz"))
    sc = surface_scene(60, 2, 32, 32, seed=13, sh_degree=3)
    for k in ("xyz", "f_dc", "opacity"):
        assert np.array_equal(sc.params[k].numpy(), z["init_" + k])
    KEYS = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")
    T = lambda a: torch.from_numpy(np.asarray(a)).to(DEV)

    def close(a, ref, what):
        np.testing.assert_allclose(a.detach().cpu().numpy().reshape(ref.shape), ref, rtol=4e-6, atol=2e-7, err_msg=what)

    # ---- (a) JointTrainer
    cfg = I.OptimConfig()
    cfg.iterations = 1000
    tr = I.JointTrainer(sc, DEV, cfg=cfg)
    tr.cfg.optim_pose = False

    def tr_step(tag):
        tr.iteration = int(z[f"{tag}_iteration"])
        for k in KEYS:
            tr.view(tr.grads, k).copy_(T(z[f"{tag}_g_{k}"]).reshape(tr.P, -1))
        tr.optimizer_step()
        for k in KEYS:
            close(tr.view(tr.params, k), z[f"{tag}_p_{k}"], f"trainer {tag} p {k}")
            close(tr.view(tr.exp_avg, k), z[f"{tag}_m_{k}"], f"trainer {tag} m {k}")
            close(tr.view(tr.exp_avg_sq, k), z[f"{tag}_v_{k}"], f"trainer {tag} v {k}")

    tr_step("s1"); tr_step("s2")
    tr.prune_points(T(z["prune_mask"]))
    assert tr.P == int((~z["prune_mask"]).sum())
    tr_step("s3")
    tr.densification_postfix(T(z["new_xyz"]), T(z["new_f_dc"]), T(z["new_f_rest"]), T(z["new_opacity"]),
                             T(z["new_scaling"]), T(z["new_rotation"]), T(z["new_ppl"]))
    tr_step("s4")
    tr.reset_opacity()
    close(tr.view(tr.params, "opacity"), z["reset_opacity"], "trainer reset_opacity")
    tr_step("s5")
    # the resized trainer still renders and trains
    gts = torch.rand(2, 3, 32, 32, device=DEV)
    tr.gt = gts
    tr.step(0)
    assert torch.isfinite(tr.params).all() and tr.last_R > 0

    # ---- (b) mirror GaussianModel + PerPointAdam drop-in
    gm = I.GaussianModel.from_scene(sc, DEV)
    gm.training_setup_pp(I.optimization_defaults(iterations=1000))
    attr = gm._ATTR

    def gm_step(tag):
        gm.update_learning_rate(int(z[f"{tag}_iteration"]))
        for k in KEYS:
            p = getattr(gm, attr[k])
            p.grad = T(z[f"{tag}_g_{k}"]).reshape(p.shape).contiguous()
        gm.P.grad = None
        gm.optimizer.step()
        for k in KEYS:
            p = getattr(gm, attr[k])
            close(p, z[f"{tag}_p_{k}"], f"model {tag} p {k}")
            close(gm.optimizer.state[p]["exp_avg"], z[f"{tag}_m_{k}"], f"model {tag} m {k}")
            close(gm.optimizer.state[p]["exp_avg_sq"], z[f"{tag}_v_{k}"], f"model {tag} v {k}")

    gm_step("s1"); gm_step("s2")
    gm.prune_points(T(z["prune_mask"]))
    gm_step("s3")
    gm.densification_postfix(T(z["new_xyz"]), T(z["new_f_dc"]), T(z["new_f_rest"]), T(z["new_opacity"]),
                             T(z["new_scaling"]), T(z["new_rotation"]), T(z["new_ppl"]))
    gm_step("s4")
    gm.reset_opacity()
    close(gm._opacity, z["reset_opacity"], "model reset_opacity")
    gm_step("s5")
    assert gm.get_xyz.shape[0] == tr.P


def test_graph_replay_matches_eager_and_survives_overflow():
    """JointTrainer(use_graph=True) replays each view's iteration from a CUDA graph (step sizes through device memory,
    R never on the host).  Same losses as the eager trainer; and when the binning capacity is exceeded (forced here)
    the device-gated optimizer skips the update, the host notices lazily, enlarges the buffer and repeats the iteration
    -- in both launch modes -- ending where an undisturbed trainer ends."""
    import instantsplat_b200 as I
    sc, gts, cams = make_inputs(P=30_000, W=256, H=160, seed=53)
    n = 12
    views = [k % sc.n_views for k in range(n)]

    def run(use_graph, sabotage_at=None):
        tr = I.JointTrainer(sc, DEV, gt_images=gts, use_graph=use_graph)
        losses = []
        for k in range(n):
            if k == sabotage_at:
                tr._size_binning(0)                  # capacity 65536 instances: far below the real count
                assert tr.cap < tr.last_R
            tr.step(views[k])
            losses.append(float(tr.loss_value()))
        torch.cuda.synchronize()
        return tr, losses

    eager, l_eager = run(False)
    graph, l_graph = run(True)
    assert len(graph._graphs) >= sc.n_views, "every view should have been captured"
    assert max(abs(a - b) for a, b in zip(l_eager, l_graph)) < 1e-5, (l_eager, l_graph)
    assert graph.opt_step == eager.opt_step == n and graph.iteration == eager.iteration == n
    for use_graph in (False, True):
        tr, l_ovf = run(use_graph, sabotage_at=7)
        assert tr.overflows == 1 and tr.opt_step == n
        assert max(abs(a - b) for a, b in zip(l_eager, l_ovf)) < 1e-5, (use_graph, l_eager, l_ovf)
        # same trajectory up to atomic-order noise (a last-bit difference of a near-zero gradient becomes a full Adam
        # step of either sign, so individual parameters may differ by a few learning rates)
        diff = (tr.params - eager.params).abs()
        assert float((diff > 1e-3).float().mean()) < 2e-3 and float(diff.max()) < 0.3, \
            (float(diff.max()), float((diff > 1e-3).float().mean()))
