"""Pose-only tracking mode (-m gpu; SURVEY.md section 8 row f2): the device-resident loop of
instantsplat_b200/tracking.py against a CPU restatement of render.py:113-161 built from the oracle's
renderer and torch's own Adam + CosineAnnealingLR (the classes the reference instantiates)."""
import math

import pytest
import torch

from oracle import gs_oracle as O
from instantsplat_b200.scenes import surface_scene

pytestmark = pytest.mark.gpu
DEV = "cuda"


def reference_tracking(sc, view, gt, init_pose, num_iter, deg):
    """render.py:113-161 on the CPU oracle (l1_loss_mask: utils/loss_utils.py:17-23)."""
    cam = O.Camera.instantsplat(sc.width, sc.height, sc.fovx, sc.fovy, sh_degree=deg)
    p = {k: v.clone() for k, v in sc.params.items()}
    T = init_pose[-3:].clone().requires_grad_()
    q = init_pose[:4].clone().requires_grad_()
    opt = torch.optim.Adam([{"params": [T], "lr": 0.003}, {"params": [q], "lr": 0.001}], betas=(0.9, 0.999),
                           weight_decay=1e-4)
    sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, T_max=num_iter, eta_min=0.0001)
    cand_q, cand_T, best = q.clone().detach(), T.clone().detach(), float(1e20)
    losses = []
    for it in range(num_iter):
        img, _ = O.render_instantsplat(p["xyz"], p["rotation"], p["scaling"], p["opacity"], p["f_dc"], p["f_rest"],
                                       torch.cat([q, T]), cam)
        mask = (img > 0.0).float()
        loss = ((img - gt).abs() * mask).sum() / mask.sum()
        loss.backward()
        with torch.no_grad():
            opt.step()
            opt.zero_grad(set_to_none=True)
            losses.append(float(loss))
            if float(loss) < best:
                best = float(loss)
                cand_q, cand_T = q.clone().detach(), T.clone().detach()
        sched.step()
    return torch.cat([cand_q, cand_T]), best, losses, torch.cat([q, T]).detach()


def test_tracking_loop_matches_reference_restatement():
    from instantsplat_b200.tracking import PoseTracker, cosine_lr
    sc = surface_scene(6000, 3, 128, 96, seed=61, sh_degree=2)
    view, n_it = 1, 12
    cam = O.Camera.instantsplat(sc.width, sc.height, sc.fovx, sc.fovy, sh_degree=2)
    with torch.no_grad():
        gt, _ = O.render_instantsplat(sc.params["xyz"], sc.params["rotation"], sc.params["scaling"], sc.params["opacity"],
                                      sc.params["f_dc"], sc.params["f_rest"], sc.poses[view], cam)
    init = sc.poses[view] + torch.tensor([0.0, 0.004, -0.003, 0.002, 0.01, -0.008, 0.012])
    ref_pose, ref_best, ref_losses, ref_last = reference_tracking(sc, view, gt, init, n_it, 2)
    tr = PoseTracker(sc.params["xyz"], sc.params["rotation"], sc.params["scaling"], sc.params["opacity"], sc.params["f_dc"],
                     sc.params["f_rest"], sc.width, sc.height, sc.fovx, sc.fovy, sh_degree=2, device=DEV)
    pose, best, trace = tr.optimize(init, gt, num_iter=n_it, return_trace=True)
    # the schedule helper is the closed form of CosineAnnealingLR
    assert abs(cosine_lr(0.003, 5, n_it) - (1e-4 + (0.003 - 1e-4) * (1 + math.cos(math.pi * 5 / n_it)) / 2)) < 1e-12
    assert ref_losses[-1] < ref_losses[0], "tracking is expected to reduce the loss"
    dl = max(abs(a - float(b)) for a, b in zip(ref_losses, trace))
    assert dl < 2e-5, (dl, ref_losses, trace.tolist())
    assert abs(best - ref_best) < 2e-5
    assert float((pose - ref_pose).abs().max()) < 2e-4, (pose, ref_pose)
    # rendering at the optimised pose is closer to the target than at the initial one
    e0 = float((tr.render(init).cpu() - gt).abs().mean())
    e1 = float((tr.render(pose).cpu() - gt).abs().mean())
    assert e1 < e0


def test_masked_l1_kernel_matches_reference_formula():
    import ctypes
    from instantsplat_b200 import _lib
    L = _lib.lib()
    g = torch.Generator().manual_seed(0)
    # n < 4 runs only the scalar tail (no group of four), n = 5 one group and a tail
    for shape in ((3, 37, 53), (3, 64, 64), (1, 1, 1), (1, 1, 2), (3, 1, 1), (1, 1, 5)):
        img = torch.rand(*shape, generator=g) - 0.3       # some non-positive entries -> masked out
        gt = torch.rand(*shape, generator=g)
        a = img.clone().requires_grad_(True)
        mask = (a > 0.0).float()
        loss = ((a - gt).abs() * mask).sum() / mask.sum()      # utils/loss_utils.py:17-23
        loss.backward()
        ic, gc = img.to(DEV).contiguous(), gt.to(DEV).contiguous()
        sums = torch.zeros(2, dtype=torch.float64, device=DEV)
        dL = torch.empty_like(ic)
        _lib.check(L.gsb_l1_mask_fwd_bwd(shape[0], shape[1], shape[2], ic.data_ptr(), gc.data_ptr(), 0.0, sums.data_ptr(),
                                         dL.data_ptr(), _lib.stream_ptr()), "gsb_l1_mask_fwd_bwd")
        s = sums.cpu()
        assert abs(float(s[0] / s[1]) - float(loss)) < 1e-6 and float(s[1]) == float(mask.sum())
        assert float((dL.cpu() / float(s[1]) - a.grad).abs().max()) < 1e-9
