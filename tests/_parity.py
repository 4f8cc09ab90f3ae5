"""Shared machinery of the GPU parity tests: one comparison protocol, north_star tolerances, recorded results.

Protocol (BASELINE.json north_star: render <= 1e-4 max abs per pixel, gradients <= 1e-3 relative):

1. Both arms render the same seeded inputs (CUDA path through the C ABI / the reference-shaped boundary, CPU
   oracle).  Every pixel whose colour differs by more than 1e-4 must be one the ORACLE flagged as *threshold
   ambiguous* (a pair within fp32 rounding of alpha >= 1/255, T < 1e-4 or power > 0 -- SURVEY.md section 7
   "hard parts": such a pair may be kept by one implementation and skipped by another).  The number of such
   pixels is counted, bounded, and recorded.
2. Gradients are compared on a loss of the form sum(w * image) whose weights are ZERO on the oracle-flagged
   pixels in BOTH arms, so a legitimate flip cannot leak into the comparison; the tolerance stays 1e-3 for every
   tensor (no relaxation when a pixel flips).  When the weights are the real training-loss gradient dL/dimage
   (L1 + D-SSIM), the CUDA loss kernels' dL/dimage is compared with the oracle's as well.
3. Every case appends its numbers to a report that conftest.py writes at the end of the session.
"""
import math

import torch

from oracle import gs_oracle as O

DEV = "cuda"
NAMES = ("xyz", "rotation", "scaling", "opacity", "f_dc", "f_rest")
IMG_TOL = 1e-4
GRAD_TOL = 1e-3
REPORT = []          # list of dicts, one per parity case


def rel_err(a, b):
    a, b = a.detach().cpu().double().reshape(-1), b.detach().cpu().double().reshape(-1)
    return float((a - b).abs().max() / (b.abs().max() + 1e-20))


def settings_for(sc, deg, bg, debug=False):
    import instantsplat_b200 as I
    from instantsplat_b200.camera import projection_matrix
    return I.GaussianRasterizationSettings(
        image_height=sc.height, image_width=sc.width, tanfovx=math.tan(sc.fovx * 0.5),
        tanfovy=math.tan(sc.fovy * 0.5), bg=bg.to(DEV), scale_modifier=1.0,
        viewmatrix=torch.eye(4, device=DEV),
        projmatrix=projection_matrix(0.01, 100.0, sc.fovx, sc.fovy).t().contiguous().to(DEV),
        sh_degree=deg, campos=torch.zeros(3, device=DEV), prefiltered=False, debug=debug)


def flip_budget(npix):
    """How many compared pixels may exceed 1e-4 (all of them oracle-flagged): 1 in 20 000, at least 2.
    Measured rates are recorded in the session's parity report."""
    return max(2, int(5e-5 * npix))


def image_stats(img_c, img_o, amb, mask=None):
    """-> dict(n_pix, n_over_tol, n_flagged, n_unexplained, max_abs_err, max_abs_err_unflagged)."""
    err = (img_c.detach().cpu() - img_o.detach()).abs().max(0)[0]
    if mask is None:
        mask = torch.ones_like(err, dtype=torch.bool)
    err = err * mask
    bad = err > IMG_TOL
    flagged = amb & mask
    return dict(n_pix=int(mask.sum()), n_over_tol=int(bad.sum()), n_flagged=int(flagged.sum()),
                n_unexplained=int((bad & ~amb).sum()), max_abs_err=float(err.max()),
                max_abs_err_unflagged=float((err * (~amb)).max()))


def assert_image(stats, what=""):
    assert stats["n_unexplained"] == 0, \
        f"{what}: {stats['n_unexplained']} pixels over {IMG_TOL} not explained by threshold ambiguity ({stats})"
    assert stats["n_over_tol"] <= flip_budget(stats["n_pix"]), f"{what}: too many threshold flips ({stats})"
    assert stats["max_abs_err_unflagged"] <= IMG_TOL


def dilate(mask, r):
    m = mask[None, None].float()
    return torch.nn.functional.max_pool2d(m, 2 * r + 1, stride=1, padding=r)[0, 0] > 0


def compare_fused(name, sc, view, deg, bg, gt=None, tiles=None, names=None, record=True, weight_seed=11):
    """The InstantSplat path (`rasterize_fused`: raw parameters + pose) against `O.render_instantsplat`.
    gt given (full frame only) -> weights = dL/dimage of the training loss, and the CUDA loss kernels are checked
    too; otherwise seeded random weights on the compared tiles.  Returns the record."""
    import instantsplat_b200 as I
    if names is None:
        names = NAMES if deg > 0 else tuple(n for n in NAMES if n != "f_rest")
    cam = O.Camera.instantsplat(sc.width, sc.height, sc.fovx, sc.fovy, bg=bg, sh_degree=deg)
    po = {k: v.clone().requires_grad_(True) for k, v in sc.params.items()}
    pose_o = sc.poses[view].clone().requires_grad_(True)
    m2o = torch.zeros(sc.P, 3, requires_grad=True)
    img_o, radii_o, aux = O.render_instantsplat(po["xyz"], po["rotation"], po["scaling"], po["opacity"], po["f_dc"],
                                                po["f_rest"], pose_o, cam, means2D=m2o, tiles=tiles, return_aux=True)
    pc = {k: v.to(DEV).clone().requires_grad_(True) for k, v in sc.params.items()}
    pose_c = sc.poses[view].to(DEV).clone().requires_grad_(True)
    m2c = torch.zeros(sc.P, 3, device=DEV, requires_grad=True)
    img_c, radii_c = I.rasterize_fused(pc["xyz"], pc["rotation"], pc["scaling"], pc["opacity"], pc["f_dc"],
                                       pc["f_rest"], pose_c, m2c, settings_for(sc, deg, bg))
    mask = None
    if tiles is not None:
        gx = (sc.width + 15) // 16
        mask = torch.zeros(sc.height, sc.width, dtype=torch.bool)
        for t in tiles:
            ty, tx = divmod(t, gx)
            mask[ty * 16:(ty + 1) * 16, tx * 16:(tx + 1) * 16] = True
    amb = aux["ambiguous"]
    st = image_stats(img_c, img_o, amb, mask)
    rec = dict(case=name, P=sc.P, width=sc.width, height=sc.height, view=int(view), sh_degree=deg,
               tiles_compared=(len(tiles) if tiles is not None else ((sc.width + 15) // 16) * ((sc.height + 15) // 16)),
               **st)
    rec["radii_mismatch_frac"] = float((radii_c.cpu() != radii_o).float().mean())
    # ---- weights
    if gt is not None:
        assert tiles is None
        im_o = img_o.detach().clone().requires_grad_(True)
        loss_o = O.training_loss(im_o, gt)
        loss_o.backward()
        w = im_o.grad.clone()
        im_c = img_c.detach().clone().requires_grad_(True)
        loss_c = I.fused_training_loss(im_c, gt.to(DEV))
        loss_c.backward()
        err = (img_c.detach().cpu() - img_o.detach()).abs().max(0)[0]
        near_flip = dilate(err > IMG_TOL, 5)          # SSIM's 11x11 window spreads a flipped pixel over its neighbours
        keep = (~near_flip)[None].expand_as(w)
        rec["loss_abs_err"] = abs(float(loss_c) - float(loss_o))
        rec["loss_grad_rel_err"] = rel_err(im_c.grad.cpu() * keep, w * keep)
        assert rec["loss_abs_err"] < 2e-5 + 4e-3 * st["n_over_tol"] / st["n_pix"], rec
        assert rec["loss_grad_rel_err"] < 1e-4, rec
        w = w / w.abs().max()
    else:
        w = torch.rand(3, sc.height, sc.width, generator=torch.Generator().manual_seed(weight_seed))
        if mask is not None:
            w = w * mask
    w = w * (~amb)[None]                              # flagged pixels carry no weight in EITHER arm
    (img_o * w).sum().backward()
    (img_c * w.to(DEV)).sum().backward()
    ge = {k: rel_err(pc[k].grad, po[k].grad) for k in names}
    ge["pose"] = rel_err(pose_c.grad, pose_o.grad)
    ge["means2D"] = rel_err(m2c.grad, m2o.grad)
    if "f_rest" not in names:
        assert float(pc["f_rest"].grad.abs().max()) == 0.0
    rec["grad_rel_err"] = ge
    rec["grad_rel_err_max"] = max(ge.values())
    if record:
        REPORT.append(rec)
    assert_image(st, name)
    assert rec["radii_mismatch_frac"] < 2e-3, rec
    bad = {k: v for k, v in ge.items() if not v < GRAD_TOL}
    assert not bad, f"{name}: gradient relative errors over {GRAD_TOL}: {bad} (all: {ge})"
    return rec
