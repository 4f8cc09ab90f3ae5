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
3. Every gradient tensor is also compared row by row (one row per Gaussian, `row_err`): the whole-tensor metric
   divides by the tensor's largest gradient, so it cannot see an error confined to Gaussians with small gradients
   (deep in a list, behind low transmittance, seen through an edge tile).  The oracle computes the truth in fp64, so
   the per-row metric does not measure the oracle's own fp32 rounding.
4. Every forward's tile lists are checked exactly on all tiles (tests/_binning.py `check_lists`), not only on the
   compared ones, and its per-pixel state on the compared, unflagged pixels: final_T within IMG_TOL of the oracle's,
   and the last contributor (n_contrib) exactly.
5. Every case appends its numbers to a report that conftest.py writes at the end of the session.
"""
import math

import torch

from oracle import gs_oracle as O

import _binning as BL
import _blend as BD

DEV = "cuda"
NAMES = ("xyz", "rotation", "scaling", "opacity", "f_dc", "f_rest")
IMG_TOL = 1e-4
GRAD_TOL = 1e-3
ROW_TAU = 1e-3       # per-row metric: floor of the denominator, relative to the tensor's largest gradient
# bounds on the 99.9th percentile of the per-row error where it is asserted, set from H100 measurements with a margin
# (DESIGN.md section 2): random scenes on tile subsets, and the constructed one-tile scenes of test_binning_lists.py
ROW_TOL = 2e-3
ROW_TOL_SCENES = 1e-4
REPORT = []          # list of dicts, one per parity case


def rel_err(a, b):
    a, b = a.detach().cpu().double().reshape(-1), b.detach().cpu().double().reshape(-1)
    return float((a - b).abs().max() / (b.abs().max() + 1e-20))


def row_err(a, b, tau=ROW_TAU):
    """Per-Gaussian error of a gradient tensor (rows = first dimension): e_i = max|a_i - b_i| / (max|b_i| +
    tau * max|b|), over the rows where either arm is non-zero.  -> dict(rows, p50, p99, p999, max); the
    percentiles take the next higher sample, so an error shared by >= 0.1 % of the rows shows in p999."""
    import numpy as np
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    a, b = a.reshape(a.shape[0], -1), b.reshape(b.shape[0], -1)
    d = (a - b).abs().amax(1)
    m = b.abs().amax(1)
    live = (m > 0) | (a.abs().amax(1) > 0)
    e = (d / (m + tau * b.abs().max() + 1e-300))[live].numpy()
    if e.size == 0:
        return dict(rows=0, p50=0.0, p99=0.0, p999=0.0, max=0.0)
    q = np.quantile(e, [0.5, 0.99, 0.999], method="higher")
    return dict(rows=int(e.size), p50=float(q[0]), p99=float(q[1]), p999=float(q[2]), max=float(e.max()))


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


def _oracle_arm(sc, view, deg, bg, tiles):
    """fp64 oracle render of `view` (tiles: optional subset) -> (image, radii, aux, finish) where finish(w)
    back-propagates sum(w * image) and returns the gradients.  The tile lists (rects, depth order) are those of the
    fp32 projection, which the kernels share to within the ambiguities the lists checks allow; the blend and its
    gradients are computed in fp64."""
    lists = O.build_tile_lists(BL.oracle_proj(sc, view, deg))
    cam = O.Camera.instantsplat(sc.width, sc.height, sc.fovx, sc.fovy, bg=bg, sh_degree=deg, dtype=torch.float64)
    po = {k: v.double().clone().requires_grad_(True) for k, v in sc.params.items()}
    pose_o = sc.poses[view].double().clone().requires_grad_(True)
    m2o = torch.zeros(sc.P, 3, dtype=torch.float64, requires_grad=True)
    img_o, radii_o, aux = O.render_instantsplat(po["xyz"], po["rotation"], po["scaling"], po["opacity"], po["f_dc"],
                                                po["f_rest"], pose_o, cam, means2D=m2o, tiles=tiles, return_aux=True,
                                                lists=lists)

    def finish(w):
        (img_o * w.double()).sum().backward()
        g = {k: po[k].grad for k in po}
        g["pose"], g["means2D"] = pose_o.grad, m2o.grad
        return g
    return img_o, radii_o, aux, finish


def compare_fused(name, sc, view, deg, bg, gt=None, tiles=None, names=None, record=True, weight_seed=11,
                  row_tol=None, oracle_cache=None, state=None):
    """The InstantSplat path (`rasterize_fused`: raw parameters + pose) against `O.render_instantsplat` in fp64.
    gt given (full frame only) -> weights = dL/dimage of the training loss, and the CUDA loss kernels are checked
    too; otherwise seeded random weights on the compared tiles.  Every tile list of the CUDA forward is checked
    (`_binning.check_lists`).  row_tol: bound on the 99.9th percentile of the per-row gradient error of every tensor.
    oracle_cache: a dict that keeps the oracle arm of a random-weight comparison for the next call on the same scene,
    view and weights (e.g. the same frame under another blend kernel).  state: a dict that receives the CUDA forward's
    state `st`, its radii and both arms' gradients (`grads`, `grads_oracle`), for checks per Gaussian.  Returns the
    record."""
    import instantsplat_b200 as I
    if names is None:
        names = NAMES if deg > 0 else tuple(n for n in NAMES if n != "f_rest")
    if oracle_cache is not None and "img" in oracle_cache:
        assert gt is None
        img_o, radii_o, aux, g_o = (oracle_cache[k] for k in ("img", "radii", "aux", "grads"))
        finish = None
    else:
        img_o, radii_o, aux, finish = _oracle_arm(sc, view, deg, bg, tiles)
    img_o = img_o.detach()
    pc = {k: v.to(DEV).clone().requires_grad_(True) for k, v in sc.params.items()}
    pose_c = sc.poses[view].to(DEV).clone().requires_grad_(True)
    m2c = torch.zeros(sc.P, 3, device=DEV, requires_grad=True)
    img_c, radii_c = I.rasterize_fused(pc["xyz"], pc["rotation"], pc["scaling"], pc["opacity"], pc["f_dc"],
                                       pc["f_rest"], pose_c, m2c, settings_for(sc, deg, bg))
    lists_c = BL.decode(img_c.grad_fn.st)
    lists = BL.check_lists(lists_c)
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
    rec["lists"] = lists
    # per-pixel state of the forward: final_T, and n_contrib as the id of the last contributor (the kernel's culled
    # lists and the oracle's rect lists number their entries differently)
    ft_c, nc_c = BD.decode_image(img_c.grad_fn.st)
    sel = ~amb if mask is None else mask & ~amb
    last_c = BD.last_contributor(lists_c["ids"].cpu(), lists_c["ranges"].cpu(), nc_c, sc.width)
    last_o = BD.last_contributor(aux["gids"], aux["ranges"], aux["n_contrib"], sc.width)
    rec["final_T_max_abs_err"] = float((ft_c.double() - aux["final_T"].double()).abs()[sel].max())
    rec["n_contrib_mismatch"] = int((last_c != last_o)[sel].sum())
    rec["radii_mismatch_frac"] = float((radii_c.cpu() != radii_o).float().mean())
    # ---- weights
    if gt is not None:
        assert tiles is None
        im_o = img_o.clone().requires_grad_(True)
        loss_o = O.training_loss(im_o, gt.double())
        loss_o.backward()
        w = im_o.grad.clone()
        im_c = img_c.detach().clone().requires_grad_(True)
        loss_c = I.fused_training_loss(im_c, gt.to(DEV))
        loss_c.backward()
        err = (img_c.detach().cpu() - img_o).abs().max(0)[0]
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
    if finish is not None:
        g_o = finish(w)
        if oracle_cache is not None and gt is None:
            oracle_cache.update(img=img_o, radii=radii_o, aux=aux, grads=g_o)
    (img_c * w.float().to(DEV)).sum().backward()
    g_c = {k: pc[k].grad for k in pc}
    g_c["pose"], g_c["means2D"] = pose_c.grad, m2c.grad
    if state is not None:
        state.update(st=img_c.grad_fn.st, radii=radii_c, grads=g_c, grads_oracle=g_o)
    ge = {k: rel_err(g_c[k], g_o[k]) for k in names + ("pose", "means2D")}
    if "f_rest" not in names:
        assert int(pc["f_rest"].grad.count_nonzero()) == 0
    rec["grad_rel_err"] = ge
    rec["grad_rel_err_max"] = max(ge.values())
    rows = {k: row_err(g_c[k], g_o[k]) for k in names + ("means2D",)}
    rec["grad_row_err"] = rows
    rec["grad_row_err_p999_max"] = max(r["p999"] for r in rows.values())
    if record:
        REPORT.append(rec)
    assert_image(st, name)
    assert rec["final_T_max_abs_err"] <= IMG_TOL, f"{name}: final_T differs from the oracle's: {rec}"
    assert rec["n_contrib_mismatch"] == 0, f"{name}: the last contributor differs on {rec['n_contrib_mismatch']} pixels"
    assert rec["radii_mismatch_frac"] < 2e-3, rec
    bad = {k: v for k, v in ge.items() if not v < GRAD_TOL}
    assert not bad, f"{name}: gradient relative errors over {GRAD_TOL}: {bad} (all: {ge})"
    if row_tol is not None:
        bad = {k: r for k, r in rows.items() if not r["p999"] <= row_tol}
        assert not bad, f"{name}: per-Gaussian gradient errors (99.9th percentile) over {row_tol}: {bad}"
    return rec
