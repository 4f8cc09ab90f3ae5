"""The Mip filters' per-Gaussian forward and backward (project_geometry<true>, project_bwd<true>) at the edges of their
regimes, checked Gaussian by Gaussian against the fp64 restatement of tests/_mip.py.

Each population of tests/_mip.py drives one regime -- h2 at its floor, within 1 % of it, sub-pixel and frame-filling;
kernel sizes 0, 0.3 and 4; the 2D filter with the frustum clamp and at the near plane; the 3D filter from f/s = 1e-3
to 1e3, log-scales whose square underflows in fp32, f = 0, scale_modifier 0.5 -- and is checked three ways:

* every record the forward stored (tests/_geom.py) against the fp64 record, opacity o3 h2 included;
* image and every gradient over the full frame, whole tensor and per Gaussian (99.9th percentile and maximum) on the
  rows whose decisions do not lie within fp32 rounding (`_mip.edge_flags`, counted and bounded);
* the regime was reached (`_mip.reached`; tests/test_mip_edges_cpu.py pins the counts without a GPU).

Where a wrong fp64 variant is close to the truth (a gradient through h2 at its floor, no gradient through h3) the
kernel must also be farther from the variant than the bound, and on the clamp, near-plane and h2 populations the
tracking (pose-only) backward and the full one must give the fp64 pose gradient.
"""
import math

import pytest
import torch

import _geom as GM
import _mip as MIP
from _parity import DEV, GRAD_TOL, NAMES, REPORT, assert_image, image_stats, rel_err, row_err, settings_for
from oracle import gs_oracle as O
from test_projection_edges import ROW_TOL_EDGES

pytestmark = pytest.mark.gpu

# per-Gaussian bounds on the unflagged rows: the 99.9th percentile at ROW_TOL_EDGES (2.9x the largest H100
# measurement here, 1.7e-4: h2 population, xyz); the maximum at 3.7x the largest measured one (2.2e-4, same row set).
# H100 80GB HBM3, 700 W power limit.
ROW_MAX_MIP = 8e-4
BG = torch.tensor([0.1, 0.2, 0.3])


def _inputs(pop, f3d):
    sc = pop["sc"]
    return sc, (pop["f3d"] if isinstance(f3d, str) else f3d)


def _kernel(pop, kappa, f3d, w, pose_only=False):
    """rasterize_fused of view 0 with the filters and sum(w * image) back-propagated -> (image, radii, grads, st)."""
    import instantsplat_b200 as I
    sc = pop["sc"]
    rs = settings_for(sc, sc.sh_degree, BG)._replace(scale_modifier=pop["smod"], kernel_size=kappa)
    prm = {k: v.to(DEV).clone().requires_grad_(not pose_only) for k, v in sc.params.items()}
    pose = sc.poses[0].to(DEV).clone().requires_grad_(True)
    img, radii = I.rasterize_fused(prm["xyz"], prm["rotation"], prm["scaling"], prm["opacity"], prm["f_dc"],
                                   prm["f_rest"], pose, torch.zeros(sc.P, 3, device=DEV), rs,
                                   None if f3d is None else f3d.to(DEV))
    st = img.grad_fn.st
    (img * w.to(DEV)).sum().backward()
    g = {k: v.grad for k, v in prm.items()}
    g["pose"] = pose.grad
    return img.detach(), radii, g, st


def _oracle(pop, kappa, f3d, lists, **variant):
    sc = pop["sc"]
    po = {k: v.double().clone().requires_grad_(True) for k, v in sc.params.items()}
    pose = sc.poses[0].double().clone().requires_grad_(True)
    img, radii, aux = MIP.render_mip(po["xyz"], po["rotation"], po["scaling"], po["opacity"], po["f_dc"],
                                     po["f_rest"], pose, MIP.camera_of_pop(pop), kappa,
                                     None if f3d is None else f3d.double(), return_aux=True, lists=lists, **variant)

    def finish(w):
        (img * w.double()).sum().backward()
        g = {k: po[k].grad for k in po}
        g["pose"] = pose.grad
        return g
    return img.detach(), radii, aux, finish


def check_mip(name, pop, kappa, f3d="pop", pose_check=False, variant=None, row_tol=ROW_TOL_EDGES,
              row_max=ROW_MAX_MIP):
    """One population against the fp64 restatement: image, records, whole-tensor and per-row gradients, zero gradients
    of rows without tiles; optionally the pose-only backward's pose gradient, and the distance from a wrong variant
    (variant = (kwargs of render_mip, row mask)).  -> record (also appended to the session's report)."""
    sc, f3d = _inputs(pop, f3d)
    P = sc.P
    with torch.no_grad():       # tile lists of the fp32 projection
        p = sc.params
        means, rots = O.pose_pretransform(p["xyz"], p["rotation"], sc.poses[0])
        s, o = torch.exp(p["scaling"]), torch.sigmoid(p["opacity"]).reshape(-1)
        if f3d is not None:
            s, o = MIP.apply_filter3d(s, o, f3d)
        lists = O.build_tile_lists(MIP.project_mip(means, s, rots, o, torch.cat([p["f_dc"], p["f_rest"]], 1),
                                                   MIP.camera_of_pop(pop, torch.float32), kappa))
    img_o, radii_o, aux, finish = _oracle(pop, kappa, f3d, lists)
    amb = aux["ambiguous"]
    w = torch.rand(3, sc.height, sc.width, generator=torch.Generator().manual_seed(11)) * (~amb)[None]
    g_o = finish(w)
    img_c, radii_c, g_c, st = _kernel(pop, kappa, f3d, w)
    stats = image_stats(img_c, img_o, amb)
    rec = dict(case=f"mip edges: {name}", P=P, width=sc.width, height=sc.height, kernel_size=kappa,
               scale_modifier=pop["smod"], filter3D=f3d is not None, **stats,
               radii_mismatch_frac=float((radii_c.cpu() != radii_o).float().mean()))
    # ---- records
    o = MIP.mip_records(sc.params, sc.poses[0], MIP.camera_of_pop(pop), kappa, f3d)
    d = GM.decode(st)
    mf = MIP.mip_flags(o, kappa)
    fl = MIP.edge_flags(o, kappa)
    # the record opacity of an ill-conditioned row is bounded on the scale of its conditioning, one whose h3 lies below
    # fp32's range (log-scales <= -45 under a filter f > 0) by 1e-30; both are then taken as the kernel's
    rel = (d["opacity"] - o["opacity"]).abs() / o["opacity"].abs().clamp(min=1e-300)
    ill, tiny = mf["ill"], o["opacity"] < 1e-30
    assert bool((rel[ill] <= 2e-5 + 2e-7 * mf["cond"][ill]).all()), name
    assert bool((d["opacity"][tiny] < 1e-30).all()), name
    o["opacity"] = torch.where(ill | tiny, d["opacity"], o["opacity"])
    rec["records"] = GM.check_records(d, o)
    rec["reached"] = MIP.reached(name, pop, kappa, o) if name in REACHED else {}
    rec["flagged"] = dict(h2_floor=int(mf["h2_floor"].sum()), ill=int(ill.sum()), any=int(fl.sum()),
                          below_fp32_range=int((tiny & o["visible"]).sum()))
    # ---- gradients
    names = NAMES + ("pose",)
    ge = {k: rel_err(g_c[k], g_o[k]) for k in names}
    ok = ~fl
    rows = {k: row_err(g_c[k][ok.to(DEV)], g_o[k][ok]) for k in NAMES}
    rec.update(grad_rel_err=ge, grad_row_err=rows, grad_row_err_p999_max=max(r["p999"] for r in rows.values()),
               grad_row_err_max=max(r["max"] for r in rows.values()))
    dead = (d["radii"] == 0) | (d["tiles"] == 0)
    zc = GM.zero_rows({k: g_c[k] for k in NAMES}, dead)
    gf = GM.flags(o)
    sure = dead & ~gf["visibility"] & ~gf["rect"] & ~gf["cutoff"]
    zo = GM.zero_rows({k: g_o[k] for k in NAMES}, sure)
    rec["dead"] = int(dead.sum())
    if pose_check:
        _, _, g_t, _ = _kernel(pop, kappa, f3d, w, pose_only=True)
        rec["pose_only_rel_err"] = rel_err(g_t["pose"], g_o["pose"])
        rec["pose_only_vs_full"] = rel_err(g_t["pose"], g_c["pose"])
        assert all(v is None for k, v in g_t.items() if k != "pose")
    if variant is not None:
        kw, sel = variant
        _, _, _, fin_v = _oracle(pop, kappa, f3d, lists, **kw)
        g_v = fin_v(w)
        e = torch.stack([MIP.row_errors(g_c[k], g_v[k])[0] for k in ("xyz", "rotation", "scaling")], 1).amax(1)
        live = torch.stack([MIP.row_errors(g_c[k], g_o[k])[1] for k in ("xyz", "rotation", "scaling")], 1).any(1)
        sel = sel & ok & live
        rec["can_tell"] = dict(variant=str(kw), rows=int(sel.sum()),
                               share_beyond_bound=float((e[sel] > row_tol).double().mean()) if bool(sel.any()) else 0.0)
    REPORT.append(rec)
    # ---- assertions
    assert_image(stats, rec["case"])
    assert rec["radii_mismatch_frac"] < 2e-3, rec
    assert int(fl.sum()) < 0.05 * P, rec["flagged"]
    assert max(ge.values()) < GRAD_TOL, (name, ge)
    bad = {k: r for k, r in rows.items() if not (r["p999"] <= row_tol and r["max"] <= row_max)}
    assert not bad, f"{name}: per-Gaussian gradient errors over {row_tol} (p99.9) / {row_max} (max): {bad}"
    assert max(zc.values()) == 0.0, f"{name}: Gaussians without tiles have a gradient: {zc}"
    assert max(zo.values()) == 0.0, f"{name}: the fp64 side has a gradient for Gaussians the kernel gave no tiles: {zo}"
    for k in NAMES:
        assert bool(torch.isfinite(g_c[k]).all()), (name, k)
    if pose_check:
        assert rec["pose_only_rel_err"] < GRAD_TOL and ge["pose"] < GRAD_TOL, rec
        assert rec["pose_only_vs_full"] < 1e-5, rec
    if variant is not None:
        assert rec["can_tell"]["rows"] >= 30 and rec["can_tell"]["share_beyond_bound"] > 0.6, rec["can_tell"]
    return rec, o, d


REACHED = ("h2", "mixed k0", "mixed k0.3", "mixed k4", "clamp", "near", "3d", "3d smod 0.5")


def test_h2_regimes():
    """kernel_size 0.1: needles far below the floor, r within 1 % of it, h2 from 0.05 to 0.9, frame-filling
    Gaussians (k_big_rects); the gradient through sqrt(r) is cut exactly at the floor."""
    pop = MIP.population_h2()
    o = MIP.mip_records(pop["sc"].params, pop["sc"].poses[0], MIP.camera_of_pop(pop), 0.1, None)
    straddle = o["h2_clamp"] & MIP.group_mask(pop, "straddle")
    rec, o, d = check_mip("h2", pop, 0.1, pose_check=True, variant=(dict(floor_grad=True), straddle))
    r = rec["reached"]
    assert r["needles_clamped"] >= 290 and r["straddle_clamped"] >= 100 and r["straddle_free"] >= 100, r
    assert r["frame_h2_gt_0_999"] >= 35 and d["n_big"] >= 5, (r, d["n_big"])
    # the floored rows reach alpha 1/255 somewhere: their gradient is checked, not zero on both sides
    fl = MIP.group_mask(pop, "needles", "straddle") & (d["tiles"] > 0)
    assert int(fl.sum()) >= 400


@pytest.mark.parametrize("kappa", [0.0, 0.3, 4.0])
def test_kernel_sizes(kappa):
    """One mixed population (sigma 0.02-8 px) at kernel sizes 0 (r exactly 1), 0.3 and 4 (ordinary Gaussians at the
    floor)."""
    pop = MIP.population_mixed()
    rec, o, d = check_mip(f"mixed k{kappa:g}", pop, kappa)
    r = rec["reached"]
    if kappa == 0.0:
        assert r["r_is_1"] == r["visible"] >= 850, r
        # no dilation and no compensation: the record opacity is the activated one
        sig = torch.sigmoid(pop["sc"].params["opacity"].double()).reshape(-1)
        vis = d["radii"] > 0
        assert float(((d["opacity"] - sig).abs() / sig)[vis].max()) < 2e-6
    else:
        assert r["clamped"] >= (100 if kappa == 4.0 else 20), r


def test_frustum_clamp():
    pop = MIP.population_clamp()
    rec, _, _ = check_mip("clamp", pop, 0.1, pose_check=True)
    r = rec["reached"]
    assert r["clamp_x"] >= 150 and r["clamp_y"] >= 150 and r["both"] >= 50, r


def test_near_plane():
    pop = MIP.population_near()
    rec, _, d = check_mip("near", pop, 0.1, pose_check=True)
    r = rec["reached"]
    assert r["visible_below_0_25"] >= 150 and r["behind_near"] >= 3 and d["n_big"] >= 10, (r, d["n_big"])


@pytest.mark.parametrize("smod", [1.0, 0.5])
def test_filter3d(smod):
    """f/s from 1e-3 to 1e3 (per axis and on all axes), log-scales -45, -52, -60 with f > 0 (h3 = 0: no tiles, no
    gradient) and with f = 0 (h3 = 1); the gradient through h3 is there (a variant without it is told apart)."""
    pop = MIP.population_3d(smod=smod)
    o = MIP.mip_records(pop["sc"].params, pop["sc"].poses[0], MIP.camera_of_pop(pop), 0.1, pop["f3d"])
    sel = (o["h3"] < 0.99) & (pop["f3d"] > 0)
    name = "3d" if smod == 1.0 else "3d smod 0.5"
    rec, o, d = check_mip(name, pop, 0.1, variant=(dict(h3_grad=False), sel))
    r = rec["reached"]
    assert r["h3_below_cutoff"] >= 50 and r["s_near_f"] >= 10 and r["s_far_above_f"] >= 20, r
    a, b = pop["groups"]["tiny_f"]
    assert int(d["tiles"][a:b].count_nonzero()) == 0
    a, b = pop["groups"]["tiny_f0"]
    sig = torch.sigmoid(pop["sc"].params["opacity"][a:b, 0].double())
    assert torch.allclose(d["opacity"][a:b], sig * math.sqrt(MIP.H2_MIN), rtol=1e-6)
    assert int(d["tiles"][a:b].count_nonzero()) == b - a


@pytest.mark.parametrize("kappa", [None, 0.1])
def test_filter3d_zero_is_the_unfiltered_path(kappa):
    """f = 0 everywhere is no 3D filter, at log-scales of -52 and -60 too (s*s is 0 in fp32 there; (s*s)/(s*s + f^2)
    used to make the opacity NaN).  With the 2D filter both renders run the filtered kernels: image, radii and every
    gradient are equal bit for bit.  Without it the render without the 3D filter runs the reference instantiation of
    the per-Gaussian kernels instead, a separately compiled copy of the same arithmetic: equal to within rounding."""
    pop = MIP.population_3d()
    sc = pop["sc"]
    w = torch.rand(3, sc.height, sc.width, generator=torch.Generator().manual_seed(5))
    img0, radii0, g0, st0 = _kernel(pop, kappa, torch.zeros(sc.P), w)
    img1, radii1, g1, _ = _kernel(pop, kappa, None, w)
    d = GM.decode(st0)
    assert bool(torch.isfinite(d["opacity"]).all()) and bool(torch.isfinite(img0).all())
    assert torch.equal(radii0, radii1)
    rec = dict(case=f"mip edges: f = 0, kernel_size {kappa}", image_max_abs_diff=float((img0 - img1).abs().max()),
               grad_rel_diff={k: rel_err(g0[k], g1[k]) for k in g0})
    REPORT.append(rec)
    if kappa is not None:
        assert torch.equal(img0, img1)
        for k in g0:
            assert torch.equal(g0[k], g1[k]), k
    else:
        assert rec["image_max_abs_diff"] <= 1e-5 and max(rec["grad_rel_diff"].values()) <= 1e-4, rec
    a, b = pop["groups"]["tiny_f0"]
    assert int(d["tiles"][a:b].count_nonzero()) == b - a
