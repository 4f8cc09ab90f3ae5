"""The Mip filters' edge populations (tests/_mip.py) without a GPU: each builder reaches its regime in the fp64
restatement with the counts tests/test_mip_edges.py relies on, the flags cover every decision fp32 takes the other way,
the wrong variants the GPU test tells apart really differ from the restatement, and the kernels' own arithmetic
(tests/host_mip.cpp: gs_math.cuh compiled for the host) matches fp64 row by row, f = 0 included."""
import ctypes
import math

import numpy as np
import pytest
import torch

import _mip as MIP
from oracle import gs_oracle as O
from test_host_math import _cam, _fp
from test_mip_cpu import _host_lib

# share of a population's rows that may be flagged (their decision lies within fp32 rounding)
FLAG_SHARE = 0.05
# per-row bound of the host build against fp64 (per-Gaussian cotangents, no blend)
HOST_ROW_TOL = 2e-3
# the GPU test's per-row bound (tests/test_projection_edges.py ROW_TOL_EDGES): a variant must miss it
CAN_TELL_TOL = 5e-4


def cases():
    """(name, population, kappa) of every GPU case."""
    mixed = MIP.population_mixed()
    return [("h2", MIP.population_h2(), 0.1), ("mixed k0", mixed, 0.0), ("mixed k0.3", mixed, 0.3),
            ("mixed k4", mixed, 4.0), ("clamp", MIP.population_clamp(), 0.1), ("near", MIP.population_near(), 0.1),
            ("3d", MIP.population_3d(), 0.1), ("3d smod 0.5", MIP.population_3d(smod=0.5), 0.1)]


def records(pop, kappa, f3d="pop"):
    sc = pop["sc"]
    return MIP.mip_records(sc.params, sc.poses[0], MIP.camera_of_pop(pop), kappa,
                           pop["f3d"] if isinstance(f3d, str) else f3d)


# what each GPU case relies on
NEED = {
    "h2": dict(needles_clamped=290, needles_det0_fp32_le_0=30, straddle_clamped=100, straddle_free=100,
               frame_h2_gt_0_999=35, frame_big_rects=5, clamped_reaching_cutoff=400),
    "mixed k0": dict(visible=850), "mixed k0.3": dict(clamped=20), "mixed k4": dict(clamped=100),
    "clamp": dict(clamp_x=150, clamp_y=150, both=50),
    "near": dict(visible_below_0_25=150, behind_near=3, big_rects=10),
    "3d": dict(h3_below_cutoff=50, s_near_f=10, s_far_above_f=20, tiny_f_no_tiles=9, tiny_f0_h3_1=9,
               plain_f0_h3_1=30),
}
NEED["3d smod 0.5"] = NEED["3d"]


def test_populations_reach_their_regimes():
    for name, pop, kappa in cases():
        o = records(pop, kappa)
        got = MIP.reached(name, pop, kappa, o)
        short = {k: (got[k], v) for k, v in NEED[name].items() if not got[k] >= v}
        assert not short, (name, short, got)
        fl = MIP.edge_flags(o, kappa)
        assert int(fl.sum()) < FLAG_SHARE * pop["sc"].P, (name, int(fl.sum()))
        if name == "h2":
            assert got["straddle_r_off"] <= 0.0101 and got["subpixel_h2_min"] >= 0.05 - 1e-9
            assert got["subpixel_h2_max"] <= 0.9 + 1e-9
        if name == "mixed k0":               # no dilation: det1 is det0, r is exactly 1 on every visible row
            assert got["r_is_1"] == got["visible"], got
        if name.startswith("3d"):
            assert got["rho_min"] < 2e-3 and got["rho_max"] > 5e2 and got["per_axis_spread"] > 1.0, got


def test_flags_cover_every_fp32_decision(tmp_path_factory):
    """Every row whose h2-floor decision the host build takes the other way from fp64 is flagged, rows far from the
    floor are not, and a needle far below the floor is surely clamped rather than ill-conditioned."""
    L = _host_lib(tmp_path_factory)
    for name, pop, kappa in cases():
        if kappa is None:
            continue
        o = records(pop, kappa)
        geom, h2 = host_forward(L, pop, kappa, pop["f3d"])
        mf = MIP.mip_flags(o, kappa)
        vis = o["visible"] & torch.from_numpy(geom[:, 11] > 0)
        other = vis & (torch.from_numpy(h2[:, 1] > 0) != o["h2_clamp"])
        assert not bool((other & ~mf["h2_floor"]).any()), (name, torch.nonzero(other & ~mf["h2_floor"])[:8])
    # constructed rows (dilated a, b, c; kappa 0.1): r at the floor, 1 % above it, a needle far below it, an
    # ill-conditioned needle above it
    k = 0.1
    t_at = MIP.H2_MIN ** 0.5 * k / (1 - MIP.H2_MIN ** 0.5)           # isotropic a0 = c0 = t: sqrt(r) = t / (t + k)
    t_up = 1.01 ** 0.5 * MIP.H2_MIN ** 0.5 * k / (1 - 1.01 ** 0.5 * MIP.H2_MIN ** 0.5)
    abc = torch.tensor([[t_at + k, 0.0, t_at + k], [t_up + k, 0.0, t_up + k], [4.0 + k, 2.0 - 1e-9, 1.0 + k],
                        [4.0 + k, 2.0 - 1e-4, 1.0 + k]], dtype=torch.float64)
    f = MIP.mip_flags(dict(visible=torch.ones(4, dtype=torch.bool), cov2d=abc), k)
    assert f["h2_floor"].tolist() == [True, False, False, False], f
    assert f["sure_clamp"].tolist() == [False, False, True, False], f
    assert f["ill"].tolist() == [False, False, False, True], f


def _cotangent(P, vis, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(P, 9, generator=g, dtype=torch.float64) * vis[:, None]


def _fp64_grads(pop, kappa, f3d, ds, **variant):
    """fp64 gradients of sum(ds * (xy, conic, o_eff, rgb)) with respect to every raw parameter and the pose."""
    sc = pop["sc"]
    prm = {k: v.double().clone().requires_grad_(True) for k, v in sc.params.items()}
    pose = sc.poses[0].double().clone().requires_grad_(True)
    means, rots = O.pose_pretransform(prm["xyz"], prm["rotation"], pose)
    s, o = torch.exp(prm["scaling"]), torch.sigmoid(prm["opacity"]).reshape(-1)
    if f3d is not None:
        s, o = MIP.apply_filter3d(s, o, f3d.double(), variant.get("h3_grad", True))
    pr = MIP.project_mip(means, s, rots, o, torch.cat([prm["f_dc"], prm["f_rest"]], 1), MIP.camera_of_pop(pop),
                         kappa, floor_grad=variant.get("floor_grad", False))
    lo = (ds[:, 0:2] * pr["xy"]).sum() + (ds[:, 2:5] * pr["conic"]).sum() + (ds[:, 5] * pr["opacity"]).sum() \
        + (ds[:, 6:9] * pr["rgb"]).sum()
    lo.backward()
    out = {k: prm[k].grad for k in ("xyz", "scaling", "rotation", "opacity")}
    out["pose"] = pose.grad
    return out


def test_can_tell_variants_differ_from_restatement():
    """On the rows the GPU test uses, the wrong variants' gradients miss the restatement's by more than the GPU test's
    per-row bound: differentiating through sqrt(r) at the floor (h2 population, the clamped straddle rows; on the
    needles r is so small that sqrt(r) moves the gradient by less than the bound), dropping
    dh3 f^2 / s~^2 (3D population, rows with h3 < 0.99 that reach the cutoff)."""
    pop = MIP.population_h2()
    o = records(pop, 0.1)
    mf = MIP.mip_flags(o, 0.1)
    sel = o["h2_clamp"] & o["visible"] & (mf["r"] > 0) & ~MIP.edge_flags(o, 0.1) & MIP.group_mask(pop, "straddle")
    ds = _cotangent(pop["sc"].P, sel, 3)
    ref = _fp64_grads(pop, 0.1, None, ds)
    var = _fp64_grads(pop, 0.1, None, ds, floor_grad=True)
    e = torch.stack([MIP.row_errors(var[k], ref[k])[0] for k in ("xyz", "scaling", "rotation")], 1).amax(1)
    share = float((e[sel] > CAN_TELL_TOL).double().mean())
    assert int(sel.sum()) >= 100 and share > 0.9, (int(sel.sum()), share)
    pop = MIP.population_3d()
    o = records(pop, 0.1)
    sel = o["visible"] & (o["h3"] < 0.99) & (o["opacity"] * 255 >= 1.0) & ~MIP.edge_flags(o, 0.1)
    ds = _cotangent(pop["sc"].P, sel, 4)
    ref = _fp64_grads(pop, 0.1, pop["f3d"], ds)
    var = _fp64_grads(pop, 0.1, pop["f3d"], ds, h3_grad=False)
    e = MIP.row_errors(var["scaling"], ref["scaling"])[0]
    share = float((e[sel] > CAN_TELL_TOL).double().mean())
    assert int(sel.sum()) >= 100 and share > 0.9, (int(sel.sum()), share)


# ---- the kernels' arithmetic, compiled for the host ---------------------------------------------------------------
def _args(L, pop, kappa, f3d):
    sc = pop["sc"]
    h = _cam(sc, sc.sh_degree, MIP.camera_of_pop(pop, torch.float32))
    h.scale_mod = pop["smod"]
    np_in = {k: np.ascontiguousarray(v.float().numpy()) for k, v in sc.params.items()}
    fa = None if f3d is None else np.ascontiguousarray(f3d.float().numpy())
    keep = (np_in, fa)
    return keep, (ctypes.byref(h), sc.P, _fp(np_in["xyz"]), _fp(np_in["scaling"]), _fp(np_in["rotation"]),
                  _fp(np_in["opacity"]), _fp(np_in["f_dc"]), _fp(np_in["f_rest"]), int(kappa is not None),
                  ctypes.c_float(kappa or 0.0), None if fa is None else _fp(fa))


def host_forward(L, pop, kappa, f3d):
    P = pop["sc"].P
    geom, h2 = np.zeros((P, 12), np.float32), np.zeros((P, 2), np.float32)
    keep, args = _args(L, pop, kappa, f3d)
    L.host_project_mip(*args, _fp(geom), _fp(h2))
    return geom, h2


def host_backward(L, pop, kappa, f3d, ds):
    P = pop["sc"].P
    out = [np.zeros(sh, np.float32) for sh in ((P, 3), (P, 3), (P, 4), (P,), (7,))]
    keep, args = _args(L, pop, kappa, f3d)
    dsf = np.ascontiguousarray(ds.float().numpy())
    L.host_project_bwd_mip(*args, _fp(dsf), *(_fp(a) for a in out))
    return dict(zip(("xyz", "scaling", "rotation", "opacity", "pose"), (torch.from_numpy(a) for a in out)))


@pytest.mark.parametrize("case", ["h2", "mixed k0", "mixed k0.3", "mixed k4", "clamp", "near", "3d", "3d smod 0.5"])
def test_host_compiled_mip_math_matches_fp64_row_by_row(tmp_path_factory, case):
    L = _host_lib(tmp_path_factory)
    name, pop, kappa = next(c for c in cases() if c[0] == case)
    o = records(pop, kappa)
    geom, h2 = host_forward(L, pop, kappa, pop["f3d"])
    assert np.isfinite(geom).all() and np.isfinite(h2).all()
    fl = MIP.edge_flags(o, kappa)
    mf = MIP.mip_flags(o, kappa)
    vis = o["visible"] & torch.from_numpy(geom[:, 11] > 0)
    ok = vis & ~fl
    # record opacity o3 h2 per row (ill-conditioned rows on their own scale; an h3 below fp32's range is 0), conic on
    # its conditioning scale
    op = torch.from_numpy(geom[:, 5]).double()
    rel = (op - o["opacity"]).abs() / (o["opacity"].abs() + 1e-30)
    assert float(rel[ok & ~mf["ill"]].max()) < 2e-5, float(rel[ok].max())
    a, b, c = o["cov2d"].unbind(-1)
    cs = torch.maximum(o["conic"][:, 0].abs(), o["conic"][:, 2].abs()) * (a * c + b * b) / (a * c - b * b)
    conic = torch.from_numpy(geom[:, 2:5]).double()
    assert float(((conic - o["conic"]).abs().amax(1) / cs)[ok].max()) < 2e-5
    ds = _cotangent(pop["sc"].P, ok, 7)
    ref = _fp64_grads(pop, kappa, pop["f3d"], ds)
    mine = host_backward(L, pop, kappa, pop["f3d"], ds)
    worst = {}
    for k in ("xyz", "scaling", "rotation", "opacity"):
        assert bool(torch.isfinite(mine[k]).all()), k
        e, live = MIP.row_errors(mine[k], ref[k])
        worst[k] = float(e[ok & live].max())
    worst["pose"] = float((mine["pose"].double() - ref["pose"]).abs().max() / ref["pose"].abs().max())
    assert max(worst.values()) < HOST_ROW_TOL, (case, worst)


def test_host_f0_is_the_unfiltered_path(tmp_path_factory):
    """f = 0 is no 3D filter: forward and backward equal the unfiltered ones bit for bit, with and without the 2D
    filter -- also at log-scales of -52 and -60, where s*s is 0 in fp32 and (s*s)/(s*s + f^2) used to be 0/0."""
    L = _host_lib(tmp_path_factory)
    pop = MIP.population_3d()
    P = pop["sc"].P
    zero = torch.zeros(P)
    for kappa in (None, 0.1):
        o = records(pop, kappa, None)
        ds = _cotangent(P, o["visible"], 9)
        g0, h0 = host_forward(L, pop, kappa, zero)
        g1, h1 = host_forward(L, pop, kappa, None)
        assert np.isfinite(g0).all() and np.array_equal(g0, g1) and np.array_equal(h0, h1), kappa
        b0, b1 = host_backward(L, pop, kappa, zero, ds), host_backward(L, pop, kappa, None, ds)
        for k in b0:
            assert bool(torch.isfinite(b0[k]).all()) and torch.equal(b0[k], b1[k]), (kappa, k)
    # the tiny rows in the population's own filter (f = 0 on them): h3 = 1, o_eff = sigma(logit) * sqrt(2.5e-5)
    geom, _ = host_forward(L, pop, 0.1, pop["f3d"])
    a, b = pop["groups"]["tiny_f0"]
    sig = torch.sigmoid(pop["sc"].params["opacity"][a:b, 0].double())
    assert torch.allclose(torch.from_numpy(geom[a:b, 5]).double(), sig * math.sqrt(MIP.H2_MIN), rtol=1e-6)
