"""Restatements of the optimizer kernels' arithmetic, and their checks without a GPU.

`adam32` writes k_adam's documented arithmetic (gs_adam.cu) in numpy float32 one rounded operation at a time, with the
fp32 constants the kernel receives; `adam64` is the reference optimizer (oracle per_point_adam_step) in float64 given
the same constants; `adam_bounds` are the few fp32 roundings by which the kernel may differ from `adam64`.  The GPU
tests (test_optimizer_edges.py) compare every kernel case with both.  Here: the two restatements agree with each other
within those bounds, the reference's gate on NaN, Inf and -0.0, and tracking's cosine learning rates against torch's
recursive CosineAnnealingLR.
"""
import math

import numpy as np
import torch

from oracle import gs_oracle as O

F32, F64 = np.float32, np.float64
U = 2.0 ** -24                      # unit roundoff of fp32


def consts(beta1=0.9, beta2=0.999, eps=1e-15, weight_decay=0.0, grad_scale=1.0):
    """The fp32 constants k_adam receives (build_args in gs_adam.cu)."""
    return dict(b1=F32(beta1), omb1=F32(1.0 - beta1), b2=F32(beta2), omb2=F32(1.0 - beta2), eps=F32(eps),
                wd=F32(weight_decay), gscale=F32(grad_scale))


def gate32(g, p, c):
    """The kernel's whole-tensor gate: some element with g*g > 0 and no NaN (the reference's grad.norm() > 0)."""
    with np.errstate(all="ignore"):
        gd = (g.astype(F32) * c["gscale"]).astype(F32)
        if c["wd"] != 0:
            gd = (gd.astype(F64) + F64(c["wd"]) * p.astype(F64)).astype(F32)
        return bool(np.any(gd * gd > F32(0))) and not bool(np.any(np.isnan(gd)))


def adam32(p, g, m, v, step, c, lr_mul=None, gate=None):
    """One k_adam step in numpy float32: returns (p, m, v).  step: the step size (rounded to fp32 here, as the kernel
    does); lr_mul: the per-element per-row multiplier (float32) or None.  With weight decay the kernel's FMA is
    restated as a float64 sum rounded once to fp32, which may differ from it by one rounding: compare with a bound."""
    p, g, m, v = (np.asarray(x, dtype=F32) for x in (p, g, m, v))
    if gate is None:
        gate = gate32(g, p, c)
    with np.errstate(all="ignore"):
        g = g * c["gscale"]
        if c["wd"] != 0:
            g = (F64(c["wd"]) * p.astype(F64) + g.astype(F64)).astype(F32)
        if gate:
            m = m * c["b1"] + g * c["omb1"]
            v = v * c["b2"] + (c["omb2"] * g) * g
        denom = np.sqrt(v) + c["eps"]
        upd = m / denom
        s = F32(step) if lr_mul is None else F32(step) * np.asarray(lr_mul, dtype=F32)
        p = p + (-s) * upd
    return p.astype(F32), m.astype(F32), v.astype(F32)


def adam64(p, g, m, v, step, c, ppl=None):
    """The reference optimizer (oracle per_point_adam_step) in float64 on the kernel's fp32 constants: it is given
    beta = 1 - (1-beta)_32, so its (1 - beta) is the kernel's constant and its beta is within half an fp32 ulp of the
    kernel's, and the lr that makes its bias-corrected step size `step` (rounded to fp32).  ppl: the per-row
    multiplier shaped [rows, 1, ...] like the parameter, or None.  Returns (p, m, v) as float64 arrays."""
    b1, b2 = 1.0 - F64(c["omb1"]), 1.0 - F64(c["omb2"])
    t = lambda x: torch.from_numpy(np.array(x, dtype=F64))
    p64, m64, v64 = t(p), t(m), t(v)
    g64 = t(g) * F64(c["gscale"])
    lr = F64(F32(step)) * (1.0 - b1) / math.sqrt(1.0 - b2)        # step 1: lr * sqrt(bc2) / bc1 == step
    with np.errstate(all="ignore"):
        O.per_point_adam_step(p64, g64, m64, v64, 1, lr, beta1=b1, beta2=b2, eps=F64(c["eps"]),
                              weight_decay=F64(c["wd"]), per_point_lr=None if ppl is None else t(ppl))
    return p64.numpy(), m64.numpy(), v64.numpy()


def adam_bounds(p, g, m, v, step, c, lr_mul=None):
    """Per-element bounds on |kernel - adam64| for m, v, p, from the terms that form them, in units u = 2^-24 (an fp32
    rounding is within u of its value).  m: its three roundings and the half-ulp gap between the kernel's beta and
    adam64's, 4u.  v: one more rounding, and the scaled gradient's own enters squared, 5u.  p: the final rounding,
    u (|p| + |update|), plus the update's chain (m, sqrt, eps, divide, step times multiplier, multiply), 10u of the
    largest update the terms allow: the moments may cancel and the bound must not shrink with them."""
    p, g, m, v = (np.asarray(x, dtype=F64) for x in (p, g, m, v))
    with np.errstate(all="ignore"):
        gd = g * F64(c["gscale"]) + F64(c["wd"]) * p
        gate = gate32(np.asarray(g, F32), np.asarray(p, F32), c)
        tm = np.abs(F64(c["b1"]) * m) + (np.abs(F64(c["omb1"]) * gd) if gate else 0.0)
        tv = np.abs(F64(c["b2"]) * v) + (F64(c["omb2"]) * gd * gd if gate else 0.0)
        vn = F64(c["b2"]) * v + F64(c["omb2"]) * gd * gd if gate else v
        s = abs(F64(F32(step))) * (1.0 if lr_mul is None else np.abs(np.asarray(lr_mul, F64)))
        dmax = s * tm / (np.sqrt(vn) + F64(c["eps"]))
        return 4 * U * tm, 5 * U * tv, U * (np.abs(p) + 10 * dmax)


def close_within(kern, ref, bound):
    """kernel values within `bound` of the float64 reference; non-finite entries must agree in position (and
    infinities in sign)."""
    kern, ref = np.asarray(kern, F64), np.asarray(ref, F64)
    fk, fr = np.isfinite(kern), np.isfinite(ref)
    if not np.array_equal(fk, fr) or not np.array_equal(np.isnan(kern), np.isnan(ref)):
        return False
    inf = ~fk & ~np.isnan(kern)
    if not np.array_equal(kern[inf], ref[inf]):
        return False
    bound = np.broadcast_to(bound, kern.shape)
    return bool(np.all(np.abs(kern[fk] - ref[fk]) <= bound[fk]))


def same_bits(a, b):
    """Bit-identical fp32 arrays, except that any NaN equals any NaN (payloads differ between CPU and GPU)."""
    a, b = np.ascontiguousarray(a, F32), np.ascontiguousarray(b, F32)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32),
                                                                              b[~nb].view(np.uint32))


# ------------------------------------------------------------------------------------------------------------------
def _case(n, seed, scale=1.0):
    r = np.random.default_rng(seed)
    p = r.standard_normal(n).astype(F32)
    g = (r.standard_normal(n) * scale).astype(F32)
    m = (r.standard_normal(n) * 0.1).astype(F32)
    v = (r.random(n) * 0.01).astype(F32)
    return p, g, m, v


def test_restatements_agree_within_bounds():
    for seed, (wd, gs, eps, scale) in enumerate([(0.0, 1.0, 1e-15, 1.0), (1e-2, 1.0, 1e-8, 1e-3),
                                                   (0.0, 1 / 3, 1e-15, 1e2), (0.0, 0.125, 1e-8, 1e-6)]):
        p, g, m, v = _case(4099, seed, scale)
        c = consts(weight_decay=wd, grad_scale=gs, eps=eps)
        step = 1e-3 * math.sqrt(1 - 0.999 ** 3) / (1 - 0.9 ** 3)
        k = adam32(p, g, m, v, step, c)
        r = adam64(p, g, m, v, step, c)
        bm, bv, bp = adam_bounds(p, g, m, v, step, c)
        for x, y, b in zip(k, r, (bp, bm, bv)):
            assert close_within(x, y, b)


def test_restatements_agree_with_per_row_multiplier():
    p, g, m, v = _case(7 * 300, 9)
    ppl = np.random.default_rng(1).uniform(0.25, 4.0, 300).astype(F32)
    c = consts()
    lm = np.repeat(ppl, 7)
    k = adam32(p, g, m, v, 2e-2, c, lr_mul=lm)
    r = adam64(p.reshape(300, 7), g.reshape(300, 7), m.reshape(300, 7), v.reshape(300, 7), 2e-2, c,
               ppl=ppl.reshape(300, 1))
    bm, bv, bp = adam_bounds(p, g, m, v, 2e-2, c, lr_mul=lm)
    for x, y, b in zip(k, r, (bp, bm, bv)):
        assert close_within(x, y.reshape(-1), b)


def test_bounds_see_a_wrong_multiplier_and_a_stale_gate():
    """The float64 arm must fail on the errors it exists for: a multiplier taken from the wrong row, moments updated
    when the gate is false."""
    p, g, m, v = _case(3 * 64, 4)
    ppl = np.random.default_rng(2).uniform(0.5, 2.0, 64).astype(F32)
    c = consts()
    lm = np.repeat(ppl, 3)
    wrong = lm.reshape(-1, 4)[:, :1].repeat(4, 1).reshape(-1)         # one multiplier per float4 group
    kp = adam32(p, g, m, v, 1e-2, c, lr_mul=wrong)[0]
    r = adam64(p.reshape(64, 3), g.reshape(64, 3), m.reshape(64, 3), v.reshape(64, 3), 1e-2, c, ppl=ppl[:, None])
    assert not close_within(kp, r[0].reshape(-1), adam_bounds(p, g, m, v, 1e-2, c, lr_mul=lm)[2])
    z = np.zeros_like(g)
    km = adam32(p, z, m, v, 1e-2, c, gate=True)[1]
    assert not close_within(km, adam64(p, z, m, v, 1e-2, c)[1], adam_bounds(p, z, m, v, 1e-2, c)[0])


def test_reference_gate_on_nan_inf_and_negative_zero():
    """grad.norm() > 0: a NaN anywhere freezes both moments (the parameter still moves, finitely); an Inf opens the
    gate; -0.0 everywhere keeps it shut.  gate32 states the same rule."""
    p, g, m, v = _case(8, 3)
    c = consts()
    gn = g.copy()
    gn[5] = np.nan
    pn, mn, vn = adam64(p, gn, m, v, 1e-2, c)
    assert np.array_equal(mn, m.astype(F64)) and np.array_equal(vn, v.astype(F64)) and np.all(np.isfinite(pn))
    assert not np.array_equal(pn, p.astype(F64))
    assert not gate32(gn, p, c)
    gi = np.zeros_like(g)
    gi[2] = np.inf
    assert gate32(gi, p, c)
    pi, mi, vi = adam64(p, gi, m, v, 1e-2, c)
    assert np.isinf(mi[2]) and np.isinf(vi[2]) and np.isnan(pi[2]) and np.all(np.isfinite(pi[np.arange(8) != 2]))
    nz = np.full(8, -0.0, F32)
    assert not gate32(nz, p, c)
    _, mz, vz = adam64(p, nz, m, v, 1e-2, c)
    assert np.array_equal(mz, m.astype(F64)) and np.array_equal(vz, v.astype(F64))
    assert gate32(np.zeros(8, F32), p, consts(weight_decay=1e-3))


def test_cosine_lr_matches_torch_scheduler_over_500_steps():
    """tracking.cosine_lr (closed form) against CosineAnnealingLR's recursive rates for render.py's two groups."""
    from instantsplat_b200.tracking import cosine_lr
    n = 500
    q, T = torch.zeros(4, dtype=torch.float64, requires_grad=True), torch.zeros(3, dtype=torch.float64,
                                                                                 requires_grad=True)
    opt = torch.optim.Adam([{"params": [q], "lr": 0.001}, {"params": [T], "lr": 0.003}], betas=(0.9, 0.999),
                           weight_decay=1e-4)
    sch = torch.optim.lr_scheduler.CosineAnnealingLR(opt, T_max=n, eta_min=1e-4)
    worst = 0.0
    for k in range(n):
        for grp, base in zip(opt.param_groups, (0.001, 0.003)):
            ours = cosine_lr(base, k, n, 1e-4)
            worst = max(worst, abs(ours - grp["lr"]) / grp["lr"])
        opt.step()
        sch.step()
    assert worst < 1e-13, worst
