"""The references and bounds of tests/_loss.py, checked without a device.

* The separable fp64 reference equals the reference's own formula (`O.ssim_map`, `O.training_loss` under autograd,
  2-D convolutions) to 1e-12, maps included; the crop reference equals the full-frame one on the inner box.
* The bounds can discriminate: each mutant below, computed in fp32, is a plausible kernel bug, and must exceed the
  bound by at least 10x in the region it affects.  This is the ceiling on `_loss.K`.
"""
import pytest
import torch
import torch.nn.functional as F

import _loss as L
from oracle import gs_oracle as O

SHAPE = (3, 53, 77)


def _tol(r64, r32, key):
    """1e-12 of the largest value, or on ill-conditioned content 1e-6 of the fp32 restatement's error: two fp64
    evaluations differ by fp64's share of the same cancellation, about 2^-29 of fp32's (flat content: 3e-11)."""
    return max(1e-12 * float(r64[key].abs().max()), 1e-6 * float((r32[key].double() - r64[key]).abs().max()))


@pytest.mark.parametrize("kind", ["uniform", "raw", "flat", "impulses", "checker"])
def test_separable_reference_matches_oracle_2d(kind):
    a, b = L.content(kind, *SHAPE, seed=1)
    a, b = a.double(), b.double()
    smap = O.ssim_map(a, b)
    for lam in (0.0, 0.2, 1.0):
        x = a.clone().requires_grad_(True)
        O.training_loss(x, b, lam).backward()
        r64, r32 = L.both(a, b, lam=lam)
        assert float((r64["ssim"] - smap).abs().max()) <= _tol(r64, r32, "ssim")
        assert float((r64["grad"] - x.grad).abs().max()) <= _tol(r64, r32, "grad"), lam
    for up in (1.0, -0.2, 3.7):
        x = a.clone().requires_grad_(True)
        (O.ssim(x[None], b[None]) * up).backward()
        r64, r32 = L.both(a, b, up=up)
        assert float((r64["grad"] - x.grad).abs().max()) <= _tol(r64, r32, "grad"), up


def test_derivative_maps_are_the_partials_of_ssim():
    """maps = dS/dmu1, dS/dE[a^2], dS/dE[ab] of the ssim formula at fixed b, by autograd on the window statistics."""
    a, b = L.content("raw", *SHAPE, seed=2)
    a, b = a.double(), b.double()
    g = L.window(torch.float64)
    mu1, e11, e12 = (L.conv(t, g).requires_grad_(True) for t in (a, a * a, a * b))
    mu2, e22 = L.conv(b, g), L.conv(b * b, g)
    s1, s2, s12 = e11 - mu1 ** 2, e22 - mu2 ** 2, e12 - mu1 * mu2
    S = ((2 * mu1 * mu2 + L.C1) * (2 * s12 + L.C2)) / ((mu1 ** 2 + mu2 ** 2 + L.C1) * (s1 + s2 + L.C2))
    S.sum().backward()
    maps = L.reference(a, b)["maps"]
    for i, t in enumerate((mu1, e11, e12)):
        assert float((maps[i] - t.grad).abs().max()) <= 1e-12 * float(t.grad.abs().max()), i


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_crop_reference_equals_full_frame(dtype):
    FH, FW = 70, 100
    a, b = L.content("raw", 3, FH, FW, seed=3)
    full = L.reference(a, b, lam=0.2, dtype=dtype)
    for (y0, y1, x0, x1) in ((0, 20, 0, 30), (50, 70, 70, 100), (25, 41, 30, 62), (0, 70, 45, 46), (33, 34, 0, 100)):
        (iy, ix), (oy, ox) = L.crop_box(FH, FW, y0, y1, x0, x1)
        crop = L.reference(a[:, iy, ix], b[:, iy, ix], lam=0.2, N=a.numel(), dtype=dtype)
        for k in ("ssim", "grad", "l1"):
            assert torch.equal(crop[k][:, oy, ox], full[k][:, y0:y1, x0:x1]), (k, y0, x0)
        assert torch.equal(crop["maps"][:, :, oy, ox], full["maps"][:, :, y0:y1, x0:x1])


def test_regions_partition_the_frame():
    for H, W in ((1, 1), (21, 21), (53, 77), (240, 416)):
        R = L.regions(H, W)
        tot = sum(m.int() for m in R.values())
        assert torch.equal(tot, torch.ones(H, W, dtype=tot.dtype)), (H, W)
    R = L.regions(53, 77)
    assert bool(R["seam"][24, 27]) and bool(R["seam"][24, 36]) and not bool(R["seam"][24, 37])
    assert bool(R["seam"][15, 20]) and bool(R["seam"][20, 20]) and not bool(R["seam"][21, 20])
    assert bool(R["border"][9, 40]) and not bool(R["border"][10, 40]) and bool(R["interior"][24, 20])
    # a crop classifies its pixels by their frame coordinates
    C = L.regions(20, 40, y0=1060, x0=1880, FH=1080, FW=1920)
    assert bool(C["border"][-1, -1]) and bool(C["seam"][0, 0]) and bool(C["interior"][6, 1])   # y 1066, x 1881


# ---- mutants -------------------------------------------------------------------------------------------------------
def _shift_x(t, dx):
    """t(p + dx) along x, zero outside."""
    return F.pad(t, (0, dx))[..., dx:] if dx > 0 else F.pad(t, (-dx, 0))[..., :dx]


def _shift_y(t, dy):
    return _shift_x(t.transpose(-1, -2), dy).transpose(-1, -2)


def mutant_grad(a, b, lam, kind, N=None):
    """dL/da of the training loss in fp32 with one bug."""
    a, b = a.float(), b.float()
    N = a.numel() if N is None else N
    g = L.window(torch.float32)
    cv_fwd = cv_bwd = lambda x: L.conv(x, g)
    if kind == "replicate_padding":              # halo loads clamp to the frame instead of reading zeros
        def rep(x):
            p = F.pad(x, (L.HALO,) * 4, mode="replicate")
            return L.conv(p, g)[..., L.HALO:-L.HALO, L.HALO:-L.HALO]
        cv_fwd = cv_bwd = rep
    elif kind == "window_shift":                 # the forward's taps one off: c_win[t + 1]
        gs = torch.cat([g[1:], g.new_zeros(1)])
        cv_fwd = lambda x: L.conv(x, gs)
    elif kind == "adjoint_offset":               # the backward reads its maps' halo one pixel off
        cv_bwd = lambda x: _shift_y(L.conv(x, g), 1)
    S, maps = L.ssim_maps(a, b, cv_fwd)
    s_ssim, s_l1 = L.scales(lam, 1.0, N, torch.float32)
    if kind == "drop_s1":                        # 2 x conv(m_s1) left out
        adj = cv_bwd(maps[0]) + b * cv_bwd(maps[2])
    else:
        adj = L.adjoint(maps, a, b, cv_bwd)
    sign = torch.sign(a - b)
    if kind == "sign0_plus":                     # sign(0) = +1 in the L1 term
        sign = torch.where(a == b, torch.ones_like(sign), sign)
    return s_ssim * adj + s_l1 * sign


def _mutant_ratio(got, r64, r32, mask):
    c = L.region_check(got, r64["grad"], r32["grad"], mask)
    return c["err"] / c["bound"]


MUTANTS = [("replicate_padding", "border"), ("window_shift", "interior"), ("window_shift", "border"),
           ("adjoint_offset", "interior"), ("adjoint_offset", "seam"), ("drop_s1", "interior")]


@pytest.mark.parametrize("kind", ["uniform", "raw", "flat"])
def test_mutants_exceed_the_bound_tenfold(kind):
    """On flat content the bound is loose by design (e32 is 1e-3 of the gradient there), and a one-pixel shift of the
    backward's nearly uniform maps stays under 10x of it; that mutant is caught on the other contents."""
    a, b = L.content(kind, *SHAPE, seed=4)
    r64, r32 = L.both(a, b, lam=0.2)
    R = L.regions(*SHAPE[1:])
    ratios = {}
    for mut, region in MUTANTS:
        if kind == "flat" and mut == "adjoint_offset":
            continue
        ratios[(mut, region)] = _mutant_ratio(mutant_grad(a, b, 0.2, mut), r64, r32, R[region])
    assert min(ratios.values()) >= 10, ratios
    # the correct formula in fp32 is within the bound everywhere (K >= 1 by construction)
    for region, mask in R.items():
        assert L.region_check(r32["grad"], r64["grad"], r32["grad"], mask)["ok"]


def test_mutant_sign_of_zero():
    """sign(0) = +1 shows at the tie pixels of the ties content, and only there."""
    a, b = L.content("ties", *SHAPE, seed=5)
    r64, r32 = L.both(a, b, lam=0.2)
    tie = (a == b).all(0)
    assert 0.3 < float(tie.float().mean()) < 0.7
    got = mutant_grad(a, b, 0.2, "sign0_plus")
    assert _mutant_ratio(got, r64, r32, tie) >= 10
    assert L.region_check(got, r64["grad"], r32["grad"], ~tie)["ok"]


def test_mutant_gt_row_off_by_one_plane():
    """A batched loss that reads the target plane after gt_row[v] * C + c."""
    V, C, H, W = 3, 3, 37, 70
    g = torch.Generator().manual_seed(6)
    img, gt = torch.rand(V, C, H, W, generator=g), torch.rand(4, C, H, W, generator=g)
    gt_row = torch.tensor([2, 0, 2])
    planes = gt.reshape(-1, H, W)
    z = (gt_row[:, None] * C + torch.arange(C)).reshape(-1)
    b, b_bad = planes[z].reshape(V, C, H, W), planes[z + 1].reshape(V, C, H, W)
    r64, r32 = L.both(img, b, lam=0.2, N=C * H * W)
    got = L.reference(img, b_bad, lam=0.2, N=C * H * W, dtype=torch.float32)
    for region, mask in L.regions(H, W).items():
        assert _mutant_ratio(got["grad"], r64, r32, mask) >= 10, region
