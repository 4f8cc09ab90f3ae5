"""fp64 references, pixel regions and calibrated bounds for the SSIM / L1 loss kernels (csrc/gs_loss.cu).

What the kernels compute on every plane (11x11 window w = g g^T, g = `O.gaussian_window` rounded to fp32, zero 'same'
padding, C1 = 1e-4, C2 = 9e-4):

  forward   mu1 = w*a, mu2 = w*b, e11 = w*(a a), e22 = w*(b b), e12 = w*(a b) -> the ssim map S and the three
            derivative maps m_mu = dS/dmu1, m_s1 = dS/de11, m_s12 = dS/de12 (b held fixed)
  backward  dL/da = s_ssim (w*m_mu + 2 a (w*m_s1) + b (w*m_s12)) + s_l1 sign(a - b), the adjoint of the forward's
            convolutions (w is symmetric), with s_ssim = -lambda / N, s_l1 = (1 - lambda) / N for the training loss
            and s_ssim = upstream / N, s_l1 = 0 for fused_ssim

`reference` evaluates that chain in any dtype: float64 is the truth, float32 is the "fp32 restatement" whose distance
from the truth calibrates the bounds.  The convolutions are separable and sum their taps in the kernel's order, so
the fp32 restatement rounds like the kernel up to FMA contraction; in float64 they agree with `O.ssim_map` /
`O.training_loss` under autograd to 1e-12 (tests/test_loss_edges_cpu.py).  The kernels normalise their window with a
sequential fp32 sum, so some taps differ from `O.gaussian_window`'s by one ulp; the bounds absorb that.

Bounds.  SSIM in fp32 is badly conditioned on bright flat content (sigma^2 = E[x^2] - mu^2 cancels), so one fixed
tolerance cannot serve both random and flat images.  Each check is calibrated on its own inputs, region by region:
e32 = max |fp32 restatement - fp64| over the region, and the kernel must satisfy

    max |kernel - fp64| <= K e32 + 4 ulp(max |fp64|)          (ulp of an fp32 value)

K = 17 is 3.5x the largest kernel / e32 ratio measured on an H100 (see `K`).  Regions: every check reports its worst pixel
per region, so an interior maximum cannot hide an error at the frame border (`border`: within 10 px of the frame edge,
where the zero padding enters) or at a tile seam of the kernels' 32 x 16 output tiles (`seam`: within 5 px of a
32-column or 16-row boundary, where the staged halo ends).  Sums are bounded by K sum|t32 - t64| + 10 2^-24 sum|t64|
over their terms t: the fp32 CTA sums add 9 levels of rounding on top of each term's own.

Large frames are checked on crops: a gradient pixel depends on the inputs within 10 px (5 for the maps, 5 more for the
adjoint), so `crop_box` adds 10 px of context, clipped at the frame, and the crop's reference equals the full frame's
on the inner box.
"""
import math

import torch
import torch.nn.functional as F

from oracle import gs_oracle as O

# K: 3.5x the largest kernel / e32 ratio over every case and region of tests/test_loss_edges.py (the `k_needed` of
# its records in the parity report), measured on an NVIDIA H100 80GB HBM3 at its 700 W power limit: 4.77, the
# derivative map dS/dmu1 of a == b at 3 x 240 x 416 (the map is 0 there and both arms give rounding noise; the kernel
# contracts into FMAs what the fp32 restatement rounds twice).  The largest on other content: 4.38 (fused_ssim's
# gradient at 2 x 1 x 21 x 33).  tests/test_loss_edges_cpu.py keeps every mutant 10x or more over this bound.
K = 17.0
C1, C2 = 0.01 ** 2, 0.03 ** 2
HALO = 5
CTX = 2 * HALO
TW, TH = 32, 16
REPORT_TAG = "loss"


def conv(x, g):
    """Zero-padded 'same' 11x11 window g g^T on planes x [..., H, W]: rows first, then columns, each summing its taps
    in order t = 0..10 (the kernels' order)."""
    H, W = x.shape[-2:]
    p = F.pad(x, (HALO, HALO))
    h = g[0] * p[..., 0:W]
    for t in range(1, 11):
        h = h + g[t] * p[..., t:t + W]
    p = F.pad(h, (0, 0, HALO, HALO))
    v = g[0] * p[..., 0:H, :]
    for t in range(1, 11):
        v = v + g[t] * p[..., t:t + H, :]
    return v


def window(dtype):
    return O.gaussian_window(11, 1.5, dtype)


def ssim_maps(a, b, cv):
    """-> (S, maps [3, ...]) of planes a, b as k_ssim_fwd writes them: maps = dS/dmu1, dS/dE[a^2], dS/dE[ab].
    cv: the window, x -> conv(x, g)."""
    mu1, mu2 = cv(a), cv(b)
    e11, e22, e12 = cv(a * a), cv(b * b), cv(a * b)
    mu1_sq, mu2_sq, mu12 = mu1 * mu1, mu2 * mu2, mu1 * mu2
    s1, s2, s12 = e11 - mu1_sq, e22 - mu2_sq, e12 - mu12
    A1, A2 = 2 * mu12 + C1, 2 * s12 + C2
    B1, B2 = mu1_sq + mu2_sq + C1, s1 + s2 + C2
    inv = 1 / (B1 * B2)
    S = A1 * A2 * inv
    m_mu = 2 * mu2 * (A2 - A1) * inv - S * 2 * mu1 * (B2 - B1) * inv
    return S, torch.stack([m_mu, -S / B2, 2 * A1 * inv])


def adjoint(maps, a, b, cv):
    """w*m_mu + 2 a (w*m_s1) + b (w*m_s12) (k_ssim_bwd before scaling): d(sum S)/da, given the maps of S."""
    return cv(maps[0]) + 2 * a * cv(maps[1]) + b * cv(maps[2])


def scales(lam, up, N, dtype):
    """(s_ssim, s_l1) as the kernels round them: the loss's from -lam / N and (1 - lam) / N in double, fused_ssim's
    as fp32 1/N times the upstream scalar."""
    if lam is not None:
        return torch.tensor(-lam / N, dtype=dtype), torch.tensor((1.0 - lam) / N, dtype=dtype)
    return torch.tensor(1.0 / N, dtype=dtype) * torch.tensor(up, dtype=dtype), torch.tensor(0.0, dtype=dtype)


def reference(a, b, lam=None, up=1.0, N=None, dtype=torch.float64):
    """Planes a, b [..., H, W] (any float dtype; computed in `dtype`) -> dict(ssim, maps, grad, l1) per pixel:
    the training loss's dL/da for lam given (gsb_loss_backward), else fused_ssim's under the upstream scalar `up`.
    N: the normalisation (default a.numel(); a crop or a batch of views passes its frame's)."""
    a, b = a.to(dtype), b.to(dtype)
    N = a.numel() if N is None else N
    g = window(dtype)
    cv = lambda x: conv(x, g)
    S, maps = ssim_maps(a, b, cv)
    s_ssim, s_l1 = scales(lam, up, N, dtype)
    grad = s_ssim * adjoint(maps, a, b, cv)
    d = a - b
    if float(s_l1) != 0.0:
        grad = grad + s_l1 * torch.sign(d)
    return dict(ssim=S, maps=maps, grad=grad, l1=d.abs())


def both(a, b, **kw):
    """(fp64 reference, fp32 restatement)."""
    return reference(a, b, dtype=torch.float64, **kw), reference(a, b, dtype=torch.float32, **kw)


# ---- regions -------------------------------------------------------------------------------------------------------
def regions(H, W, y0=0, x0=0, FH=None, FW=None):
    """Boolean [H, W] masks of an H x W box at (y0, x0) of an FH x FW frame (default: the box is the frame):
    border (within CTX px of the frame edge), seam (within HALO px of a tile boundary, not border), interior.
    Empty regions are left out."""
    FH, FW = (H if FH is None else FH), (W if FW is None else FW)
    y = torch.arange(y0, y0 + H)[:, None].expand(H, W)
    x = torch.arange(x0, x0 + W)[None, :].expand(H, W)
    border = (x < CTX) | (x >= FW - CTX) | (y < CTX) | (y >= FH - CTX)
    seam = ((x % TW < HALO) | (x % TW >= TW - HALO) | (y % TH < HALO) | (y % TH >= TH - HALO)) & ~border
    out = dict(border=border, seam=seam, interior=~border & ~seam)
    return {k: v for k, v in out.items() if bool(v.any())}


def crop_box(FH, FW, y0, y1, x0, x1):
    """Output box [y0, y1) x [x0, x1) of an FH x FW frame -> (input slices with CTX px of context clipped at the frame,
    slices of the output box inside that crop)."""
    cy0, cy1, cx0, cx1 = max(0, y0 - CTX), min(FH, y1 + CTX), max(0, x0 - CTX), min(FW, x1 + CTX)
    return (slice(cy0, cy1), slice(cx0, cx1)), (slice(y0 - cy0, y1 - cy0), slice(x0 - cx0, x1 - cx0))


# ---- bounds --------------------------------------------------------------------------------------------------------
def ulp32(x):
    """Spacing of fp32 numbers at |x| (0 for 0)."""
    x = abs(float(x))
    if x == 0.0 or not math.isfinite(x):
        return 0.0
    return 2.0 ** (math.frexp(x)[1] - 24)


def region_check(got, ref64, ref32, mask, K=K):
    """Worst pixel of one region (mask [H, W] over planes [..., H, W]) -> dict(err, e32, bound, ratio, k_needed, ok).
    ratio = err / e32; k_needed = the K this region alone needs (err above the ulp floor, over e32)."""
    m = mask.expand_as(ref64)
    r = ref64.double()[m]
    err = float((got.double()[m] - r).abs().max())
    e32 = float((ref32.double()[m] - r).abs().max())
    floor = 4 * ulp32(r.abs().max())
    bound = K * e32 + floor
    ratio = err / e32 if e32 > 0 else (0.0 if err == 0 else math.inf)
    k_needed = max(0.0, err - floor) / e32 if e32 > 0 else (0.0 if err <= floor else math.inf)
    return dict(err=err, e32=e32, bound=bound, ratio=ratio, k_needed=k_needed, ok=bool(err <= bound))


def check_maps(case, got, ref, regs, quantities=("grad", "m_mu", "m_s1", "m_s12"), K=K):
    """got: dict of kernel outputs among `quantities` (planes [..., H, W]); ref: (fp64, fp32) from `both` (or crops of
    them).  -> one record per region with every quantity's numbers and `ok`."""
    r64, r32 = ref
    recs = []
    for rn, mask in regs.items():
        rec = dict(case=case, kind=REPORT_TAG, region=rn, pixels=int(mask.sum()))
        ok = True
        for q in quantities:
            if q not in got:
                continue
            if q == "grad":
                g64, g32 = r64["grad"], r32["grad"]
            else:
                i = ("m_mu", "m_s1", "m_s12").index(q)
                g64, g32 = r64["maps"][i], r32["maps"][i]
            c = region_check(got[q], g64, g32, mask, K)
            rec[q] = c
            ok &= c["ok"]
        rec["ok"] = ok
        recs.append(rec)
    return recs


def sum_bound(t64, t32, K=K):
    """Bound on |kernel sum - sum t64| for the kernels' fp32 CTA sums of per-pixel terms t."""
    return K * float((t32.double() - t64).abs().sum()) + 10 * 2.0 ** -24 * float(t64.abs().sum())


def check_sum(case, name, got, t64, t32, K=K):
    want = float(t64.sum())
    err, bound = abs(float(got) - want), sum_bound(t64, t32, K)
    return dict(case=case, kind=REPORT_TAG, region="sum", quantity=name, got=float(got), want=want, err=err,
                bound=bound, ok=bool(err <= bound))


def worst(recs):
    """The largest k_needed over records (for the report and the calibration of K)."""
    ks = [v["k_needed"] for r in recs for v in r.values() if isinstance(v, dict) and "k_needed" in v]
    return max(ks) if ks else 0.0


# ---- content -------------------------------------------------------------------------------------------------------
def content(kind, C, H, W, seed=0):
    """(a, b) fp32 [C, H, W] of one regime: uniform, raw (a render in [-0.2, 3] against [0, 1]), flat (2.7 +- 1e-3
    against 2.69), equal (a == b), ties (a == b at a random half of the
    pixels, all channels), impulses (ones at the frame corners and
    across tile seams, on black, against black), checker (a 0/1 checkerboard against uniform)."""
    g = torch.Generator().manual_seed(seed)
    u = lambda: torch.rand(C, H, W, generator=g)
    if kind == "uniform":
        return u(), u()
    if kind == "raw":
        return u() * 3.2 - 0.2, u()
    if kind == "flat":
        return torch.full((C, H, W), 2.7) + 1e-3 * u(), torch.full((C, H, W), 2.69)
    if kind == "equal":
        a = u()
        return a, a.clone()
    if kind == "ties":
        a, b = u(), u()
        return a, torch.where(torch.rand(1, H, W, generator=g) < 0.5, a, b)
    if kind == "impulses":
        a = torch.zeros(C, H, W)
        for y, x in impulse_points(H, W):
            a[:, y, x] = 1.0
        return a, torch.zeros(C, H, W)
    if kind == "checker":
        y, x = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
        return ((y + x) % 2).float().expand(C, H, W).contiguous(), u()
    raise ValueError(kind)


def impulse_points(H, W):
    """The four corners and the pixels on either side of the tile seams (y 15 | 16, x 31 | 32) that fit."""
    pts = {(0, 0), (0, W - 1), (H - 1, 0), (H - 1, W - 1)}
    for y, x in ((TH - 1, TW - 1), (TH, TW), (TH - 1, TW), (TH, 2 * TW - 1), (2 * TH, TW)):
        if y < H and x < W:
            pts.add((y, x))
    return sorted(pts)


CONTENTS = ("uniform", "raw", "flat", "equal", "ties", "impulses", "checker")
