"""fp64 restatement of the evaluation metrics kernel (gsb_image_metrics_batch in csrc/gs_loss.cu, DESIGN.md 4.11).

What the kernel computes for view v of imgs [V, C, H, W] against the target planes gts[gt_row[v]]:

  transform  both images through the mode's input map as the halo is staged; the zero padding stays zero:
             clamp  torch.clamp(x, 0, 1), which keeps NaN (training_report);
             png8   save_image's x.mul(255).add_(0.5).clamp_(0, 255).to(uint8) on the CPU, then to_tensor's / 255 in
                    fp32 (render.py -> metrics.py); NaN gives 0, +inf 255, -inf 0
  partials   one CTA per 32 x 16 output tile of each plane bc = v C + c writes its fp32 sums
             {sum |a - b|, sum ssim, sum (a - b)^2} as three doubles to scratch[3 cta], cta = (bc gy + by) gx + bx
             (gy x gx tiles per plane, T = gy gx)
  reduce     out[v] = {sum of the view's C T l1 partials, of its C T ssim partials, then for each channel c the sum of
             its T squared-error partials}, in fp64 (k_metrics_reduce)
  metrics    metrics_from_sums: l1 and ssim over C H W, per-channel mse over H W, psnr_channels = 20 log10(1 /
             sqrt(mse)), psnr the same of the whole image's mse

`terms` gives the per-pixel terms of the transformed planes in fp64 (the truth) and in fp32 (the restatement that
rounds like the kernel, tests/_loss.py); `tile_sums` adds them over the kernel's tiles.  Every partial and every sum
is bounded as the loss's sums are (`_loss.sum_bound`): K sum|t32 - t64| + 10 2^-24 sum|t64| over its terms, where
|t32 - t64| of the SSIM is raised to `product_floor` where it is smaller.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

import _loss as L

MODES = {"clamp": 1, "png8": 2}       # GSB_METRIC_CLAMP, GSB_METRIC_PNG8
REPORT_TAG = "metrics"
QUANTITIES = ("l1", "ssim", "sq")     # the order of a CTA's three partials
SENTINEL = -1.0e300                   # what the tests fill the scratch with, so an unwritten slot shows
SUB = 2.0 ** -149                     # the smallest fp32 subnormal


# ---- the transforms ------------------------------------------------------------------------------------------------
def png8(x):
    """save_image's 8-bit quantisation of fp32 x, on the CPU as torchvision does it, then to_tensor's / 255 (fp32).
    Returned on x's device."""
    q = x.detach().to("cpu", torch.float32).mul(255).add_(0.5).clamp_(0, 255).to(torch.uint8)
    return q.to(torch.float32).div(255).to(x.device)


def transform(x, mode):
    if mode == "clamp":
        return torch.clamp(x, 0, 1)
    if mode == "png8":
        return png8(x)
    raise ValueError(mode)


def tie_values(levels=(0, 1, 127, 254)):
    """fp32 x with x * 255 == k + 0.5 exactly in fp32 (save_image rounds them up to k + 1), and the fp32 numbers next
    to each."""
    up, down = np.float32(2), np.float32(-2)
    out = []
    for k in levels:
        x = np.float32((k + 0.5) / 255)
        for _ in range(8):
            x = np.nextafter(x, down)
        for _ in range(17):
            if np.float32(x * np.float32(255)) == np.float32(k + 0.5):
                out += [float(np.nextafter(x, down)), float(x), float(np.nextafter(x, up))]
            x = np.nextafter(x, up)
    return sorted(set(out))


ONE_UP, ONE_DOWN = float(np.nextafter(np.float32(1), np.float32(2))), float(np.nextafter(np.float32(1), np.float32(0)))
# render and target values where the transforms go wrong: NaN, the infinities, signed zeros, the smallest subnormals,
# 1 +- 1 ulp and save_image's tie values with their neighbours
SPECIALS = [math.nan, math.inf, -math.inf, 0.0, -0.0, SUB, -SUB, ONE_UP, ONE_DOWN] + tie_values()


# ---- per-pixel terms and the tiles ---------------------------------------------------------------------------------
def terms(a, b, dtype):
    """Transformed planes a, b [P, H, W] -> [3, P, H, W] per-pixel |a - b|, ssim, (a - b)^2, computed in dtype."""
    a, b = a.to(dtype), b.to(dtype)
    g = L.window(dtype).to(a.device)
    S, _ = L.ssim_maps(a, b, lambda x: L.conv(x, g))
    d = a - b
    return torch.stack([d.abs(), S, d * d])


def product_floor(a, b):
    """u |mu1 mu2| |dS/dE[ab]| per pixel, in fp64: what one rounding of the product mu1 mu2 moves the SSIM by.  The
    kernel's compiler may contract s12 = E[ab] - mu1 mu2 into an FMA and round the products of s1 and s2, or the other
    way round.  On identical planes (saturated flat content: both planes 1 after the transform) the fp32 restatement is
    exactly symmetric, s1 = s2 = s12, and its SSIM is right to the last bit, while the kernel's is off by that
    rounding over s ~ 1e-7 against C2 = 9e-4.  There the floor makes the bound loose by design; on random content it
    raises a view's SSIM bound by about a tenth."""
    a, b = a.double(), b.double()
    g = L.window(torch.float64).to(a.device)
    cv = lambda x: L.conv(x, g)
    _, maps = L.ssim_maps(a, b, cv)
    return 2.0 ** -24 * (cv(a) * cv(b)).abs() * maps[2].abs()


def grid(H, W):
    """(gy, gx): the kernel's tiles per plane."""
    return -(-H // L.TH), -(-W // L.TW)


def tile_sums(t):
    """Per-pixel values t [..., H, W] -> their sums over the kernel's 32 x 16 output tiles [..., gy, gx]."""
    H, W = t.shape[-2:]
    gy, gx = grid(H, W)
    p = F.pad(t, (0, gx * L.TW - W, 0, gy * L.TH - H))
    return p.reshape(*t.shape[:-2], gy, L.TH, gx, L.TW).sum((-3, -1))


def tile_regions(H, W):
    """Boolean [gy, gx] masks: `border` tiles hold a pixel within 10 px of the frame edge (where the zero padding
    enters their windows), `seam` tiles are the others (their halos cross the tile seams on all four sides)."""
    gy, gx = grid(H, W)
    by = torch.arange(gy)[:, None].expand(gy, gx)
    bx = torch.arange(gx)[None, :].expand(gy, gx)
    border = (by * L.TH < L.CTX) | (bx * L.TW < L.CTX) | ((by + 1) * L.TH > H - L.CTX) | ((bx + 1) * L.TW > W - L.CTX)
    return {k: m for k, m in dict(border=border, seam=~border).items() if bool(m.any())}


# ---- the restatement -----------------------------------------------------------------------------------------------
def restate(img, gt, rows, mode):
    """imgs [V, C, H, W] against gts[rows] (on any device; computed there) -> dict of fp64 tensors:
      a, b      the transformed planes [V, C, H, W] (fp32)
      part      the fp64 sum of each tile's terms [V C, gy, gx, 3] (the kernel's scratch, reshaped)
      e32, tot  per tile and quantity: sum|t32 - t64| and sum|t64|, for the bounds
      out, out_e32, out_tot  the same per view [V, 2 + C], laid out as the kernel's out."""
    V, C, H, W = img.shape
    rows = torch.as_tensor(rows, dtype=torch.long, device=gt.device)
    a, b = transform(img, mode), transform(gt[rows], mode)
    t64 = terms(a.reshape(V * C, H, W), b.reshape(V * C, H, W), torch.float64)
    t32 = terms(a.reshape(V * C, H, W), b.reshape(V * C, H, W), torch.float32)
    e = (t32.double() - t64).abs()
    del t32
    e[1] = torch.maximum(e[1], product_floor(a.reshape(V * C, H, W), b.reshape(V * C, H, W)))
    part, e32, tot = (tile_sums(x).permute(1, 2, 3, 0).contiguous() for x in (t64, e, t64.abs()))
    del t64, e
    return dict(a=a, b=b, part=part, e32=e32, tot=tot,
                out=view_sums(part, V, C), out_e32=view_sums(e32, V, C), out_tot=view_sums(tot, V, C))


def view_sums(part, V, C):
    """Tile values [V C, gy, gx, 3] -> the kernel's out layout [V, 2 + C]: l1 and ssim over the view's tiles, then the
    squared error of each channel's tiles."""
    p = part.reshape(V, C, -1, 3)
    return torch.cat([p[..., 0].sum((1, 2))[:, None], p[..., 1].sum((1, 2))[:, None], p[..., 2].sum(2)], 1)


# ---- the kernel ----------------------------------------------------------------------------------------------------
def metrics_kernel(img, gt, rows, mode, scratch=None):
    """gsb_image_metrics_batch on device tensors imgs [V, C, H, W], gts [N, C, H, W] (contiguous; their data_ptr may
    be anywhere) -> (every CTA's partials [V C, gy, gx, 3], out [V, 2 + C]), fp64 on the device.  The scratch is
    filled with SENTINEL first."""
    from instantsplat_b200 import _lib
    K = _lib.lib()
    V, C, H, W = img.shape
    gy, gx = grid(H, W)
    need = K.gsb_image_metrics_scratch_bytes(V, C, H, W)
    assert need == V * C * gy * gx * 3 * 8, need
    if scratch is None:
        scratch = torch.empty(V * C * gy * gx * 3, dtype=torch.float64, device=img.device)
    scratch.fill_(SENTINEL)
    out = torch.full((V, 2 + C), SENTINEL, dtype=torch.float64, device=img.device)
    row_dev = torch.tensor(list(rows), dtype=torch.int32, device=img.device)
    _lib.check(K.gsb_image_metrics_batch(V, C, H, W, img.data_ptr(), gt.data_ptr(), row_dev.data_ptr(), MODES[mode],
                                         out.data_ptr(), scratch.data_ptr(), need, _lib.stream_ptr()),
               "gsb_image_metrics_batch")
    return scratch.view(V * C, gy, gx, 3), out


# ---- checks --------------------------------------------------------------------------------------------------------
def bound_check(got, want, e32, tot, K=L.K):
    """Elementwise |got - want| <= K e32 + 10 2^-24 tot (`_loss.sum_bound`), with NaN exactly where `want` is NaN ->
    dict(n, err, ratio (worst err / bound), k_needed (the K the worst needs), nan_mismatch, ok)."""
    got, want, e32, tot = (x.double().reshape(-1) for x in (got, want, e32, tot))
    nan_w = torch.isnan(want)
    mismatch = int((nan_w != torch.isnan(got)).sum())
    fin = ~nan_w
    got, want, e32, tot = got[fin], want[fin], e32[fin], tot[fin]
    err = (got - want).abs()
    err = torch.where(torch.isnan(err), torch.full_like(err, math.inf), err)
    floor = 10 * 2.0 ** -24 * tot
    bound = K * e32 + floor
    ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300),
                        torch.where(err > 0, torch.full_like(err, math.inf), torch.zeros_like(err)))
    need = torch.where(e32 > 0, (err - floor).clamp_min(0) / e32.clamp_min(1e-300),
                       torch.where(err > floor, torch.full_like(err, math.inf), torch.zeros_like(err)))
    n = int(err.numel())
    return dict(n=n, err=float(err.max()) if n else 0.0, ratio=float(ratio.max()) if n else 0.0,
                k_needed=float(need.max()) if n else 0.0, nan_mismatch=mismatch,
                ok=bool(mismatch == 0 and (n == 0 or bool((err <= bound).all()))))


def check_partials(case, part, R, K=L.K):
    """Every CTA's three partials [V C, gy, gx, 3] against the restatement's tile sums, one record per tile region."""
    H, W = R["a"].shape[-2:]
    part = part.to(R["part"].device)
    recs = []
    for rn, mask in tile_regions(H, W).items():
        mask = mask.to(part.device)
        rec = dict(case=case, kind=REPORT_TAG, region=rn, tiles=int(mask.sum()) * part.shape[0])
        ok = True
        for i, q in enumerate(QUANTITIES):
            sel = lambda x: x[..., i][:, mask]
            c = bound_check(sel(part), sel(R["part"]), sel(R["e32"]), sel(R["tot"]), K)
            rec[q] = c
            ok &= c["ok"]
        rec["ok"] = ok
        recs.append(rec)
    return recs


def psnr_of(s, n):
    """20 log10(1 / sqrt(s / n)) in fp64, as metrics_from_sums and utils/image_utils.py psnr."""
    return 20.0 * torch.log10(1.0 / torch.sqrt(s / n))


def check_views(case, out, metrics, R, K=L.K):
    """out [V, 2 + C] against the restatement's view sums, and the PSNRs within the bound the squared-error bound
    gives them: |psnr - psnr64| <= 10 log10(m / (m - e)) for an mse m known to within e (inf where e >= m); inf
    exactly where the fp64 squared error is 0, NaN where it is NaN."""
    V, CC = out.shape
    C = CC - 2
    H, W = R["a"].shape[-2:]
    out = out.to(R["out"].device)
    want, e32, tot = R["out"], R["out_e32"], R["out_tot"]
    recs = []
    rec = dict(case=case, kind=REPORT_TAG, region="view")
    for i, q in ((0, "l1"), (1, "ssim")):
        rec[q] = bound_check(out[:, i], want[:, i], e32[:, i], tot[:, i], K)
    rec["sq"] = bound_check(out[:, 2:], want[:, 2:], e32[:, 2:], tot[:, 2:], K)
    ok = rec["l1"]["ok"] and rec["ssim"]["ok"] and rec["sq"]["ok"]
    # PSNR: per channel, and of the whole image
    sq_bound = K * e32[:, 2:] + 10 * 2.0 ** -24 * tot[:, 2:]
    for name, s64, eb, n, got in (("psnr_channels", want[:, 2:], sq_bound, H * W, metrics["psnr_channels"]),
                                  ("psnr", want[:, 2:].sum(1), sq_bound.sum(1), C * H * W, metrics["psnr"])):
        ref = psnr_of(s64, float(n))
        got = got.to(ref.device)
        m, e = s64 / n, eb / n
        pb = torch.where(m > e, 10.0 * torch.log10(m / (m - e).clamp_min(1e-300)), torch.full_like(m, math.inf))
        pb = pb + 1e-12 * (ref.abs().nan_to_num(posinf=0.0) + 1.0)
        inf_ok = torch.equal(torch.isposinf(ref), torch.isposinf(got))
        nan_ok = torch.equal(torch.isnan(ref), torch.isnan(got))
        fin = torch.isfinite(ref)
        err = (got[fin] - ref[fin]).abs()
        r = dict(err=float(err.max()) if err.numel() else 0.0, inf_match=inf_ok, nan_match=nan_ok,
                 ok=bool(inf_ok and nan_ok and bool((err <= pb[fin]).all())))
        rec[name] = r
        ok &= r["ok"]
    rec["ok"] = ok
    recs.append(rec)
    return recs


def worst(recs):
    """The largest k_needed over records (for the report and DESIGN.md)."""
    ks = [v["k_needed"] for r in recs for v in r.values() if isinstance(v, dict) and "k_needed" in v]
    return max(ks) if ks else 0.0


def bits(x):
    """x's bit pattern, so NaNs compare equal to themselves."""
    x = x.contiguous()
    return x.view(torch.int64) if x.dtype == torch.float64 else x.view(torch.int32)


def same_bits(x, y):
    return x.shape == y.shape and torch.equal(bits(x), bits(y))
