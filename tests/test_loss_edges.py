"""The SSIM / L1 loss kernels (gs_loss.cu) and the masked L1 of tracking (gs_track.cu), pixel by pixel against fp64
at frame borders, tile seams, small frames, ill-conditioned content and large frames (-m gpu).

Every map and gradient is checked per region (tests/_loss.py: border, seam, interior) against the fp64 reference with
the bound K e32 + 4 ulp, calibrated on each case's own fp32 restatement; sums against K sum|t32 - t64| plus the CTA
sums' rounding.  Each case's numbers go to the parity report (kind "loss"), and a test asserts after recording all of
its cases.  Some cases are exact: the L1 part of a == b is 0, the gradient of lambda = 0 is sign(a - b) (float)(1/N),
a zero upstream gradient gives zeros, and pixels farther than 10 px from every impulse get exactly 0.
"""
import math

import pytest
import torch
import torch.nn.functional as F

import _loss as L
from _parity import DEV, REPORT
from instantsplat_b200 import GsbError

pytestmark = pytest.mark.gpu

HS = (1, 2, 5, 6, 10, 11, 15, 16, 17, 21, 31, 32, 33)
WS = (1, 3, 5, 11, 31, 32, 33, 37, 42, 43, 64, 65)


def _L():
    from instantsplat_b200 import _lib
    return _lib, _lib.lib()


def loss_kernel(a, b, lam):
    """gsb_loss_forward + gsb_loss_backward on [C, H, W] -> (sums [2], maps [3, C, H, W], dL/da) on the CPU."""
    lib, K = _L()
    a, b = a.to(DEV).contiguous(), b.to(DEV).contiguous()
    C, H, W = a.shape
    sums = torch.zeros(2, dtype=torch.float64, device=DEV)
    maps = torch.empty(3, C, H, W, device=DEV)
    out = torch.empty_like(a)
    lib.check(K.gsb_loss_forward(C, H, W, a.data_ptr(), b.data_ptr(), sums.data_ptr(), maps.data_ptr(),
                                 lib.stream_ptr()), "gsb_loss_forward")
    lib.check(K.gsb_loss_backward(C, H, W, a.data_ptr(), b.data_ptr(), maps.data_ptr(), lam, out.data_ptr(),
                                  lib.stream_ptr()), "gsb_loss_backward")
    return sums.cpu(), maps.cpu(), out.cpu()


def loss_kernel_batch(img, gt, gt_row, lam):
    """gsb_loss_forward_batch + gsb_loss_backward_batch -> (sums [V, 2], maps [3, V C, H, W], dL/dimg) on the CPU."""
    lib, K = _L()
    V, C, H, W = img.shape
    img, gt, rows = img.to(DEV).contiguous(), gt.to(DEV).contiguous(), gt_row.to(DEV, torch.int32).contiguous()
    sums = torch.zeros(V, 2, dtype=torch.float64, device=DEV)
    maps = torch.empty(3, V * C, H, W, device=DEV)
    out = torch.empty_like(img)
    lib.check(K.gsb_loss_forward_batch(V, C, H, W, img.data_ptr(), gt.data_ptr(), rows.data_ptr(), sums.data_ptr(),
                                       maps.data_ptr(), lib.stream_ptr()), "gsb_loss_forward_batch")
    lib.check(K.gsb_loss_backward_batch(V, C, H, W, img.data_ptr(), gt.data_ptr(), rows.data_ptr(), maps.data_ptr(),
                                        lam, out.data_ptr(), lib.stream_ptr()), "gsb_loss_backward_batch")
    return sums.cpu(), maps.cpu(), out.cpu()


def ssim_kernel(a, b, up):
    """fused_ssim on [B, C, H, W] with the upstream gradient `up` (a device scalar) -> (value, dL/da)."""
    import instantsplat_b200 as I
    x = a.to(DEV).requires_grad_(True)
    s = I.fused_ssim(x, b.to(DEV))
    s.backward(torch.tensor(up, device=DEV))
    return float(s.detach()), x.grad.cpu()


def check_loss(case, a, b, lam, ref=None):
    """Kernel vs fp64 for the training loss on [C, H, W] -> (records, kernel outputs)."""
    sums, maps, grad = loss_kernel(a, b, lam)
    r64, r32 = ref if ref is not None else L.both(a, b, lam=lam)
    recs = L.check_maps(case, dict(grad=grad, m_mu=maps[0], m_s1=maps[1], m_s12=maps[2]), (r64, r32),
                        L.regions(*a.shape[-2:]))
    recs.append(L.check_sum(case, "ssim", sums[1], r64["ssim"], r32["ssim"]))
    recs.append(L.check_sum(case, "l1", sums[0], r64["l1"], r32["l1"]))
    return recs, (sums, maps, grad)


def check_ssim(case, a, b, up):
    """Kernel vs fp64 for fused_ssim on [B, C, H, W] -> (records, gradient)."""
    val, grad = ssim_kernel(a, b, up)
    r64, r32 = L.both(a, b, up=up)
    recs = L.check_maps(case, dict(grad=grad), (r64, r32), L.regions(*a.shape[-2:]))
    # the value comes back as fp32 sum / n: one more rounding of the sum
    recs.append(L.check_sum(case, "ssim", val * a.numel(), r64["ssim"], r32["ssim"]))
    return recs, grad


def record(recs):
    """Add the records to the parity report; -> the failing ones."""
    REPORT.extend(recs)
    return [r for r in recs if not r["ok"]]


def assert_ok(recs, exact=()):
    """Record every check, then fail on any over its bound and on any exact check (name, passed) that did not hold."""
    bad = record(recs)
    assert not bad, f"{len(bad)} of {len(recs)} checks over the bound (K = {L.K}, worst k_needed " \
                    f"{L.worst(recs):.3g}): {bad[:6]}"
    wrong = [name for name, ok in exact if not ok]
    assert not wrong, f"exact checks that failed: {wrong}"


# ---- 1. sizes ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("family", ["loss", "fused_ssim"])
def test_size_sweep(family):
    """Frames smaller than the window, than one tile, and one pixel either side of a tile edge, through both entry
    families: every map and gradient per region, and the sums."""
    recs = []
    for H in HS:
        for W in WS:
            if family == "loss":
                a, b = L.content("uniform", 3, H, W, seed=100 * H + W)
                recs += check_loss(f"sizes loss 3x{H}x{W}", a, b, 0.2)[0]
            else:
                a, b = L.content("raw", 2, H, W, seed=100 * H + W)
                recs += check_ssim(f"sizes fused_ssim 2x1x{H}x{W}", a[:, None], b[:, None], 1.0)[0]
    assert_ok(recs)


# ---- 2, 3. content, lambda and the upstream scalar -----------------------------------------------------------------
def far_from_impulses(a):
    """Pixels farther than 10 px (in x or y) from every non-zero pixel of a [C, H, W]."""
    hot = (a != 0).any(0).float()[None, None]
    return ~(F.max_pool2d(hot, 2 * L.CTX + 1, stride=1, padding=L.CTX)[0, 0] > 0)


@pytest.mark.parametrize("shape", [(3, 53, 77), (3, 240, 416)])
@pytest.mark.parametrize("kind", L.CONTENTS)
def test_content_regimes(kind, shape):
    a, b = L.content(kind, *shape, seed=7)
    N = a.numel()
    recs, exact = [], []
    far = far_from_impulses(a)
    if kind == "impulses":
        assert bool(far.any())
    for lam in (0.0, 0.2, 1.0):
        rs, (sums, _, grad) = check_loss(f"{kind} loss {'x'.join(map(str, shape))} lambda {lam}", a, b, lam)
        recs += rs
        if lam == 0.0:      # the SSIM part is scaled by -0: the gradient is the L1 term's, bit for bit
            exact.append(("lambda 0: sign(a - b) / N",
                          torch.equal(grad, torch.sign(a - b) * torch.tensor(1.0 / N, dtype=torch.float32))))
        if kind == "equal":
            exact.append((f"lambda {lam}: l1 sum of a == b is 0", float(sums[0]) == 0.0))
        if kind == "impulses":
            exact.append((f"lambda {lam}: 0 far from the impulses", bool((grad[:, far] == 0).all())))
    for up in (1.0, -0.2, 3.7, 0.0):
        rs, grad = check_ssim(f"{kind} fused_ssim {'x'.join(map(str, shape))} upstream {up}", a[None], b[None], up)
        recs += rs
        if up == 0.0:
            exact.append(("upstream 0: zeros", bool((grad == 0).all())))
        if kind == "impulses":
            exact.append((f"upstream {up}: 0 far from the impulses", bool((grad[0][:, far] == 0).all())))
    assert_ok(recs, exact)


# ---- 4. batched entries --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("V", [1, 3, 7])
def test_batched_loss_equals_single_views(V, C):
    """View v of gsb_loss_*_batch is bit-identical to gsb_loss_forward / backward against gt[gt_row[v]], with
    gt_row permuted and repeated, and within the bounds of fp64."""
    H, W, G = 37, 70, 4
    g = torch.Generator().manual_seed(10 * V + C)
    img = torch.rand(V, C, H, W, generator=g) * 3.2 - 0.2
    gt = torch.rand(G, C, H, W, generator=g)
    gt_row = torch.tensor([3, 1, 1, 0, 2, 3, 0][:V] if V > 1 else [2])
    sums, maps, grad = loss_kernel_batch(img, gt, gt_row, 0.2)
    recs = []
    for v in range(V):
        s1, m1, g1 = loss_kernel(img[v], gt[gt_row[v]], 0.2)
        assert torch.equal(g1, grad[v]), v
        assert torch.equal(m1, maps[:, v * C:(v + 1) * C]), v
        # the double sums of fp32 CTA partials are exact here, so the atomics' order cannot show
        assert torch.equal(s1, sums[v]), v
        r64, r32 = L.both(img[v], gt[gt_row[v]], lam=0.2)
        recs += L.check_maps(f"batch V{V} C{C} view {v}", dict(grad=grad[v]), (r64, r32), L.regions(H, W))
        recs.append(L.check_sum(f"batch V{V} C{C} view {v}", "ssim", sums[v, 1], r64["ssim"], r32["ssim"]))
    assert_ok(recs)


@pytest.mark.parametrize("V,C", [(65535, 1), (21845, 3)])
def test_batched_loss_at_the_grid_z_limit(V, C):
    """V C = 65535 planes (the grid's z limit) on 4 x 4 frames: accepted, and every view within its bounds."""
    H = W = 4
    G = 7
    g = torch.Generator().manual_seed(V)
    img = torch.rand(V, C, H, W, generator=g)
    gt = torch.rand(G, C, H, W, generator=g)
    gt_row = torch.randint(0, G, (V,), generator=g)
    sums, maps, grad = loss_kernel_batch(img, gt, gt_row, 0.2)
    b = gt[gt_row]
    r64, r32 = L.both(img, b, lam=0.2, N=C * H * W)
    recs = L.check_maps(f"batch limit V{V} C{C}", dict(grad=grad, m_mu=maps[0].view(V, C, H, W)), (r64, r32),
                        L.regions(H, W))
    # per-view sums
    for q, i in (("ssim", 1), ("l1", 0)):
        t64, t32 = r64[q].flatten(1), r32[q].flatten(1)
        bound = L.K * (t32.double() - t64).abs().sum(1) + 10 * 2.0 ** -24 * t64.abs().sum(1)
        err = (sums[:, i] - t64.sum(1)).abs()
        recs.append(dict(case=f"batch limit V{V} C{C}", kind=L.REPORT_TAG, region="sum", quantity=f"{q} per view",
                         worst_err_over_bound=float((err / bound).max()), ok=bool((err <= bound).all())))
    assert_ok(recs)


@pytest.mark.parametrize("V,C", [(65536, 1), (32768, 2), (21846, 3)])
def test_batched_loss_refuses_more_than_65535_planes(V, C):
    lib, K = _L()
    x = torch.zeros(16, device=DEV)
    rows = torch.zeros(1, dtype=torch.int32, device=DEV)
    sums = torch.zeros(2, dtype=torch.float64, device=DEV)
    with pytest.raises(GsbError):
        lib.check(K.gsb_loss_forward_batch(V, C, 1, 1, x.data_ptr(), x.data_ptr(), rows.data_ptr(), sums.data_ptr(),
                                           x.data_ptr(), lib.stream_ptr()), "gsb_loss_forward_batch")
    with pytest.raises(GsbError):
        lib.check(K.gsb_loss_backward_batch(V, C, 1, 1, x.data_ptr(), x.data_ptr(), rows.data_ptr(), x.data_ptr(),
                                            0.2, x.data_ptr(), lib.stream_ptr()), "gsb_loss_backward_batch")


# ---- 5. large frames -----------------------------------------------------------------------------------------------
def large_frame_boxes(H, W):
    """Output boxes (y0, y1, x0, x1): the 4 corners, the 4 edge midpoints and 8 tile-seam crossings."""
    bh, bw = 32, 64
    ym, xm = (H // 2) // 16 * 16, (W // 2) // 32 * 32
    boxes = [(0, bh, 0, bw), (0, bh, W - bw, W), (H - bh, H, 0, bw), (H - bh, H, W - bw, W),
             (0, bh, xm - bw // 2, xm + bw // 2), (H - bh, H, xm - bw // 2, xm + bw // 2),
             (ym - bh // 2, ym + bh // 2, 0, bw), (ym - bh // 2, ym + bh // 2, W - bw, W)]
    for i in range(1, 9):
        y = round(i * H / (9 * 16)) * 16
        x = round(i * W / (9 * 32)) * 32
        boxes.append((y - bh // 2, y + bh // 2, x - bw // 2, x + bw // 2))
    return boxes


@pytest.mark.parametrize("H,W", [(1080, 1920), (2160, 3840)])
def test_large_frames(H, W):
    """The full frame on the device, checked on crops with 10 px of context; the sums against the full frame in fp64."""
    a, b = L.content("raw", 3, H, W, seed=H)
    sums, maps, grad = loss_kernel(a, b, 0.2)
    recs = []
    for (y0, y1, x0, x1) in large_frame_boxes(H, W):
        (iy, ix), (oy, ox) = L.crop_box(H, W, y0, y1, x0, x1)
        r64, r32 = L.both(a[:, iy, ix], b[:, iy, ix], lam=0.2, N=a.numel())
        crop = lambda r: {k: (v[..., oy, ox] if k != "maps" else v[:, :, oy, ox]) for k, v in r.items()}
        got = dict(grad=grad[:, y0:y1, x0:x1], m_mu=maps[0, :, y0:y1, x0:x1], m_s1=maps[1, :, y0:y1, x0:x1],
                   m_s12=maps[2, :, y0:y1, x0:x1])
        recs += L.check_maps(f"large {H}x{W} box y{y0} x{x0}", got, (crop(r64), crop(r32)),
                             L.regions(y1 - y0, x1 - x0, y0, x0, H, W))
    # the sums: the full frame one plane at a time
    acc = dict(s64=0.0, s32=0.0, sabs=0.0, l64=0.0, l32=0.0, labs=0.0)
    for c in range(3):
        r64, r32 = L.both(a[c], b[c], lam=0.2)
        acc["s64"] += float(r64["ssim"].sum())
        acc["s32"] += float((r32["ssim"].double() - r64["ssim"]).abs().sum())
        acc["sabs"] += float(r64["ssim"].abs().sum())
        acc["l64"] += float(r64["l1"].sum())
        acc["l32"] += float((r32["l1"].double() - r64["l1"]).abs().sum())
        acc["labs"] += float(r64["l1"].sum())
        del r64, r32
    for name, got, want, e32, tot in (("ssim", sums[1], acc["s64"], acc["s32"], acc["sabs"]),
                                      ("l1", sums[0], acc["l64"], acc["l32"], acc["labs"])):
        err, bound = abs(float(got) - want), L.K * e32 + 10 * 2.0 ** -24 * tot
        recs.append(dict(case=f"large {H}x{W}", kind=L.REPORT_TAG, region="sum", quantity=name, got=float(got),
                         want=want, err=err, bound=bound, ok=bool(err <= bound)))
    assert_ok(recs)


# ---- 6. masked L1 (tracking) ---------------------------------------------------------------------------------------
def masked_l1_kernel(img, gt, V=1):
    """gsb_l1_mask_fwd_bwd_batch with threshold 0 on V views [V, C, H, W] (device tensors) -> (sums [V, 2], dL)."""
    lib, K = _L()
    _, C, H, W = img.shape
    sums = torch.zeros(V, 2, dtype=torch.float64, device=DEV)
    dL = torch.empty_like(img)
    lib.check(K.gsb_l1_mask_fwd_bwd_batch(V, C, H, W, img.data_ptr(), gt.data_ptr(), 0.0, sums.data_ptr(),
                                          dL.data_ptr(), lib.stream_ptr()), "gsb_l1_mask_fwd_bwd_batch")
    return sums, dL


SUB = 2.0 ** -149     # the smallest fp32 subnormal


@pytest.mark.parametrize("special", ["zeros_subnormal", "inf", "nan", "neg_inf"])
@pytest.mark.parametrize("n", [2, 3, 5, 13])
def test_masked_l1_threshold_edges(special, n):
    """img > 0 exactly as torch takes it: 0 and -0 are masked out, the smallest subnormal is kept; a NaN or -inf pixel
    is masked out yet makes the loss NaN (NaN * 0), with dL = 0 there, as torch's formula does.  n < 4 runs only the
    scalar tail, n = 5 and 13 groups of four and a tail (which holds a special value too)."""
    vals = dict(zeros_subnormal=[SUB, 0.0, -0.0, -SUB], inf=[SUB, math.inf, 0.0], nan=[SUB, math.nan, -0.0],
                neg_inf=[SUB, -math.inf, 0.0])[special]
    g = torch.Generator().manual_seed(n)
    img = torch.rand(n, generator=g) - 0.3
    gt = torch.rand(n, generator=g)
    k = min(len(vals), n)
    img[:k] = torch.tensor(vals[:k])
    if n > len(vals):
        img[n - 1] = vals[1]                   # in the scalar tail too
    a = img.clone().requires_grad_(True)
    mask = (a > 0.0).float()
    assert float(mask.sum()) > 0
    loss = ((a - gt).abs() * mask).sum() / mask.sum()          # utils/loss_utils.py:17-23
    loss.backward()
    sums, dL = masked_l1_kernel(img.view(1, 1, 1, n).to(DEV), gt.view(1, 1, 1, n).to(DEV))
    s, dL = sums[0].cpu(), dL.cpu().view(n)
    assert float(s[1]) == float(mask.sum())
    want = float(((a - gt).abs() * mask).sum().detach())
    if math.isnan(want) or math.isinf(want):
        assert (math.isnan(float(s[0])) and math.isnan(want)) or float(s[0]) == want, (float(s[0]), want)
    else:
        assert abs(float(s[0]) - want) <= 1e-6 * abs(want), (float(s[0]), want)
    assert torch.equal(dL / float(s[1]), a.grad), (img, dL, a.grad)


def test_masked_l1_4k_sums():
    """Three 4K views: the mask count exact, the sum within the rounding of the kernel's fp32 partial sums."""
    V, C, H, W = 3, 3, 2160, 3840
    g = torch.Generator(device=DEV).manual_seed(1)
    img = torch.rand(V, C, H, W, generator=g, device=DEV) - 0.3
    gt = torch.rand(V, C, H, W, generator=g, device=DEV)
    sums, dL = masked_l1_kernel(img, gt, V)
    sums = sums.cpu()
    mask = img > 0.0
    d = ((img.double() - gt.double()).abs() * mask).flatten(1)
    want, tot = d.sum(1).cpu(), d.abs().sum(1).cpu()
    # terms per thread, from gsb_l1_mask_fwd_bwd_batch's launch: blocks = min(ceil(n4 / 256) + 1, 8 SMs)
    n = C * H * W
    n4 = n // 4
    blocks = min(-(-n4 // 256) + 1, 8 * torch.cuda.get_device_properties(0).multi_processor_count)
    stride = blocks * 256
    terms = 4 * -(-n4 // stride) + -(-(n - 4 * n4) // stride)
    bound = (terms + 8) * 2.0 ** -24 * tot
    err = (sums[:, 0] - want).abs()
    rec = dict(case="masked l1 4K x 3", kind=L.REPORT_TAG, region="sum", quantity="masked l1", terms=terms,
               err=float(err.max()), bound=float(bound.min()), ok=bool((err <= bound).all()))
    record([rec])
    assert torch.equal(sums[:, 1], mask.flatten(1).sum(1).double().cpu())
    assert rec["ok"], rec
    assert torch.equal(dL, torch.sign(img - gt) * mask)
