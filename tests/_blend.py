"""Read the per-pixel state and the fixed-point moments the blend kernels (gs_blend.cu) leave behind, and restate the
blend and its backward in fp64 on the kernel's own splat records and tile lists.

The image buffer is laid out by `img_view` in instantsplat_b200/csrc/gs_internal.cuh (ImgView), for V views of W x H:

    final_T    [V H W] f32   transmittance after the last contributor
    n_contrib  [V H W] u32   1 + list position of the last contributor (0: none), at byte align_up(4 V H W)

`image_layout` restates that; a CPU test pins it to `gsb_image_bytes` and `gsb_image_bytes_batch`.

After a backward, the geometry buffer's `dacc` part holds nine 64-bit fixed-point sums per Gaussian and `dscale` the
float bits of M = max |dL/dpixel|.  Slot k of Gaussian i counts in units of 1 / fix_scale(k, e_i, M) =
2^-50 M (e_i + 1)^fix_exp(k), e_i the record's extent.  `decode_moments` converts them with the exact unit; the device
computes its scale with rcp.approx, so a decoded value may differ from the device's by a few ulps of itself.

`restate` computes, in fp64 from the same records and lists, everything the blend forward writes (image, final_T,
n_contrib) and the nine sums of its backward, per Gaussian:

    [S w dx, S w dy, S w dx^2, S w dx dy, S w dy^2, S w, dL/dr, dL/dg, dL/db],   w = dL/dalpha * opacity * G

(dx = x - pixel, alpha straight through min(0.99f, .) as in `O.blend`), together with each sum's error scale: the
same sum over the absolute values of every part of every term, each weighted by its pixel's conditioning
kappa = 1 + S_live (1 + alpha / (1 - alpha) unless alpha is clamped): the transmittance the backward rebuilds from
final_T divides by every 1 - alpha, which turns an fp32 rounding of alpha into alpha / (1 - alpha) roundings of T; a
clamped alpha is the same constant in both arms.
"""
import torch

from oracle import gs_oracle as O

import _binning as BL
import _geom as GM

FIX_EXP = (3, 3, 4, 4, 4, 2, 2, 2, 2)      # fix_exp(k) of gs_internal.cuh
EPS32 = 2.0 ** -24
ALPHA_MAX = float(torch.tensor(0.99, dtype=torch.float32))   # the kernels' clamp, min(0.99f, alpha)
HEADROOM_BITS = 13                          # the unit 2^-50 M (e + 1)^k leaves |slot| < 2^13 M (e + 1)^k in 63 bits


def image_layout(W, H, V=1):
    """Byte offset and length of each ImgView array, and the total (= gsb_image_bytes_batch(W, H, V))."""
    hw = max(int(V), 1) * W * H
    return dict(final_T=(0, 4 * hw), n_contrib=(BL.align_up(4 * hw), 4 * hw), total=2 * BL.align_up(4 * hw))


def decode_image(st):
    """final_T [H, W] (f32) and n_contrib [H, W] (int64) of a one-view forward (`_State`), as CPU tensors."""
    W, H = st.W, st.H
    lay = image_layout(W, H)
    assert lay["total"] <= st.image.numel(), (lay, st.image.numel())
    b = st.image.detach().cpu()
    ft = b[:4 * W * H].view(torch.float32).reshape(H, W).clone()
    off = lay["n_contrib"][0]
    nc = b[off:off + 4 * W * H].view(torch.int32).long().reshape(H, W) & 0xFFFFFFFF
    return ft, nc


def decode_moments(st, d):
    """The backward's accumulators of a one-view frame: dict(raw [P, 9] int64, M (the float dscale holds), unit [P, 9],
    value [P, 9] = raw * unit, all fp64 but raw).  d: `_geom.decode(st)` (for the extents)."""
    P = int(st.P)
    lay = GM.geom_layout(P)
    g = st.geom.detach().cpu()
    off = lay["dacc"][0]
    raw = g[off:off + 8 * 9 * P].view(torch.int64).reshape(P, 9).clone()
    off = lay["dscale"][0]
    M = float(g[off:off + 4].view(torch.float32)[0])
    unit = fix_unit(d["rec_extent"], M)
    return dict(raw=raw, M=M, unit=unit, value=raw.double() * unit)


def fix_unit(extent, M):
    """Exact unit 2^-50 max(M, 1e-20) (e + 1)^fix_exp(k) of every slot [P, 9] (fp64)."""
    m = max(float(torch.tensor(M, dtype=torch.float32)), float(torch.tensor(1e-20, dtype=torch.float32)))
    e1 = extent.double()[:, None] + 1.0
    return m * 2.0 ** -50 * e1 ** torch.tensor(FIX_EXP, dtype=torch.float64)[None]


def last_contributor(ids, ranges, n_contrib, W):
    """Gaussian id of each pixel's last contributor (-1: none), from a tile list and n_contrib [H, W]."""
    H = n_contrib.shape[0]
    gx = (W + O.BLOCK - 1) // O.BLOCK
    ys, xs = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    t = (ys // O.BLOCK) * gx + xs // O.BLOCK
    nc = n_contrib.long()
    pos = ranges[t, 0].long() + nc - 1
    out = torch.full((H, W), -1, dtype=torch.long)
    has = nc > 0
    out[has] = ids.long()[pos[has]]
    return out


# ---- the fp64 restatement ----------------------------------------------------------------------------------------
def tile_groups(lists, W, H):
    """(Gaussian ids front to back, pixel x, pixel y) of every tile with a non-empty list.  lists: (ids, ranges)."""
    ids, ranges = lists
    gx, gy = (W + O.BLOCK - 1) // O.BLOCK, (H + O.BLOCK - 1) // O.BLOCK
    for t in range(gx * gy):
        s, e = int(ranges[t, 0]), int(ranges[t, 1])
        if e <= s:
            continue
        ty, tx = divmod(t, gx)
        x0, y0 = tx * O.BLOCK, ty * O.BLOCK
        ys, xs = torch.meshgrid(torch.arange(y0, min(y0 + O.BLOCK, H)), torch.arange(x0, min(x0 + O.BLOCK, W)),
                                indexing="ij")
        yield ids[s:e].long(), xs.reshape(-1), ys.reshape(-1)


def strip_groups(g, W, H, rows=64):
    """One list `g` shared by every tile (a frame-filling Gaussian), in strips of `rows` (a multiple of 8) pixel rows:
    the restatement of a 4K frame without a Python loop over its tiles."""
    for y0 in range(0, H, rows):
        ys, xs = torch.meshgrid(torch.arange(y0, min(y0 + rows, H)), torch.arange(W), indexing="ij")
        yield g, xs.reshape(-1), ys.reshape(-1)


def restate(rec, groups, W, H, bg, dL=None, t_eps=O.T_EPS, alpha_max=ALPHA_MAX):
    """The blend forward and (dL [3, H, W] given) backward in fp64 over `groups` (tile_groups / strip_groups).

    rec: dict of fp64 per-Gaussian tensors x, y, A, B, C (conic: power = -(A dx^2 + C dy^2) / 2 - B dx dy), opacity,
    rgb [P, 3] (`_geom.decode` gives exactly these for the kernel's records).  Returns dict with per pixel [H, W]:
    image [3, H, W], final_T, n_contrib, kappa, ambiguous (`O.blend`'s rule, with the termination window widened to
    the fp32 rounding of the transmittance: 8 eps kappa T), stop_pos (list position of the entry that ended the walk,
    -1: none); per Gaussian: blocks8 / blocks4 (warp blocks of 8x8 (v2) / 8x4 (v1) pixels with a live pixel), pairs
    (live (pixel, Gaussian) pairs), clamped (live pairs with opacity * G > alpha_max); and with dL: mom [P, 9],
    mom_abs [P, 9].  alpha_max: 0.99 restates `O.blend`, whose clamp is the fp64 0.99."""
    P = rec["x"].numel()
    bg = torch.as_tensor(bg, dtype=torch.float64)
    img = bg[:, None, None].expand(3, H, W).clone()
    final_T = torch.ones(H, W, dtype=torch.float64)
    n_contrib = torch.zeros(H, W, dtype=torch.long)
    kappa = torch.ones(H, W, dtype=torch.float64)
    amb = torch.zeros(H, W, dtype=torch.bool)
    stop_pos = torch.full((H, W), -1, dtype=torch.long)
    blocks8 = torch.zeros(P, dtype=torch.long)
    blocks4 = torch.zeros(P, dtype=torch.long)
    pairs = torch.zeros(P, dtype=torch.long)
    clamped = torch.zeros(P, dtype=torch.long)
    mom = torch.zeros(P, 9, dtype=torch.float64)
    mom_abs = torch.zeros(P, 9, dtype=torch.float64)
    gbx = (W + 7) // 8
    for g, px, py in groups:
        n = g.numel()
        fx, fy = px.double(), py.double()
        dx = rec["x"][g][:, None] - fx[None]
        dy = rec["y"][g][:, None] - fy[None]
        A, B, C = rec["A"][g][:, None], rec["B"][g][:, None], rec["C"][g][:, None]
        power = -0.5 * (A * dx * dx + C * dy * dy) - B * dx * dy
        op = rec["opacity"][g][:, None]
        aw = op * torch.exp(power.clamp(max=0.0))                 # opacity * G: the straight-through weight
        alpha = aw.clamp(max=alpha_max)
        amp = torch.where(aw < alpha_max, alpha / (1 - alpha), torch.zeros_like(alpha))   # rounding gain of 1 - alpha
        valid = (power <= 0) & (alpha >= O.ALPHA_MIN)
        a0 = torch.where(valid, alpha, torch.zeros_like(alpha))
        Tincl = torch.cumprod(1 - a0, 0)
        stop = valid & (Tincl < t_eps)
        done = torch.cummax(stop.to(torch.int8), 0)[0].bool()
        live = valid & ~done
        a = torch.where(live, alpha, torch.zeros_like(alpha))
        Tin = torch.cumprod(1 - a, 0)
        Tex = torch.cat([torch.ones_like(Tin[:1]), Tin[:-1]], 0)
        wgt = a * Tex
        Tf = Tin[-1]
        col = rec["rgb"][g]
        kap = 1.0 + (live * (1 + amp)).sum(0)
        # O.blend's threshold-ambiguity rule; the T window also covers the fp32 roundings of the running product
        cond = 1.0 + torch.cumsum(valid * (1 + amp), 0)
        amb_p = ((alpha * 255.0 - 1.0).abs() < 5e-4) \
            | (valid & ((Tincl - t_eps).abs() < torch.clamp(8 * EPS32 * cond * Tincl, min=1e-7))) \
            | ((power > -1e-7) & (power != 0) & (op >= O.ALPHA_MIN))
        amb_p = amb_p & ~torch.cat([torch.zeros_like(done[:1]), done[:-1]], 0)
        pos1 = torch.arange(1, n + 1)[:, None]
        img[:, py, px] = (wgt.t() @ col).t() + Tf[None] * bg[:, None]
        final_T[py, px] = Tf
        n_contrib[py, px] = (pos1 * live).amax(0)
        kappa[py, px] = kap
        amb[py, px] = amb_p.any(0)
        stop_pos[py, px] = torch.where(stop.any(0), (pos1 * stop).masked_fill(~stop, n + 1).amin(0) - 1,
                                       torch.full_like(px, -1))
        for blk, bh in ((blocks8, 8), (blocks4, 4)):
            bid = ((py // bh) * gbx + px // 8)
            ub, inv = torch.unique(bid, return_inverse=True)
            hit = torch.zeros(n, ub.numel(), dtype=torch.float64).index_add_(1, inv, live.double())
            blk.index_add_(0, g, (hit > 0).sum(1))
        pairs.index_add_(0, g, live.sum(1))
        clamped.index_add_(0, g, (live & (aw > alpha_max)).sum(1))
        if dL is None:
            continue
        dLp = dL[:, py, px].double()                              # [3, npix]
        cd = col @ dLp                                            # c_k . dL   [n, npix]
        cabs = col.abs() @ dLp.abs()
        bgd = bg @ dLp
        bgabs = bg.abs() @ dLp.abs()

        def behind(v):                                            # S_{j > k} v_j
            return torch.flip(torch.cumsum(torch.flip(v, [0]), 0), [0]) - v

        one_m = 1 - a
        # dL/dalpha_k = T_k c_k.dL - S_{j>k} alpha_j T_j c_j.dL / (1 - alpha_k) - T_final bg.dL / (1 - alpha_k)
        dLda = Tex * cd - (behind(wgt * cd) + Tf[None] * bgd[None]) / one_m
        dLda_abs = Tex * cabs + (behind(wgt * cabs) + Tf[None] * bgabs[None]) / one_m
        w = torch.where(live, dLda * aw, torch.zeros_like(aw))
        wa = torch.where(live, dLda_abs * aw, torch.zeros_like(aw)) * kap[None]
        adx, ady = dx.abs(), dy.abs()
        terms = (w * dx, w * dy, w * dx * dx, w * dx * dy, w * dy * dy, w)
        aterms = (wa * adx, wa * ady, wa * adx * adx, wa * adx * ady, wa * ady * ady, wa)
        for k in range(6):
            mom[:, k].index_add_(0, g, terms[k].sum(1))
            mom_abs[:, k].index_add_(0, g, aterms[k].sum(1))
        for c in range(3):
            mom[:, 6 + c].index_add_(0, g, (wgt * dLp[c][None]).sum(1))
            mom_abs[:, 6 + c].index_add_(0, g, (wgt * dLp[c].abs()[None] * kap[None]).sum(1))
    out = dict(image=img, final_T=final_T, n_contrib=n_contrib, kappa=kappa, ambiguous=amb, stop_pos=stop_pos,
               blocks8=blocks8, blocks4=blocks4, pairs=pairs, clamped=clamped)
    if dL is not None:
        out.update(mom=mom, mom_abs=mom_abs)
    return out


def records_of(d):
    """The restatement's inputs from `_geom.decode`: the kernel's records in fp64."""
    return {k: d[k] for k in ("x", "y", "A", "B", "C", "opacity", "rgb")}


def headroom(value, extent, M):
    """max over Gaussians and slots of |slot| / (M (e + 1)^fix_exp(k)), to hold against 2^13."""
    if M <= 0:
        return 0.0
    r = value.abs() / (fix_unit(extent, M) * 2.0 ** 50)
    return float(r.max()) if r.numel() else 0.0


def moment_errors(dec, ref, tau, blocks, slots=range(9)):
    """Each decoded slot against the restatement: |dec - mom| <= tau mom_abs + 0.5 unit blocks + 2^-20 |mom|
    (the last term: the device's scale, rcp.approx, differs from the exact unit by a few ulps).  -> (worst ratio of
    error to bound, its (Gaussian, slot), worst error over tau-scale alone among the Gaussians whose quantisation term
    is below a tenth of it (the measured fp32 error))."""
    val, unit = dec["value"], dec["unit"]
    worst, where, fp = 0.0, None, 0.0
    for k in slots:
        err = (val[:, k] - ref["mom"][:, k]).abs()
        q = 0.5 * unit[:, k] * blocks.double()
        bound = tau * ref["mom_abs"][:, k] + q + 2.0 ** -20 * ref["mom"][:, k].abs()
        r = err / torch.clamp(bound, min=1e-300)
        i = int(r.argmax()) if r.numel() else 0
        if r.numel() and float(r[i]) > worst:
            worst, where = float(r[i]), (i, k)
        sel = (q < 0.1 * tau * ref["mom_abs"][:, k]) & (ref["mom_abs"][:, k] > 0)
        if bool(sel.any()):
            fp = max(fp, float((torch.clamp(err - q, min=0) / ref["mom_abs"][:, k])[sel].max()))
    return worst, where, fp
