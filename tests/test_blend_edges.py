"""The blend stage (gs_blend.cu) alone, checked pixel by pixel and Gaussian by Gaussian against an fp64 restatement
(tests/_blend.py) that blends the kernel's own splat records over the kernel's own tile lists, so that every
difference is the blend's.

Each population drives one regime on purpose, asserts with counts that it got there, and is run with every blend
kernel (v2 with bulk staging, v2 cooperative, v1) and in tracking mode (the pose the only input that requires grad:
the 8-slot accumulator layout).  On every pixel the restatement does not flag as threshold-ambiguous, the image,
final_T and n_contrib (exactly) are checked; every slot of every Gaussian's fixed-point accumulator is checked
against tau * (its absolute sum) + 0.5 unit * (warp blocks that flushed it), and the fixed-point scale M bit for bit.
dL/dpixel is zero on the ambiguous pixels, so a legitimate threshold flip cannot reach a moment.
"""
import math

import pytest
import torch

import _binning as BL
import _blend as BD
import _geom as GM
from _parity import DEV, REPORT, settings_for
from test_projection_edges import build_scene, camera_of, on_screen

BLEND_VARIANTS = ((2, 1), (2, 0), (1, 0))    # (blend_version, stage_bulk): v2 bulk TMA staging, v2 cooperative, v1
CHUNK, CHUNK1 = 224, 256                     # kChunk (GSB_CHUNK) of the v2 kernels, kChunk1 of v1
SH_C0 = 0.28209479177387814
# Bounds, in units of fp32 epsilon (2^-24) times each quantity's conditioning-weighted scale (tests/_blend.py), set at
# ~4x the largest H100 measurement over every population, blend kernel and tracking mode of this file (DESIGN.md
# section 2, "Blend at the edges"):
#   MOM_TAU  a fixed-point slot, beyond its quantisation bound 0.5 unit blocks, against tau * mom_abs  (1.84 eps)
#   IMG_TAU  a pixel of the image against kappa * image (colours and bg are >= 0)                    (0.66 eps)
#   T_TAU    final_T against kappa * final_T                                                         (2.2 eps)
MOM_TAU = 8 * BD.EPS32
IMG_TAU = 3 * BD.EPS32
T_TAU = 9 * BD.EPS32


# ---- CPU: decoders and restatement ---------------------------------------------------------------------------------
def test_image_decoder_layout_matches_library():
    """tests/_blend.py restates the ImgView layout of gs_internal.cuh: its total must be gsb_image_bytes (one view)
    and gsb_image_bytes_batch (V views)."""
    import __graft_entry__ as G
    G.build()
    import instantsplat_b200 as I
    L = I.lib()
    for W, H in ((1, 1), (3, 2), (7, 3), (17, 9), (33, 20), (128, 96), (1920, 1080), (3840, 2160), (4095, 17)):
        lay = BD.image_layout(W, H)
        assert lay["total"] == L.gsb_image_bytes(W, H), (W, H)
        assert lay["n_contrib"][0] % 256 == 0 and lay["n_contrib"][0] >= 4 * W * H
        for V in (1, 2, 3, 12):
            assert BD.image_layout(W, H, V)["total"] == L.gsb_image_bytes_batch(W, H, V), (W, H, V)


def _cpu_scene(seed, W=40, H=28, n=150):
    """fp64 splats over a 40x28 frame (3 x 2 tiles, partial at the right and bottom): sigma 2-6 px, random
    orientation, centres up to 4 px outside the frame, opacities 0.3-0.95 plus 12 at 0.995-0.9999 (alpha clamped
    near their centres); every tile's list holds every Gaussian in one depth order (no cull), random but for six
    clamped ones in front."""
    g = torch.Generator().manual_seed(seed)
    r64 = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64)
    xy = torch.stack([-4 + (W + 8) * r64(n), -4 + (H + 8) * r64(n)], 1)
    s = 2.0 + 4.0 * r64(n, 2)
    th = math.pi * r64(n)
    c, sn = torch.cos(th), torch.sin(th)
    a = c * c * s[:, 0] ** 2 + sn * sn * s[:, 1] ** 2
    b = c * sn * (s[:, 0] ** 2 - s[:, 1] ** 2)
    cc = sn * sn * s[:, 0] ** 2 + c * c * s[:, 1] ** 2
    det = a * cc - b * b
    conic = torch.stack([cc / det, -b / det, a / det], 1)
    op = 0.3 + 0.65 * r64(n)
    op[:12] = 0.995 + 0.0049 * r64(12)
    xy[:12] = torch.floor(xy[:12]) + 0.02 * r64(12, 2)           # clamped centres on pixel centres
    rgb = r64(n, 3)
    order = torch.cat([torch.arange(6), 6 + torch.randperm(n - 6, generator=g)])    # six clamped ones in front
    gx, gy = (W + 15) // 16, (H + 15) // 16
    gids = order.repeat(gx * gy)
    ranges = torch.stack([torch.arange(gx * gy) * n, torch.arange(1, gx * gy + 1) * n], 1)
    return dict(xy=xy, conic=conic, opacity=op, rgb=rgb, grid=(gx, gy)), (gids, ranges)


@pytest.mark.parametrize("seed", [1, 2])
def test_restatement_matches_oracle_autograd(seed):
    """The restatement's moments are the exact gradient identities of `O.blend` (fp64, xy, conic, opacity and rgb as
    leaves): dL/dA = -S w dx^2 / 2, dL/dB = -S w dx dy, dL/dC = -S w dy^2 / 2, dL/dopacity = S w / o,
    (S w dx, S w dy) = -Sigma dL/dxy (Sigma the inverse of the conic), dL/drgb = slots 6-8; and its image, final_T,
    n_contrib equal the oracle's, its ambiguity flags contain the oracle's.  The scenes hold clamped and terminated
    pixels."""
    from types import SimpleNamespace
    from oracle import gs_oracle as O
    W, H = 40, 28
    proj, lists = _cpu_scene(seed, W, H)
    bg = torch.tensor([0.3, 0.6, 0.9], dtype=torch.float64)
    leaves = {k: proj[k].clone().requires_grad_(True) for k in ("xy", "conic", "opacity", "rgb")}
    img, aux = O.blend(dict(leaves, grid=proj["grid"]), SimpleNamespace(width=W, height=H, bg=bg), return_aux=True,
                       lists=lists)
    dL = torch.randn(3, H, W, generator=torch.Generator().manual_seed(seed + 10), dtype=torch.float64)
    (img * dL).sum().backward()
    rec = dict(x=proj["xy"][:, 0], y=proj["xy"][:, 1], A=proj["conic"][:, 0], B=proj["conic"][:, 1],
               C=proj["conic"][:, 2], opacity=proj["opacity"], rgb=proj["rgb"])
    r = BD.restate(rec, BD.tile_groups(lists, W, H), W, H, bg, dL, alpha_max=0.99)
    assert torch.allclose(r["image"], img.detach(), rtol=0, atol=1e-12)
    assert torch.allclose(r["final_T"], aux["final_T"], rtol=0, atol=1e-14)
    assert torch.equal(r["n_contrib"], aux["n_contrib"].long())
    assert bool((r["ambiguous"] | ~aux["ambiguous"]).all())
    m = r["mom"]

    def close(a, b, what):
        scale = b.abs().max()
        assert float((a - b).abs().max()) <= 1e-10 * float(scale), (what, float((a - b).abs().max()), float(scale))

    gc = leaves["conic"].grad
    close(-0.5 * m[:, 2], gc[:, 0], "dL/dA")
    close(-m[:, 3], gc[:, 1], "dL/dB")
    close(-0.5 * m[:, 4], gc[:, 2], "dL/dC")
    close(m[:, 5] / proj["opacity"], leaves["opacity"].grad, "dL/dopacity")
    close(m[:, 6:9], leaves["rgb"].grad, "dL/drgb")
    A, B, C = proj["conic"].unbind(1)
    det = A * C - B * B
    gxy = leaves["xy"].grad                                      # Sigma = [[C, -B], [-B, A]] / det
    close(m[:, 0], -(C * gxy[:, 0] - B * gxy[:, 1]) / det, "S w dx")
    close(m[:, 1], -(-B * gxy[:, 0] + A * gxy[:, 1]) / det, "S w dy")
    # the regimes the identities must hold in
    assert int((r["stop_pos"] >= 0).sum()) >= 100, int((r["stop_pos"] >= 0).sum())
    assert int(r["clamped"].sum()) >= 6, int(r["clamped"].sum())
    assert int(r["mom_abs"][:, 5].count_nonzero()) >= 100


# ---- GPU: one frame under every blend kernel -----------------------------------------------------------------------
def _set_variant(ver, bulk):
    import instantsplat_b200 as I
    L = I.lib()
    assert L.gsb_set_option(b"blend_version", ver) == 0 and L.gsb_set_option(b"stage_bulk", bulk) == 0


def _forward(sc, bg, pose_only=False):
    import instantsplat_b200 as I
    prm = {k: v.to(DEV).clone().requires_grad_(not pose_only) for k, v in sc.params.items()}
    pose = sc.poses[0].to(DEV).clone().requires_grad_(True)
    m2 = torch.zeros(sc.P, 3, device=DEV, requires_grad=not pose_only)
    img, _ = I.rasterize_fused(prm["xyz"], prm["rotation"], prm["scaling"], prm["opacity"], prm["f_dc"],
                               prm["f_rest"], pose, m2, settings_for(sc, 0, torch.tensor(bg)))
    grads = lambda: dict({k: v.grad for k, v in prm.items()}, pose=pose.grad, means2D=m2.grad)
    return img, img.grad_fn.st, grads


def _check_moments(name, dec, ref, blocks, dL, pose_only):
    """Every slot against the restatement; the 8-slot layout: slot 5 = dL/db, slot 8 untouched."""
    M = float(dL.abs().max())
    assert torch.tensor(dec["M"], dtype=torch.float32).view(torch.int32) == \
        torch.tensor(M, dtype=torch.float32).view(torch.int32), (name, dec["M"], M)
    if pose_only:
        assert int(dec["raw"][:, 8].count_nonzero()) == 0, f"{name}: slot 8 written in the 8-slot layout"
        ref = dict(mom=ref["mom"][:, [0, 1, 2, 3, 4, 8, 6, 7, 8]], mom_abs=ref["mom_abs"][:, [0, 1, 2, 3, 4, 8, 6, 7, 8]])
        slots = range(8)
    else:
        slots = range(9)
    worst, where, fp = BD.moment_errors(dec, ref, MOM_TAU, blocks, slots)
    return dict(worst=worst, where=where, tau_measured_eps=fp / BD.EPS32)


def check_frame(name, sc, bg, make_dL, variants=BLEND_VARIANTS, tracking=True, groups=None):
    """Render `sc` (view 0) under each blend kernel and tracking mode with dL/dpixel = make_dL(H, W) (zeroed on the
    ambiguous pixels) and check it against the restatement.  groups: restatement pixel groups (default: the tiles of
    the kernel's lists).  -> (record, restatement, decoded records of the first run, dL)."""
    W, H = sc.width, sc.height
    rec = dict(case=f"blend edges: {name}", P=sc.P, width=W, height=H, bg=list(bg), runs={})
    first = None
    try:
        runs = [(v, False) for v in variants] + ([((2, 1), True)] if tracking else [])
        for (ver, bulk), pose_only in runs:
            _set_variant(ver, bulk)
            img, st, grads = _forward(sc, bg, pose_only)
            d = GM.decode(st)
            lists = BL.decode(st)
            BL.check_lists(lists)
            ranges = lists["ranges"].cpu()
            ids = lists["ids"][:lists["status"][BL.ST_R]].cpu()           # the capacity beyond R is scratch
            if first is None:
                ref0 = BD.restate(BD.records_of(d), groups or BD.tile_groups((ids, ranges), W, H), W, H, bg)
                amb = ref0["ambiguous"]
                dL = make_dL(H, W).float() * (~amb)[None]
                ref = BD.restate(BD.records_of(d), groups or BD.tile_groups((ids, ranges), W, H), W, H, bg, dL)
                first = dict(d=d, ids=ids, ranges=ranges)
            else:          # the records and lists do not depend on the blend kernel
                assert all(torch.equal(d[k], first["d"][k]) for k in ("x", "y", "A", "B", "C", "opacity", "rgb"))
                assert torch.equal(ids, first["ids"]) and torch.equal(ranges, first["ranges"])
            img.backward(dL.to(DEV))
            torch.cuda.synchronize()
            ft, nc = BD.decode_image(st)
            ok = ~amb
            key = "tracking" if pose_only else f"v{ver}" + ("" if ver == 1 else (" bulk" if bulk else " coop"))
            kap = ref["kappa"]
            e_img = ((img.detach().cpu().double() - ref["image"]).abs() / (kap * ref["image"].abs()).clamp(min=1e-300)
                     ).amax(0)[ok]
            e_t = ((ft.double() - ref["final_T"]).abs() / (kap * ref["final_T"])[...])[ok]
            n_bad = int((nc != ref["n_contrib"])[ok].sum())
            dec = BD.decode_moments(st, d)
            blocks = ref["blocks4"] if ver == 1 else ref["blocks8"]
            mo = _check_moments(f"{name} {key}", dec, ref, blocks, dL, pose_only)
            r = dict(img_err_eps=float(e_img.max()) / BD.EPS32 if e_img.numel() else 0.0,
                     final_T_err_eps=float(e_t.max()) / BD.EPS32 if e_t.numel() else 0.0,
                     n_contrib_mismatch=n_bad, final_T_min=float(ft.min()), moments=mo,
                     headroom=BD.headroom(dec["value"], d["rec_extent"], dec["M"]))
            rec["runs"][key] = r
            assert n_bad == 0, f"{name} {key}: n_contrib differs on {n_bad} unflagged pixels"
            assert r["final_T_min"] >= 1e-4, f"{name} {key}: final_T below the termination threshold"
            assert r["img_err_eps"] * BD.EPS32 <= IMG_TAU, (name, key, r)
            assert r["final_T_err_eps"] * BD.EPS32 <= T_TAU, (name, key, r)
            assert mo["worst"] <= 1.0, f"{name} {key}: moment error over its bound: {mo}"
            assert r["headroom"] < 2 ** BD.HEADROOM_BITS, (name, key, r["headroom"])
            if not pose_only:
                g = grads()
                assert all(bool(torch.isfinite(v).all()) for v in g.values() if v is not None), f"{name} {key}"
    finally:
        _set_variant(2, 1)
        REPORT.append(rec)
    rec["ambiguous"] = int(amb.sum())
    rec["headroom_max"] = max(r["headroom"] for r in rec["runs"].values())
    return rec, ref, first["d"], dL


def signed_dL(seed):
    return lambda H, W: 2 * torch.rand(3, H, W, generator=torch.Generator().manual_seed(seed)) - 1


# ---- scenes ----------------------------------------------------------------------------------------------------------
def saturation_scene(W=128, H=96, n=12000, seed=401):
    """Small Gaussians (sigma 0.8-2 px) at distinct depths z 2-6, centres denser to the right (density ~ x^2, so the
    left edge stays translucent), opacities 0.3-0.9999, mostly faint at the bottom of the frame: 20-100 layers per
    pixel over most of it and culled lists of 1000-4000 entries, whose walk ends anywhere from the first staging chunk
    to the third."""
    g = torch.Generator().manual_seed(seed)
    _, _, tx, ty, fx = camera_of(W, H)
    z = 2.0 + 4.0 * torch.rand(n, generator=g, dtype=torch.float64)
    u = W * torch.rand(n, generator=g, dtype=torch.float64) ** (1 / 3)
    v = H * torch.rand(n, generator=g, dtype=torch.float64)
    pc = torch.stack([((2 * u + 1) / W - 1) * z * tx, ((2 * v + 1) / H - 1) * z * ty, z], 1)
    s_px = 0.8 + 1.2 * torch.rand(n, generator=g, dtype=torch.float64)
    sig = (s_px * z / fx)[:, None].expand(n, 3) * (0.8 + 0.4 * torch.rand(n, 3, generator=g, dtype=torch.float64))
    op = 0.3 + 0.6999 * torch.rand(n, generator=g, dtype=torch.float64) ** (1.0 + 16.0 * v / H)
    return build_scene([(pc, sig, op)], W, H, seed=seed + 1)


def clamp_scene(W=128, H=96, seed=411):
    """900 near-opaque Gaussians (opacity 0.995-0.99999, sigma 2-6 px, centres 0.1-0.3 px from a pixel centre so that
    o G > 0.99 at one to a few pixels each, none within rounding of power = 0) between a translucent layer in front (z 1.5-2, opacity 0.05-0.25) and one behind (z 6-8,
    opacity 0.2-0.7)."""
    g = torch.Generator().manual_seed(seed)
    _, _, tx, ty, fx = camera_of(W, H)
    r = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64)
    parts = []
    for n, z0, z1, o0, o1, s0, s1 in ((900, 2.5, 5.5, 0.995, 0.99999, 2.0, 6.0), (500, 1.5, 2.0, 0.05, 0.25, 2.0, 6.0),
                                      (800, 6.0, 8.0, 0.2, 0.7, 2.0, 6.0)):
        z = z0 + (z1 - z0) * r(n)
        u, v = torch.floor(W * r(n)) + 0.1 + 0.2 * r(n), torch.floor(H * r(n)) + 0.1 + 0.2 * r(n)
        pc = torch.stack([((2 * u + 1) / W - 1) * z * tx, ((2 * v + 1) / H - 1) * z * ty, z], 1)
        sig = ((s0 + (s1 - s0) * r(n)) * z / fx)[:, None].expand(n, 3).contiguous()
        parts.append((pc, sig, o0 + (o1 - o0) * r(n)))
    return build_scene(parts, W, H, seed=seed + 1, rot=torch.tensor([[1.0, 0, 0, 0]]).expand(2200, 4))


def edge_scene(W, H, seed):
    """Gaussians of sigma 0.5-4 px over a frame of W x H widened by 6 px on every side (some centred outside it),
    opacity 0.2-0.95, plus one larger one centred 3 px beyond each corner."""
    g = torch.Generator().manual_seed(seed)
    fx = camera_of(W, H)[4]
    n = max(24, 3 * W * H // 8)
    z = 2.0 + 3.0 * torch.rand(n, generator=g, dtype=torch.float64)
    pc = on_screen(n, W, H, z, g, margin=6.0)
    sig = ((0.5 + 3.5 * torch.rand(n, generator=g, dtype=torch.float64)) * z / fx)[:, None].expand(n, 3).contiguous()
    _, _, tx, ty, _ = camera_of(W, H)
    cu = torch.tensor([-3.0, W + 2.0, -3.0, W + 2.0], dtype=torch.float64)
    cv = torch.tensor([-3.0, -3.0, H + 2.0, H + 2.0], dtype=torch.float64)
    zc = torch.full((4,), 2.5, dtype=torch.float64)
    corners = torch.stack([((2 * cu + 1) / W - 1) * zc * tx, ((2 * cv + 1) / H - 1) * zc * ty, zc], 1)
    parts = [(pc, sig, 0.2 + 0.75 * torch.rand(n, generator=g, dtype=torch.float64)),
             (corners, (6.0 * zc / fx)[:, None].expand(4, 3).contiguous(), torch.full((4,), 0.8, dtype=torch.float64))]
    return build_scene(parts, W, H, seed=seed + 1)


# ---- populations -----------------------------------------------------------------------------------------------------
def _reached_saturation(ref):
    sp = ref["stop_pos"]
    H, W = sp.shape
    term = sp >= 0
    t8 = term[:H // 8 * 8].reshape(H // 8, 2, 4, W)
    return dict(terminated_frac=float(term.float().mean()),
                stop_at_chunk_m1_0_p1=[int((sp == k).sum()) for k in (CHUNK - 1, CHUNK, CHUNK + 1)],
                stop_at_v1_chunk_m1_0_p1=[int((sp == k).sum()) for k in (CHUNK1 - 1, CHUNK1, CHUNK1 + 1)],
                stop_at_group_end=int((term & (sp % 32 == 31)).sum()),
                stop_per_chunk=[int((term & (sp // CHUNK == c)).sum()) for c in range(4)],
                lane_pairs_one_terminated=int((t8[:, 0] ^ t8[:, 1]).sum()),
                pixels_final_T_over_1e_2=int((ref["final_T"] > 1e-2).sum()))


@pytest.mark.gpu
def test_saturation_stacks():
    """20-100 layers per pixel: early termination on most pixels, at list positions spread over three staging
    chunks, on both sides of every chunk boundary and at the ends of 32-entry ballot groups, and in only one pixel of
    many v2 lane pairs."""
    sc = saturation_scene()
    rec, ref, _, _ = check_frame("saturation stacks", sc, (0.3, 0.6, 0.9), signed_dL(1))
    rec["reached"] = r = _reached_saturation(ref)
    assert r["terminated_frac"] >= 0.7, r
    assert min(r["stop_at_chunk_m1_0_p1"]) >= 1 and min(r["stop_at_v1_chunk_m1_0_p1"]) >= 1, r
    assert r["stop_per_chunk"][1] >= 100 and r["stop_per_chunk"][2] >= 1 and r["stop_at_group_end"] >= 100, r
    assert r["lane_pairs_one_terminated"] >= 10, r


@pytest.mark.gpu
def test_alpha_clamp():
    """Hundreds of live (pixel, Gaussian) pairs with o G > 0.99, in front of and behind other layers: the backward
    weights their moments by the unclamped o G and rebuilds T from the clamped alpha."""
    sc = clamp_scene()
    rec, ref, d, dL = check_frame("alpha clamp", sc, (0.1, 0.2, 0.3), signed_dL(2))
    cl = ref["clamped"] > 0
    rec["reached"] = r = dict(clamped_pairs=int(ref["clamped"].sum()), clamped_gaussians=int(cl.sum()),
                              clamped_with_moment=int((cl & (ref["mom"][:, 5] != 0)).sum()))
    assert r["clamped_pairs"] >= 200 and r["clamped_with_moment"] >= 150, r


EDGE_FRAMES = ((1, 1), (3, 2), (7, 3), (8, 4), (9, 5), (15, 12), (17, 9), (33, 20), (47, 31))


@pytest.mark.gpu
def test_frame_edges():
    """Frames of every width and height remainder mod 8 these sizes allow, with lanes whose second pixel (y + 4) lies
    below the frame and Gaussians centred outside it."""
    reached = dict(w_mod8=set(), h_mod8=set(), lanes_half_off=0, centred_outside=0)
    for k, (W, H) in enumerate(EDGE_FRAMES):
        sc = edge_scene(W, H, 420 + k)
        rec, ref, d, _ = check_frame(f"frame edges {W}x{H}", sc, (0.3, 0.6, 0.9), signed_dL(3 + k))
        reached["w_mod8"].add(W % 8)
        reached["h_mod8"].add(H % 8)
        reached["lanes_half_off"] += sum(1 for y in range(H) if y % 8 < 4 and y + 4 >= H) * W
        live = ref["pairs"] > 0
        out = (d["x"] < -0.5) | (d["x"] > W - 0.5) | (d["y"] < -0.5) | (d["y"] > H - 0.5)
        reached["centred_outside"] += int((live & out).sum())
    r = dict(reached, w_mod8=sorted(reached["w_mod8"]), h_mod8=sorted(reached["h_mod8"]))
    REPORT.append(dict(case="blend edges: frame edges, reached", **r))
    assert r["w_mod8"] == [0, 1, 3, 7] and r["h_mod8"] == [1, 2, 3, 4, 5, 7], r
    assert r["lanes_half_off"] >= 20 and r["centred_outside"] >= 20, r


@pytest.mark.gpu
@pytest.mark.parametrize("bg", [(0.0, 0.0, 0.0), (1.0, 1.0, 1.0), (0.3, 0.6, 0.9)])
def test_background(bg):
    """The saturation scene under three backgrounds: the backward's T_final / (1 - alpha) bg.dL term on the pixels
    its translucent side leaves with final_T >> 1e-4."""
    sc = saturation_scene()
    rec, ref, _, _ = check_frame(f"background {bg}", sc, bg, signed_dL(4), tracking=False)
    rec["reached"] = r = dict(pixels_final_T_over_1e_2=int((ref["final_T"] > 1e-2).sum()),
                              pixels_final_T_over_0_5=int((ref["final_T"] > 0.5).sum()))
    assert r["pixels_final_T_over_1e_2"] >= 50, r


def _patch(H, W):
    dL = torch.zeros(3, H, W)
    dL[:, 40:45, 60:65] = 2 * torch.rand(3, 5, 5, generator=torch.Generator().manual_seed(5)) - 1
    return dL


def _hot(H, W):
    dL = 2 * torch.rand(3, H, W, generator=torch.Generator().manual_seed(6)) - 1
    dL[2, H - 1, W - 1] = 1e6                                      # the last element of the buffer
    return dL


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["signed", "patch", "hot last pixel", "zero"])
def test_dL_structure(kind):
    """One 128x96 scene under four dL/dpixel: signed random; zero but for a 5x5 patch; one value 1e6 times the rest at
    the last element of the buffer (M is set by it; every other Gaussian's moments are 1e-6 M or less); all zeros
    (M floored at 1e-20: every gradient exactly 0 and finite)."""
    sc = clamp_scene(seed=431)
    make = dict(signed=signed_dL(7), patch=_patch, zero=lambda H, W: torch.zeros(3, H, W))
    rec, ref, d, dL = check_frame(f"dL structure: {kind}", sc, (0.3, 0.6, 0.9), make.get(kind, _hot))
    if kind == "hot last pixel":
        assert float(dL[2, -1, -1]) == 1e6, "the hot pixel is threshold-ambiguous"
        assert int(ref["n_contrib"][-1, -1]) >= 1
    if kind == "zero":
        _set_variant(2, 1)
        try:
            img, st, grads = _forward(sc, (0.3, 0.6, 0.9))
            img.backward(torch.zeros_like(img))
            g = grads()
            assert all(bool(torch.isfinite(v).all()) and int(v.count_nonzero()) == 0 for v in g.values()), \
                "non-zero or non-finite gradient from dL = 0"
            assert int(BD.decode_moments(st, GM.decode(st))["raw"].count_nonzero()) == 0
        finally:
            _set_variant(2, 1)


@pytest.mark.gpu
@pytest.mark.parametrize("where", ["centre", "corner"])
def test_accumulator_range_4k(where):
    """One frame-filling near-opaque Gaussian (sigma 5000 px, alpha clamped over the middle of the frame) at
    3840x2160, rgb (50, 35, 20) on a black background, dL/dpixel = 1 everywhere: centred, the largest second moments
    the frame allows for its extent; at a corner, the largest first moments.  The decoded moments must equal the fp64
    sums over the pixel grid within tau: no wrap-around of the 64-bit accumulators."""
    W, H = 3840, 2160
    _, _, tx, ty, fx = camera_of(W, H)
    u, v = (W / 2 - 0.5, H / 2 - 0.5) if where == "centre" else (2.3, 3.6)
    z = 2.0
    pc = torch.tensor([[((2 * u + 1) / W - 1) * z * tx, ((2 * v + 1) / H - 1) * z * ty, z]], dtype=torch.float64)
    sc = build_scene([(pc, torch.full((1, 3), 5000.0 * z / fx, dtype=torch.float64),
                       torch.tensor([0.99999], dtype=torch.float64))], W, H, seed=441,
                     rot=torch.tensor([[1.0, 0.0, 0.0, 0.0]]))
    sc.params["f_dc"] = ((torch.tensor([50.0, 35.0, 20.0]) - 0.5) / SH_C0).reshape(1, 1, 3)
    groups = list(BD.strip_groups(torch.tensor([0]), W, H))
    rec, ref, d, dL = check_frame(f"accumulator range 4K, {where}", sc, (0.0, 0.0, 0.0),
                                  lambda H, W: torch.ones(3, H, W), groups=groups)
    assert float(d["rgb"][0, 0]) > 49.9 and int(d["radii"][0]) > 10000
    rec["reached"] = r = dict(extent=float(d["rec_extent"][0]), clamped_pixels=int(ref["clamped"][0]),
                              headroom=rec["headroom_max"], headroom_limit=2 ** BD.HEADROOM_BITS)
    assert r["clamped_pixels"] >= 1000 and r["headroom"] >= (40 if where == "centre" else 0.1), r


@pytest.mark.gpu
def test_scale_invariance_bit_for_bit():
    """dL/dpixel times 2^40 or 2^-40 multiplies every gradient the backward returns, the pose gradient included, by
    exactly that factor, in the full backward and in tracking mode: the fixed-point unit scales with M and nothing
    downstream has an absolute epsilon or a non-linearity in dL."""
    sc = clamp_scene(seed=451)
    w = 2 * torch.rand(3, sc.height, sc.width, generator=torch.Generator().manual_seed(9)) - 1
    out = {}
    for pose_only in (False, True):
        res = {}
        for f in (1.0, 2.0 ** 40, 2.0 ** -40):
            img, st, grads = _forward(sc, (0.3, 0.6, 0.9), pose_only)
            img.backward((w * f).to(DEV))
            res[f] = {k: v.detach().clone() for k, v in grads().items() if v is not None}
        for f in (2.0 ** 40, 2.0 ** -40):
            assert int(res[1.0]["pose"].count_nonzero()) > 0
            for k, v in res[1.0].items():
                assert torch.equal(res[f][k], v * f), f"{k} (pose only {pose_only}): not scaled by exactly {f}"
        out["tracking" if pose_only else "full"] = sorted(res[1.0])
    REPORT.append(dict(case="blend edges: scale invariance 2^+-40", bit_identical=True, tensors=out))
