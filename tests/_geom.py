"""Read the per-Gaussian splat records a forward left in its geometry buffer and check them against the fp64 oracle.

The geometry buffer is laid out by `geom_view` in instantsplat_b200/csrc/gs_internal.cuh (GeomView); each part starts
on a 256-byte boundary, and P-sized parts are sized for max(P, 1):

    cam        CamConst (64 words)
    rec        [3P] float4   x, y, A', B' | C', opacity, qthr', id (bits) | r, g, b, extent
                             (conic and cull threshold in the log2 domain: A' = -log2e A / 2, B' = -log2e B,
                             C' = -log2e C / 2, qthr' = log2e qthr / 2; extent: of the fixed-point unit,
                             fix_extent in gs_internal.cuh)
    brec       [P]  float4   depth, rect x (rx0 | rx1 << 16), rect y (ry0 | ry1 << 16), keep mask (bits)
    tiles      [P]  u32      tile instances after the cull
    clamped    [P]  u8       bit c: colour channel c was clamped at 0
    dacc       [9P] u64      fixed-point backward accumulators
    dscale     [1]  u32
    pose_part  [ceil(P / 128) * 16] f32
    pose_acc   [16] f32
    status     [8]  u32      (frame.py ST_*)
    aux        [64] u32      [0] = number of Gaussians queued for k_big_rects
    tcount, tstart, tcursor, q_large, q_huge   [65536] u32 each
    q_big      [P]  u32

`geom_layout` restates that; a CPU test pins it to `gsb_geom_bytes` and `gsb_status_device`.

`check_records` compares every decoded record with `O.project` in fp64.  A Gaussian whose kernel result may
legitimately differ from the fp64 one -- its depth within rounding of the near plane, its radius within rounding of an
integer or its rect of a tile boundary, a colour channel within rounding of the clamp at 0, its opacity within
rounding of the 1/255 cutoff -- is flagged, counted and exempted from the comparison that depends on the flip, and
from nothing else.
"""
import torch

from oracle import gs_oracle as O

import _binning as BL

PT = 128                 # kPT: Gaussians per CTA of the per-Gaussian kernels
MAX_TILES = 65536        # kMaxTiles
DACC_SLOTS = 9           # kDaccSlots
CAMCONST_BYTES = 256     # sizeof(CamConst): 64 four-byte words
LOG2E = float(torch.tensor(1.4426950408889634, dtype=torch.float32))   # kLog2e as the kernels hold it
NEAR = 0.2               # kNear
# bound on the relative error of every float field of a record (see check_records for each field's scale): 5x the
# largest error measured on an H100 over every population of tests/test_projection_edges.py (4.0e-6, DESIGN.md section 2)
REC_TOL = 2e-5


def geom_layout(P, V=1, ntiles=0):
    """Byte offset and length of each GeomView part, and the total (= gsb_geom_bytes(P); for a batch of V views of
    frames of ntiles 16x16 tiles, gsb_geom_bytes_batch: every per-record part holds V * P records, cam, dscale,
    pose_part and pose_acc one row per view, the per-tile parts max(V * ntiles, kMaxTiles) slots)."""
    pp = max(int(P), 1)
    nv = max(int(V), 1)
    vp = nv * pp
    nb = (pp + PT - 1) // PT
    ts = max(nv * int(ntiles), MAX_TILES)
    parts = (("cam", nv * CAMCONST_BYTES), ("rec", vp * 48), ("brec", vp * 16), ("tiles", vp * 4), ("clamped", vp),
             ("dacc", vp * DACC_SLOTS * 8), ("dscale", nv * 4), ("pose_part", nv * nb * 16 * 4),
             ("pose_acc", nv * 16 * 4), ("status", 8 * 4), ("aux", 64 * 4), ("tcount", ts * 4), ("tstart", ts * 4),
             ("tcursor", ts * 4), ("q_large", ts * 4), ("q_huge", ts * 4), ("q_big", vp * 4))
    out, off = {}, 0
    for name, nbytes in parts:
        out[name] = (off, nbytes)
        off += BL.align_up(nbytes)
    out["total"] = off
    return out


def decode(st):
    """Per-Gaussian records of a forward (`_State`: `img.grad_fn.st`) as CPU tensors."""
    P = int(st.P)
    lay = geom_layout(P)
    assert lay["total"] <= st.geom.numel(), (lay["total"], st.geom.numel())
    g = st.geom.detach().cpu()

    def part(name, n, dt):
        off = lay[name][0]
        return g[off:off + n * torch.empty(0, dtype=dt).element_size()].view(dt)

    rec = part("rec", 12 * P, torch.float32).reshape(P, 3, 4)
    recb = rec.view(torch.int32)
    brec = part("brec", 4 * P, torch.float32).reshape(P, 4)
    bb = brec.view(torch.int32).long() & 0xFFFFFFFF
    r64 = rec.double()
    return dict(
        P=P, x=r64[:, 0, 0], y=r64[:, 0, 1],
        A=r64[:, 0, 2] / (-0.5 * LOG2E), B=r64[:, 0, 3] / -LOG2E, C=r64[:, 1, 0] / (-0.5 * LOG2E),
        opacity=r64[:, 1, 1], qthr=r64[:, 1, 2] / (0.5 * LOG2E), id=recb[:, 1, 3].long() & 0xFFFFFFFF,
        rgb=r64[:, 2, :3], rec_extent=r64[:, 2, 3],
        depth=brec[:, 0].double(), rx0=bb[:, 1] & 0xFFFF, rx1=bb[:, 1] >> 16, ry0=bb[:, 2] & 0xFFFF,
        ry1=bb[:, 2] >> 16, keep=bb[:, 3],
        tiles=part("tiles", P, torch.int32).long() & 0xFFFFFFFF, clamped=part("clamped", P, torch.uint8).long(),
        n_big=int(part("aux", 1, torch.int32)[0]), radii=st.radii.detach().cpu().long())


# ---- the fp64 side -----------------------------------------------------------------------------------------------
def oracle_records(means, scales, rots, opac, shs, cam):
    """`O.project` in fp64 of the rasterizer's inputs (means in the frame the rasterizer is given, activated scales and
    opacities, raw quaternions, shs [P, M, 3] or None for precomputed colours), plus what the flags need: view-space
    coordinates `tview` [P, 3] and the SH colour before the clamp `raw_rgb`."""
    d = lambda t: None if t is None else t.detach().cpu().double()
    cam = cam.to(torch.float64)
    means, scales, rots, opac, shs = (d(t) for t in (means, scales, rots, opac, shs))
    with torch.no_grad():
        proj = O.project(means, scales, rots, opac.reshape(-1), shs, cam)
        P = means.shape[0]
        homo = torch.cat([means, torch.ones(P, 1, dtype=torch.float64)], 1)
        proj["tview"] = (homo @ cam.viewmatrix)[:, :3]
        dirs = means - cam.campos[None]
        dirs = dirs / dirs.norm(dim=1, keepdim=True)
        proj["raw_rgb"] = O.eval_sh(cam.sh_degree, shs, dirs) + 0.5
        proj["limx"], proj["limy"] = 1.3 * cam.tanfovx, 1.3 * cam.tanfovy
        proj["W"], proj["H"] = cam.width, cam.height
        proj["mean_norm"] = means.norm(dim=1)
    return proj


def oracle_records_fused(params, pose, cam, deg):
    """oracle_records of the InstantSplat path: raw parameters moved by the camera pose (pre-transform in fp64)."""
    p = {k: v.detach().cpu().double() for k, v in params.items()}
    means, rots = O.pose_pretransform(p["xyz"], p["rotation"], pose.detach().cpu().double())
    shs = torch.cat([p["f_dc"], p["f_rest"]], 1) if p["f_rest"].numel() else p["f_dc"]
    cam = O.Camera(cam.width, cam.height, cam.tanfovx, cam.tanfovy, cam.viewmatrix, cam.projmatrix, cam.campos,
                   cam.bg, deg, cam.scale_modifier)
    return oracle_records(means, torch.exp(p["scaling"]), rots, torch.sigmoid(p["opacity"]), shs, cam)


def cull_threshold(op):
    """gs_math.cuh cull_threshold in fp64: < 0 when the Gaussian can never reach alpha >= 1/255."""
    q = 2.0 * torch.log(torch.clamp(op * 255.0, min=1e-30)) * 1.0005 + 0.01
    return torch.where(op * 255.0 >= 0.999, q, torch.full_like(q, -1.0))


def flags(o):
    """Gaussians whose fp32 result may legitimately differ from the fp64 one, per kind (bool [P] / [P, 3])."""
    tz = o["tview"][:, 2]
    txtz, tytz = o["tview"][:, 0] / tz, o["tview"][:, 1] / tz
    zscale = o["mean_norm"] + o["tview"].norm(dim=1) + 1.0
    out = dict(
        visibility=(tz - NEAR).abs() <= 4e-7 * zscale,
        # the frustum clamp flag: no field of the record depends on it (the clamp is continuous), only the gradient
        clamp_x=((txtz.abs() - o["limx"]).abs() <= 1e-6 * (1.0 + txtz.abs()) * zscale / tz.abs()),
        clamp_y=((tytz.abs() - o["limy"]).abs() <= 1e-6 * (1.0 + tytz.abs()) * zscale / tz.abs()),
        rect=BL._rect_ambiguous(o, torch.arange(tz.numel())),
        clamp_bit=o["raw_rgb"].abs() <= 1e-5 * (1.0 + o["raw_rgb"].abs()),
        cutoff=(o["opacity"] * 255.0 - 0.999).abs() <= 1e-5,
    )
    return out


def check_records(d, o, tol=REC_TOL):
    """Every record of the decoded forward `d` against the fp64 projection `o` (oracle_records).  Raises
    AssertionError; returns a summary: counts of visible Gaussians and of each flag, the largest error of each float
    field (on its scale, below), and of the cull (tiles, rects).

    Float fields, each bounded by `tol` on its own scale: x, y by |x| + W (the NDC-to-pixel map); the conic by its
    largest diagonal entry times the conditioning (a c + b^2) / det of the 2-D covariance it inverts; opacity and depth
    relatively; rgb by 1 + |rgb|; the cull threshold by 1 + |qthr|.  Radius exactly.  The rect (tightened by the
    lossless cull) must lie inside the oracle's rect; tiles == popcount(keep mask) for rects of <= 24 tiles, tiles == 0
    below the opacity cutoff.  Invisible Gaussians: zero record, radius 0, no tiles."""
    P = d["P"]
    f = flags(o)
    vo = o["visible"]
    vk = d["radii"] > 0
    assert torch.equal(d["id"], torch.arange(P)), "record ids"
    bad_vis = (vo != vk) & ~f["visibility"] & ~f["rect"]
    assert not bool(bad_vis.any()), \
        f"{int(bad_vis.sum())} Gaussians visible in one arm only, e.g. {torch.nonzero(bad_vis)[:8].reshape(-1).tolist()}"
    both = vo & vk
    # ---- invisible: nothing but opacity, threshold and id in the record
    inv = ~vk
    for k in ("x", "y", "A", "B", "C", "rgb", "rec_extent", "tiles", "clamped"):
        assert int(d[k][inv].count_nonzero()) == 0, f"invisible Gaussians with a non-zero {k}"
    assert bool((d["qthr"][inv] < 0).all()), "invisible Gaussians with a cull threshold"
    # ---- radius
    rbad = both & (d["radii"] != o["radii"].long()) & ~f["rect"]
    assert not bool(rbad.any()), f"radius differs for {int(rbad.sum())} Gaussians, e.g. " \
        f"{[(int(i), int(d['radii'][i]), int(o['radii'][i])) for i in torch.nonzero(rbad)[:5].reshape(-1)]}"
    # the record's last word is the extent of the fixed-point unit: min(radius, farthest pixel centre), in fp32
    x32, y32 = d["x"].float(), d["y"].float()
    reach = torch.maximum(torch.maximum(x32.abs(), (torch.tensor(float(o["W"] - 1)) - x32).abs()),
                          torch.maximum(y32.abs(), (torch.tensor(float(o["H"] - 1)) - y32).abs()))
    ext = torch.minimum(d["radii"].float(), reach)
    assert torch.equal(d["rec_extent"][vk].float(), ext[vk]), "record extent != min(radius, reach)"
    # ---- float fields
    W, H = o["W"], o["H"]
    a, b, c = o["cov2d"].unbind(-1)
    det = a * c - b * b
    kappa = (a * c + b * b) / det
    conic = o["conic"]
    cs = torch.maximum(conic[:, 0].abs(), conic[:, 2].abs()) * kappa
    err = {}

    def field(name, kern, ora, scale, sel):
        e = ((kern - ora).abs() / scale)[sel]
        m = float(e.max()) if e.numel() else 0.0
        err[name] = m
        if m > tol:
            i = int(torch.nonzero(sel)[int(e.argmax())])
            raise AssertionError(f"record field {name}: error {m:.3g} > {tol} at Gaussian {i} "
                                 f"(kernel {kern.reshape(P, -1)[i].tolist()}, oracle {ora.reshape(P, -1)[i].tolist()})")

    sel = both & ~f["rect"]
    field("x", d["x"], o["xy"][:, 0], o["xy"][:, 0].abs() + W, sel)
    field("y", d["y"], o["xy"][:, 1], o["xy"][:, 1].abs() + H, sel)
    for k, j in (("A", 0), ("B", 1), ("C", 2)):
        field(k, d[k], conic[:, j], cs, sel)
    field("opacity", d["opacity"], o["opacity"], o["opacity"].abs(), torch.ones(P, dtype=torch.bool))
    field("depth", d["depth"], o["depth"], o["depth"].abs(), both)
    cb = f["clamp_bit"]
    rgb_sel = (both[:, None] & ~cb)
    e_rgb = ((d["rgb"] - o["rgb"]).abs() / (1.0 + o["rgb"].abs()))[rgb_sel]
    err["rgb"] = float(e_rgb.max()) if e_rgb.numel() else 0.0
    assert err["rgb"] <= tol, f"record field rgb: error {err['rgb']:.3g} > {tol}"
    bits_o = (o["clamped"].long() * torch.tensor([1, 2, 4])).sum(1)
    cmask = (~cb).long() @ torch.tensor([1, 2, 4])
    assert torch.equal((d["clamped"] & cmask)[both], (bits_o & cmask)[both]), "clamp bits"
    qo = cull_threshold(o["opacity"])
    field("qthr", d["qthr"], qo, 1.0 + qo.abs(), both & ~f["cutoff"])
    # ---- cull: rect inside the oracle's rect, tiles consistent with the keep mask, nothing below the cutoff
    ro = o["rect"]
    inside = (d["rx0"] >= ro[:, 0]) & (d["ry0"] >= ro[:, 1]) & (d["rx1"] <= ro[:, 2]) & (d["ry1"] <= ro[:, 3])
    empty = (d["rx1"] <= d["rx0"]) | (d["ry1"] <= d["ry0"])
    rbad = both & ~(inside | empty) & ~f["rect"]
    assert not bool(rbad.any()), f"{int(rbad.sum())} tightened rects outside the oracle's rect"
    area = ((d["rx1"] - d["rx0"]).clamp(min=0) * (d["ry1"] - d["ry0"]).clamp(min=0))
    assert bool((d["tiles"][vk] <= area[vk]).all()), "more tiles than the rect holds"
    small = vk & (area <= 24)
    pop = torch.tensor([bin(int(m)).count("1") for m in d["keep"][small]], dtype=torch.long)
    assert torch.equal(pop, d["tiles"][small]), "tiles != popcount(keep mask)"
    below = vk & (qo < 0) & ~f["cutoff"]
    assert int(d["tiles"][below].count_nonzero()) == 0, "a Gaussian below the opacity cutoff was given tiles"
    assert bool((d["qthr"][below] < 0).all())
    return dict(P=P, visible=int(vk.sum()), flagged={k: int(v.any(-1).sum() if v.dim() > 1 else v.sum())
                                                     for k, v in f.items()},
                flips=dict(visibility=int((vo != vk).sum()), radius=int((both & (d["radii"] != o["radii"].long())).sum()),
                           clamp_bits=int(((d["clamped"] != bits_o) & both).sum())),
                below_cutoff=int(below.sum()), n_big=d["n_big"], rec_err=err, rec_err_max=max(err.values()))


def zero_rows(grads, rows):
    """Largest |gradient| over the given rows of every per-Gaussian tensor (names -> float)."""
    out = {}
    for k, g in grads.items():
        if g is not None and g.dim() >= 1 and g.shape[0] == rows.shape[0]:
            sub = g.detach()[rows.to(g.device)]
            out[k] = float(sub.abs().max()) if sub.numel() else 0.0
    return out


def camera64(sc, deg, **kw):
    """The fused path's identity-view camera as the oracle takes it, fp64."""
    return O.Camera.instantsplat(sc.width, sc.height, sc.fovx, sc.fovy, sh_degree=deg, dtype=torch.float64, **kw)



