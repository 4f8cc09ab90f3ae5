"""Read the per-tile lists a forward left in its binning buffer and check them exactly.

The binning buffer is laid out by `bin_view` in instantsplat_b200/csrc/gs_internal.cuh (BinView), with the capacity
the forward was given (`_State.R`) as `cap`:

    pairs   [cap]       u64  (depth bits << 32 | Gaussian id), per-tile segments (sorted in place for lists > 8192)
    ids     [cap + 8]   u32  Gaussian ids, per tile in (depth bits, id) order -- what the blend kernels walk
    ranges  [tiles]     u32 x 2  [start, end) of each tile's list

each part starting on a 256-byte boundary.  `bin_layout` restates that; a CPU test pins it to `gsb_binning_bytes`.
The status words (`gv.status`, enum kSt* in the same header) are read from the device copy, after the sort has
updated the overflow and huge-tile words.

The checks are integer checks on the GPU (configs[4] has ~46 M instances), so they cost a few sorts, not a loop.
"""
import numpy as np
import torch

from instantsplat_b200.frame import ST_HUGE_TILES, ST_MAX_LIST, ST_NHUGE, ST_NLARGE, ST_OVERFLOW, ST_R, u32

BLOCK = 16
ALIGN = 256
SMALL_LIST, LARGE_LIST = 2048, 8192      # kSmallList / kLargeList: the per-tile sort's size classes
SKEW = 24                                # kSkew: a bucket longer than this sends a tile to the bitonic fallback


def align_up(v, a=ALIGN):
    return (v + a - 1) // a * a


def bin_layout(cap, W, H):
    """Byte offset and length of each BinView array, and the total (= gsb_binning_bytes(cap, W, H))."""
    rp = max(int(cap), 1)
    ntiles = ((W + BLOCK - 1) // BLOCK) * ((H + BLOCK - 1) // BLOCK)
    out, off = {}, 0
    for name, nbytes in (("pairs", rp * 8), ("ids", (rp + 8) * 4), ("ranges", ntiles * 8)):
        out[name] = (off, nbytes)
        off += align_up(nbytes)
    out["total"] = off
    return out


def status_words(st):
    """The forward's device status words (uint32, as Python ints)."""
    return [u32(x) for x in st.status.cpu().tolist()]


def decode(st):
    """Tile lists of a forward (`_State`: `img.grad_fn.st` after `rasterize_fused`) as device tensors."""
    H, W = st.cam.height, st.cam.width
    gx, gy = (W + BLOCK - 1) // BLOCK, (H + BLOCK - 1) // BLOCK
    cap = int(st.R)
    lay = bin_layout(cap, W, H)
    assert lay["total"] <= st.binning.numel(), (lay, st.binning.numel())
    b = st.binning

    def part(name, n, dt):
        off = lay[name][0]
        return b[off:off + n * torch.empty(0, dtype=dt).element_size()].view(dt)

    return dict(pairs=part("pairs", cap, torch.int64), ids=part("ids", cap, torch.int32).long() & 0xFFFFFFFF,
                ranges=part("ranges", 2 * gx * gy, torch.int32).long().reshape(gx * gy, 2) & 0xFFFFFFFF,
                status=status_words(st), P=int(st.P), W=W, H=H, gx=gx, gy=gy, cap=cap)


def check_lists(d):
    """Exact checks on every tile of a decoded forward.  Raises AssertionError; returns a summary:
    ranges contiguous from 0 and summing to R (no truncated list), status words consistent with the list lengths,
    every id < P and unique within its tile, and ids[s:e] == low 32 bits of sort(pairs[s:e]) for every tile
    (the kernel's own keys, so the check holds whichever sort path ran and whether it sorted in place)."""
    s = d["status"]
    rng = d["ranges"]
    R = s[ST_R]
    assert R <= d["cap"], f"binning overflow (R {R}, capacity {d['cap']})"
    # a render phase that overflowed its estimated capacity raised the overflow word and was repeated with an exact
    # buffer (rasterizer._forward): the lists are then those of the second pass, and the huge tiles were sorted twice
    passes = 2 if s[ST_OVERFLOW] else 1
    lens = rng[:, 1] - rng[:, 0]
    assert bool((lens >= 0).all()), "negative tile range"
    starts = torch.cumsum(lens, 0) - lens
    assert torch.equal(rng[:, 0], starts), "tile ranges are not contiguous"
    assert int(lens.sum()) == R, (int(lens.sum()), R)
    nmax = int(lens.max()) if lens.numel() else 0
    n_large = int(((lens > SMALL_LIST) & (lens <= LARGE_LIST)).sum())
    n_huge = int((lens > LARGE_LIST).sum())
    assert s[ST_MAX_LIST] == nmax, (s, nmax)
    assert s[ST_NLARGE] == n_large and s[ST_NHUGE] == n_huge and s[ST_HUGE_TILES] == passes * n_huge, \
        (s, n_large, n_huge)
    if R:
        pairs, ids = d["pairs"][:R], d["ids"][:R]
        tile = torch.repeat_interleave(torch.arange(lens.numel(), device=lens.device), lens)
        o1 = torch.sort(pairs, stable=True)[1]                 # segmented sort: by key, then stably by tile
        t1 = tile[o1]
        o2 = torch.sort(t1, stable=True)[1]
        seg = pairs[o1][o2]
        del o1, o2, t1
        assert int(ids.max()) < d["P"], "id out of range"
        bad = (seg & 0xFFFFFFFF) != ids
        nbad = int(bad.sum())
        if nbad:
            first = int(torch.nonzero(bad)[0])
            raise AssertionError(f"{nbad} list entries out of (depth, id) order; first in tile {int(tile[first])} "
                                 f"(list length {int(lens[tile[first]])}) at position {first - int(rng[tile[first], 0])}")
        dup = (seg[1:] == seg[:-1]) & (tile[1:] == tile[:-1])
        assert not bool(dup.any()), "duplicate id in a tile list"
        assert bool(((seg >> 32) > 0).all()), "non-positive depth key"
    return dict(R=R, max_list=nmax, n_large=n_large, n_huge=n_huge,
                n_tiles_nonempty=int((lens > 0).sum()))


def max_bucket(keys, cap):
    """Largest bucket of the kernel's one-pass bucket histogram over a tile's keys (tile_sort_one, gs_bin.cu, fp32
    arithmetic restated): > SKEW means the tile took the bitonic fallback."""
    dep = (np.asarray(keys, dtype=np.int64) >> 32).astype(np.uint32)
    dmin, dmax = dep.min(), dep.max()
    scale = np.float32(cap) / (np.float32(dmax - dmin) + np.float32(1.0))
    b = np.minimum(np.uint32(cap - 1), ((dep - dmin).astype(np.float32) * scale).astype(np.uint32))
    return int(np.bincount(b, minlength=cap).max())


# ---- comparison with the oracle's rect lists ---------------------------------------------------------------------
def oracle_proj(sc, view, deg):
    """Oracle projection of scene `sc` in `view` (fp32, the precision whose rounding the kernels share)."""
    from oracle import gs_oracle as O
    with torch.no_grad():
        cam = O.Camera.instantsplat(sc.width, sc.height, sc.fovx, sc.fovy, sh_degree=deg)
        means, rots = O.pose_pretransform(sc.params["xyz"], sc.params["rotation"], sc.poses[view])
        shs = torch.cat([sc.params["f_dc"], sc.params["f_rest"]], dim=1)
        return O.project(means, torch.exp(sc.params["scaling"]), rots, torch.sigmoid(sc.params["opacity"]), shs, cam)


def _rect_ambiguous(proj, g):
    """Gaussians whose tile rect is within rounding of a tile boundary (or whose radius is within rounding of an
    integer): an fp32 implementation may legitimately put them in one more or one fewer tile row / column."""
    from oracle import gs_oracle as O
    xy = proj["xy"][g].double()
    r = proj["radii"][g].double()
    cov = proj["cov2d"][g].double()
    a, b, c = cov[:, 0], cov[:, 1], cov[:, 2]
    mid = 0.5 * (a + c)
    lam = mid + torch.sqrt(torch.clamp(mid * mid - (a * c - b * b), min=0.1))
    rr = 3.0 * torch.sqrt(lam)
    near = (rr - torch.round(rr)).abs() < 1e-4 * rr
    for v in ((xy[:, 0] - r) / O.BLOCK, (xy[:, 1] - r) / O.BLOCK, (xy[:, 0] + r + O.BLOCK - 1) / O.BLOCK,
              (xy[:, 1] + r + O.BLOCK - 1) / O.BLOCK):
        near |= (v - torch.round(v)).abs() < 1e-5 * (1 + v.abs())
    return near


def _depth_bits(proj):
    return proj["depth"].detach().to(torch.float32).view(torch.int32).to(torch.int64)


def compare_with_oracle(d, proj, cull, exact=True):
    """Each tile's list against the oracle's `build_tile_lists` rect list.

    cull False: the lists must be equal element for element.  cull True: each list must be an order-preserving
    subsequence of the oracle's, and each dropped pair must have alpha < 1/255 at every pixel centre of the tile
    (per the oracle), unless it is within rounding of that threshold.  exact False (general scenes): a mismatch is
    allowed where the oracle shows why an fp32 implementation may differ -- a rect bound within rounding of a tile
    boundary, or an order swap of two Gaussians whose depths are at most 1 ulp apart; such mismatches are counted.
    Returns dict(tiles, mismatched_tiles, explained, dropped)."""
    from oracle import gs_oracle as O
    gids, oranges = O.build_tile_lists(proj)
    gids = gids.numpy()
    dbits = _depth_bits(proj).numpy()
    ids_all = d["ids"].cpu().numpy()
    rng = d["ranges"].cpu().numpy()
    T = rng.shape[0]
    assert oranges.shape[0] == T
    xy, con, op = proj["xy"].detach().double(), proj["conic"].detach().double(), proj["opacity"].detach().double()
    gx = d["gx"]
    out = dict(tiles=0, mismatched_tiles=0, explained=0, dropped=0)
    for t in range(T):
        c = ids_all[rng[t, 0]:rng[t, 1]]
        o = gids[int(oranges[t, 0]):int(oranges[t, 1])]
        if len(c) == 0 and len(o) == 0:
            continue
        out["tiles"] += 1
        if not cull and len(c) == len(o) and np.array_equal(c, o):
            continue
        pos = {int(g): i for i, g in enumerate(o)}
        where = np.array([pos.get(int(g), -1) for g in c], dtype=np.int64)
        extra = c[where < 0]                                  # in the kernel's list, not in the oracle's
        kept = where[where >= 0]
        inv = np.nonzero(np.diff(kept) <= 0)[0]               # order violations against the oracle's order
        dropped = np.setdiff1d(o, c)
        problems = len(extra) + len(inv) + (0 if cull else len(dropped))
        if problems:
            out["mismatched_tiles"] += 1
            msg = f"tile {t}: {len(extra)} extra ids, {len(inv)} order swaps, {len(dropped)} dropped (cull {cull})"
            assert not exact, msg
            unexplained = 0
            if len(extra):
                unexplained += int((~_rect_ambiguous(proj, torch.from_numpy(extra))).sum())
            for k in inv:
                a, b = o[kept[k]], o[kept[k + 1]]
                if abs(int(dbits[a]) - int(dbits[b])) > 1:
                    unexplained += 1
            if not cull and len(dropped):
                unexplained += int((~_rect_ambiguous(proj, torch.from_numpy(dropped))).sum())
            assert unexplained == 0, msg + f", {unexplained} not explained by rounding"
            out["explained"] += problems
        if cull and len(dropped):
            out["dropped"] += len(dropped)
            ty, tx = divmod(t, gx)
            x0, y0 = tx * O.BLOCK, ty * O.BLOCK
            x1, y1 = min(x0 + O.BLOCK, d["W"]), min(y0 + O.BLOCK, d["H"])
            ys, xs = torch.meshgrid(torch.arange(y0, y1, dtype=torch.float64),
                                    torch.arange(x0, x1, dtype=torch.float64), indexing="ij")
            g = torch.from_numpy(dropped)
            dx = xy[g, 0:1] - xs.reshape(1, -1)
            dy = xy[g, 1:2] - ys.reshape(1, -1)
            power = -0.5 * (con[g, 0:1] * dx * dx + con[g, 2:3] * dy * dy) - con[g, 1:2] * dx * dy
            alpha = op[g, None] * torch.exp(power.clamp(max=0.0))
            contributes = (power <= 0) & (alpha >= O.ALPHA_MIN)
            ambiguous = ((alpha * 255.0 - 1.0).abs() < 5e-4) | ((power > -1e-7) & (power != 0))
            lost = contributes & ~ambiguous
            assert not bool(lost.any()), \
                f"tile {t}: the cull dropped {int(lost.any(1).sum())} Gaussians that contribute to a pixel"
    return out
