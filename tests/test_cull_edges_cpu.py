"""The lossless culls (gs_math.cuh rect_may_contribute and row_keep_range, compiled for the host) against the blend's
pair rule, on the populations where fp32 rounding is at its worst.

Every tile (16 x 16) and every blend sub-tile (8 x 4 and 8 x 8) holding a pixel at which the pair rule passes -- in fp64
on the record, or in fp32 in pair_eval's order with or without its multiply-adds fused (tests/_cull.py) -- must be kept
by each cull; the predicates are built with and without FMA contraction.  Each population asserts that it reached its
regime, and that the culls still cull there (a "fix" that keeps everything fails).  No GPU.
"""
import math

import numpy as np
import pytest

import _cull as CU

F32 = np.float32
W_HD, H_HD = 1920, 1080
W_EDGE, H_EDGE = 30 * 16 - 5, 17 * 16 - 9        # partial last tile row and column
SUB_BLOCKS = ((8, 4), (8, 8))                    # the blend's sub-tile rectangles: v1 8x4, v2 8x8 (two 8x4 halves)
NEAR_ANGLES = (0.0, math.pi / 4, math.pi / 2, 3 * math.pi / 4)


@pytest.fixture(scope="module", params=[False, True], ids=["nofma", "fma"])
def lib(request, tmp_path_factory):
    return CU.build_host_lib(tmp_path_factory.mktemp("cull"), request.param)


def _angle(rng, i):
    """Uniform angles, and every third one within 1e-3 rad of an axis or a diagonal."""
    if i % 3:
        return rng.uniform(0.0, math.pi)
    return NEAR_ANGLES[(i // 3) % 4] + rng.uniform(-1e-3, 1e-3)


# ---- populations: (x, y, (a, b, c) 2-D covariance with low-pass, opacity) ------------------------------------------
def long_needles(rng, n):
    out = []
    for i in range(n):
        sl = math.exp(rng.uniform(math.log(50), math.log(5000)))
        ratio = math.exp(rng.uniform(math.log(1e-4), math.log(1e-1)))
        out.append((rng.uniform(0, W_HD), rng.uniform(0, H_HD), CU.needle_cov(sl, sl * ratio, _angle(rng, i)),
                    rng.uniform(0.05, 1.0)))
    return out


def huge_radii(rng, n):
    """Near-plane Gaussians, 3-sigma radius 1e3 - 1e5 px, the centre outside the frame so that the alpha >= 1/255
    ellipse reaches at most ~40 px into it (some miss it by a little)."""
    out = []
    for i in range(n):
        rad = math.exp(rng.uniform(math.log(1e3), math.log(1e5)))
        sl = rad / 3.0
        ss = sl * rng.uniform(0.05, 1.0)
        a, b, c = CU.needle_cov(sl, ss, rng.uniform(0, math.pi))
        op = rng.uniform(0.02, 1.0)
        Q = 2.0 * math.log(255.0 * op)
        side = i % 4
        depth = rng.uniform(-4.0, 40.0)
        if side < 2:                                     # left / right: x extent of the ellipse sqrt(Q a)
            hx = math.sqrt(Q * a)
            x = -hx + depth if side == 0 else W_EDGE - 1 + hx - depth
            y = rng.uniform(0, H_EDGE)
        else:
            hy = math.sqrt(Q * c)
            y = -hy + depth if side == 2 else H_EDGE - 1 + hy - depth
            x = rng.uniform(0, W_EDGE)
        out.append((x, y, (a, b, c), op))
    return out


def threshold_opacity(rng, n):
    """255 o in 0.999 - 1.02: qthr is a few hundredths, the ellipse a few pixels at most."""
    out = []
    for i in range(n):
        sl = math.exp(rng.uniform(math.log(0.3), math.log(300)))
        ss = sl * math.exp(rng.uniform(math.log(1e-3), 0.0))
        out.append((rng.uniform(0, W_EDGE), rng.uniform(0, H_EDGE), CU.needle_cov(sl, ss, _angle(rng, i)),
                    rng.uniform(0.999, 1.02) / 255.0))
    return out


def frame_edge(rng, n):
    """Centres just outside the frame (up to 3 sigma), next to the partial last tile row or column or the origin."""
    out = []
    for i in range(n):
        sl = math.exp(rng.uniform(math.log(1), math.log(200)))
        ss = sl * math.exp(rng.uniform(math.log(1e-3), 0.0))
        off = rng.uniform(0.01, 3.0) * sl
        side = i % 4
        x = (W_EDGE - 1 + off) if side == 0 else (-off if side == 1 else rng.uniform(0, W_EDGE))
        y = (H_EDGE - 1 + off) if side == 2 else (-off if side == 3 else rng.uniform(0, H_EDGE))
        out.append((x, y, CU.needle_cov(sl, ss, _angle(rng, i)), rng.uniform(0.05, 1.0)))
    return out


def degenerate(rng, n):
    """Needles so thin and long that the record's conic has det <= 0 in fp32 (A'C' - B'^2 rounds to <= 0): the row
    form's setup refuses them and k_preprocess falls back to the per-tile test."""
    out = []
    while len(out) < n:
        sl = math.exp(rng.uniform(math.log(2000), math.log(40000)))
        th = NEAR_ANGLES[1 + 2 * rng.integers(0, 2)] + rng.uniform(-0.2, 0.2)
        out.append((rng.uniform(0, W_HD), rng.uniform(0, H_HD), CU.needle_cov(sl, rng.uniform(0.0, 0.5), th),
                    rng.uniform(0.05, 1.0)))
    return out


POPULATIONS = {
    # name: (generator, count, frame)
    "long_needles": (long_needles, 300, (W_HD, H_HD)),
    "huge_radii": (huge_radii, 160, (W_EDGE, H_EDGE)),
    "threshold_opacity": (threshold_opacity, 600, (W_EDGE, H_EDGE)),
    "frame_edge": (frame_edge, 600, (W_EDGE, H_EDGE)),
    "degenerate": (degenerate, 200, (W_HD, H_HD)),
}


def run_population(lib, name, seed=0):
    gen, n, (W, H) = POPULATIONS[name]
    rng = np.random.default_rng(seed + sum(map(ord, name)))
    tiles, gx, gy = CU.tile_rects(W, H)
    subs = [(bw, bh) + CU.tile_rects(W, H, bw, bh) for bw, bh in SUB_BLOCKS]
    st = dict(gaussians=0, pairs=0, must_tiles=0, rect_outside=[], rect_dropped=[], row_dropped=[], row_fallback=0, rect_culled=0,
              row_culled=0, sub_must=0, sub_dropped=[], sub_culled=0, max_cancel=0.0, min_qthr=math.inf,
              centre_outside=0, partial_edge_tiles=0, det_le0=0, max_rect_tiles=0)
    for x, y, (a, b, c), op in gen(rng, n):
        r = CU.record(a, b, c, op, lib)
        if r is None or r["qthr"] < 0:
            continue
        st["gaussians"] += 1
        st["min_qthr"] = min(st["min_qthr"], float(r["qthr"]))
        st["det_le0"] += int(r["A"] * r["C"] - r["B"] * r["B"] <= 0)
        st["centre_outside"] += int(not (0 <= F32(x) <= W - 1 and 0 <= F32(y) <= H - 1))
        px, py = CU.candidates(x, y, r, W, H, true_conic=_true_conic(a, b, c))
        ok64, ok32, okf, s, q = CU.pair_rules(x, y, r, px, py)
        must = ok64 | ok32 | okf
        px, py, s, q = px[must], py[must], s[must], q[must]
        st["pairs"] += int(must.sum())
        if px.size:
            st["max_cancel"] = max(st["max_cancel"], float((s / np.maximum(np.abs(q), 1.0)).max()))
        # 16x16 tiles: the per-tile test (coop / big-rect walks, the fallback of the mask) and the row form
        need = np.zeros(gx * gy, bool)
        need[(py // 16) * gx + px // 16] = True
        st["must_tiles"] += int(need.sum())
        st["partial_edge_tiles"] += int(need.reshape(gy, gx)[-1].sum() + need.reshape(gy, gx)[:, -1].sum())
        st["max_rect_tiles"] = max(st["max_rect_tiles"], int(need.sum()))
        rx0, ry0, rx1, ry1 = CU.tightened_rect(lib, x, y, r, W, H)
        ty_, tx_ = np.divmod(np.nonzero(need)[0], gx)
        out = (tx_ < rx0) | (tx_ >= rx1) | (ty_ < ry0) | (ty_ >= ry1)
        st["rect_outside"] += [(x, y, a, b, c, op, int(t)) for t in np.nonzero(need)[0][out][:2]]
        keep = CU.rect_keep(lib, x, y, r, tiles)
        st["rect_culled"] += int((~keep).sum())
        lost = np.nonzero(need & ~keep)[0]
        st["rect_dropped"] += [(x, y, a, b, c, op, int(t)) for t in lost[:2]]
        rk = CU.row_keep(lib, x, y, r, W, H)
        if rk is None:
            st["row_fallback"] += 1
        else:
            rk = rk.reshape(-1)
            st["row_culled"] += int((~rk).sum())
            lost = np.nonzero(need & ~rk)[0]
            st["row_dropped"] += [(x, y, a, b, c, op, int(t)) for t in lost[:2]]
        # the blend's sub-tile test
        for bw, bh, rects, sgx, sgy in subs:
            sneed = np.zeros(sgx * sgy, bool)
            sneed[(py // bh) * sgx + px // bw] = True
            cand = np.nonzero(need[(np.arange(sgx * sgy) // sgx * bh // 16) * gx
                                   + (np.arange(sgx * sgy) % sgx * bw // 16)])[0]
            skeep = CU.rect_keep(lib, x, y, r, np.ascontiguousarray(rects[cand]))
            st["sub_must"] += int(sneed.sum())
            st["sub_culled"] += int((~skeep).sum())
            lost = cand[sneed[cand] & ~skeep]
            st["sub_dropped"] += [(x, y, a, b, c, op, bw, bh, int(t)) for t in lost[:2]]
    return st


def _true_conic(a, b, c):
    det = a * c - b * b
    return c / det, -b / det, a / det


@pytest.mark.parametrize("name", list(POPULATIONS))
def test_culls_keep_every_contributing_tile(lib, name):
    st = run_population(lib, name)
    # each population reaches its regime
    assert st["gaussians"] >= (100 if name in ("huge_radii", "degenerate") else 0.9 * POPULATIONS[name][1]), st
    assert st["must_tiles"] > 100 and st["sub_must"] > 400, st
    if name == "long_needles":
        assert st["max_cancel"] > 1e5, st["max_cancel"]          # terms of q' 1e5 x q' itself at a contributing pixel
        assert st["max_rect_tiles"] > 128                         # the needle spans a big rect's worth of tiles
    if name == "huge_radii":
        assert st["centre_outside"] == st["gaussians"] and st["gaussians"] >= 100
    if name == "threshold_opacity":
        assert st["min_qthr"] < 0.02, st["min_qthr"]
    if name == "frame_edge":
        assert st["centre_outside"] > 0.9 * st["gaussians"] and st["partial_edge_tiles"] > 50, st
    if name == "degenerate":
        assert st["det_le0"] >= 20 and st["row_fallback"] >= st["det_le0"], st
    # lossless: nothing that holds a contributing pixel is dropped, by any of the culls
    assert not st["rect_outside"], (len(st["rect_outside"]), st["rect_outside"][:4])
    assert not st["rect_dropped"], (len(st["rect_dropped"]), st["rect_dropped"][:4])
    assert not st["row_dropped"], (len(st["row_dropped"]), st["row_dropped"][:4])
    assert not st["sub_dropped"], (len(st["sub_dropped"]), st["sub_dropped"][:4])
    # and the culls still cull (the whole frame's tiles are offered, so nearly all are rejected)
    assert st["rect_culled"] > 0.5 * st["gaussians"] * (POPULATIONS[name][2][0] // 16), st
    assert st["sub_culled"] > 0.05 * st["sub_must"], st
