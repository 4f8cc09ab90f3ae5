"""The lossless culls against the blend's pair rule: populations of screen-space Gaussians where fp32 rounding is at its
worst, the kernels' records of them, and the pair rule in fp64 and fp32 on those records.

All culls (k_preprocess's row form and per-tile test, k_big_rects, the blend's sub-tile test) work on the splat
record in the log2 domain: the binning side takes A' = log2e A / 2, B' = log2e B / 2, C' = log2e C / 2 and
qthr' = log2e qthr / 2; the record holds e0z = -A', e0w = -2 B', e1x = -C' (bit for bit the same numbers, negated and
doubled).  The blend accepts a (Gaussian, pixel) pair when power' = e0z dx^2 + e0w dx dy + e1x dy^2 <= 0 and
min(0.99, o 2^power') >= 1/255 (gs_blend.cu pair_eval).  A cull may drop a tile only if no pixel of it passes that rule.
"""
import ctypes
import math
import os
import subprocess

import numpy as np

F32 = np.float32
F64 = np.float64
LOG2E = F32(1.4426950408889634)            # kLog2e
HALF_LOG2E = F32(0.5) * LOG2E              # 0.5f * kLog2e, folded by the compiler (exact)
ALPHA_MIN = F32(1.0) / F32(255.0)          # kAlphaMin
ALPHA_MAX = F32(0.99)
BLOCK = 16
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_host_lib(out_dir, contract):
    """tests/host_math.cpp as a shared library: contract False as test_host_math.py builds it (no FMA contraction),
    True with FMA contraction, which is what nvcc does to the device code."""
    out = os.path.join(str(out_dir), "libhostmath_%s.so" % ("fma" if contract else "nofma"))
    flags = ["-mfma", "-ffp-contract=fast"] if contract else ["-ffp-contract=off"]
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-x", "c++", *flags,
                           os.path.join(ROOT, "tests", "host_math.cpp"), "-o", out])
    lib = ctypes.CDLL(out)
    fp = ctypes.POINTER(ctypes.c_float)
    ip = ctypes.POINTER(ctypes.c_int)
    lib.host_cull_threshold.argtypes = [ctypes.c_float]
    lib.host_cull_threshold.restype = ctypes.c_float
    lib.host_rect_keep_many.argtypes = [ctypes.c_float] * 6 + [ctypes.c_int, fp, ip]
    lib.host_row_ranges.argtypes = [ctypes.c_float] * 6 + [ctypes.c_int] * 5 + [ip, ip]
    lib.host_row_ranges.restype = ctypes.c_int
    lib.host_tighten_cull_rect.argtypes = [ctypes.c_float] * 6 + [ip]
    return lib


# ---- records ---------------------------------------------------------------------------------------------------------
def record(a, b, c, o, lib):
    """The kernel's record of a Gaussian with 2-D covariance (a, b, c) (fp32, low-pass included) and opacity o:
    project_geometry's conic (1 / det in fp32), scaled into the log2 domain.  None when det == 0 (invisible)."""
    a, b, c, o = F32(a), F32(b), F32(c), F32(o)
    det = a * c - b * b
    if det == 0:
        return None
    inv = F32(1.0) / det
    A, B, C = c * inv, -b * inv, a * inv
    q = F32(lib.host_cull_threshold(o))
    return dict(A=HALF_LOG2E * A, B=HALF_LOG2E * B, C=HALF_LOG2E * C, o=o,
                qthr=HALF_LOG2E * q if q >= 0 else F32(-1.0),
                e0z=-(HALF_LOG2E * A), e0w=(-LOG2E) * B, e1x=-(HALF_LOG2E * C))


def needle_cov(s_long, s_short, theta, lowpass=0.3):
    c, s = math.cos(theta), math.sin(theta)
    l2, s2 = s_long * s_long, s_short * s_short
    return c * c * l2 + s * s * s2 + lowpass, c * s * (l2 - s2), s * s * l2 + c * c * s2 + lowpass


# ---- the pair rule ---------------------------------------------------------------------------------------------------
def pair_rules(x, y, r, px, py):
    """Pixels (px, py) where the pair passes the blend's rule: (fp64 on the record, fp32 in pair_eval's order without
    contraction, fp32 with pair_eval's two multiply-adds fused).  Also returns s = |A'dx^2| + |2B'dx dy| + |C'dy^2|
    and q' = A'dx^2 + 2B'dx dy + C'dy^2 in fp64."""
    x32, y32 = F32(x), F32(y)
    dx, dy = x32 - px.astype(F32), y32 - py.astype(F32)
    e0z, e0w, e1x, o = r["e0z"], r["e0w"], r["e1x"], r["o"]
    p_plain = e0z * dx * dx + (e0w * dx + e1x * dy) * dy
    t = (F64(e0w) * dx.astype(F64) + (e1x * dy).astype(F64)).astype(F32)
    p_fma = ((e0z * dx).astype(F64) * dx.astype(F64) + (t * dy).astype(F64)).astype(F32)
    out = []
    for p in (p_plain, p_fma):
        alpha = np.minimum(ALPHA_MAX, o * np.exp2(p))
        out.append((p <= 0) & (alpha >= ALPHA_MIN))
    dx64, dy64 = F64(x32) - px, F64(y32) - py
    ta, tb, tc = F64(e0z) * dx64 * dx64, F64(e0w) * dx64 * dy64, F64(e1x) * dy64 * dy64
    p64 = ta + tb + tc
    ok64 = (p64 <= 0) & (np.minimum(0.99, F64(o) * np.exp2(np.minimum(p64, 0.0))) >= 1.0 / 255.0)
    return ok64, out[0], out[1], np.abs(ta) + np.abs(tb) + np.abs(tc), -p64


def candidates(x, y, r, W, H, true_conic=None):
    """Every pixel of the W x H frame at which any of pair_rules' three evaluations can pass: the pixels with
    fp64 q' <= 1.001 Q + 0.05 + 1e-6 S_max, Q = log2(255 o) and S_max a bound on s over the frame, padded by two
    pixels per row.  (fp32 evaluation moves q' by at most ~8 2^-24 s, the qthr margins are larger than the rest.)  A
    record whose conic is not positive definite in fp64 takes the positive definite conic `true_conic` (A, B, C, fp64,
    unscaled) with a margin of 1.1 Q + 2."""
    A, B, C = -F64(r["e0z"]), -0.5 * F64(r["e0w"]), -F64(r["e1x"])
    Q = math.log2(max(255.0 * float(r["o"]), 1e-30))
    pad = (1.001, 0.05)
    if not (A > 0 and C > 0 and A * C - B * B > 0):
        A, B, C = (0.5 * float(LOG2E) * v for v in true_conic)
        pad = (1.1, 2.0)
    xs = np.array([0.0, W - 1.0]) - float(F32(x))
    ys = np.array([0.0, H - 1.0]) - float(F32(y))
    smax = 2.0 * (A * (xs * xs).max() + C * (ys * ys).max())
    Qc = pad[0] * max(Q, 0.0) + pad[1] + 1e-6 * smax
    det = A * C - B * B
    hy = math.sqrt(Qc * A / det)
    y0, y1 = max(0, math.floor(float(F32(y)) - hy) - 1), min(H - 1, math.ceil(float(F32(y)) + hy) + 1)
    if y1 < y0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    rows = np.arange(y0, y1 + 1, dtype=F64)
    dy = rows - float(F32(y))
    disc = np.maximum(Qc * A - det * dy * dy, 0.0)
    lo = float(F32(x)) + (-B * dy - np.sqrt(disc)) / A
    hi = float(F32(x)) + (-B * dy + np.sqrt(disc)) / A
    c0 = np.clip(np.floor(lo) - 2, 0, W).astype(np.int64)
    c1 = np.clip(np.ceil(hi) + 3, 0, W).astype(np.int64)
    n = np.maximum(c1 - c0, 0)
    py = np.repeat(rows.astype(np.int64), n)
    start = np.repeat(c0 - (np.cumsum(n) - n), n)
    px = start + np.arange(int(n.sum()), dtype=np.int64)
    return px, py


# ---- the culls -------------------------------------------------------------------------------------------------------
def tile_rects(W, H, bw=BLOCK, bh=BLOCK):
    """Pixel-centre rectangles (x0, y0, x1, y1) of every bw x bh block of the frame, row-major, clipped to the frame."""
    gx, gy = (W + bw - 1) // bw, (H + bh - 1) // bh
    ty, tx = np.divmod(np.arange(gx * gy), gx)
    x0, y0 = tx * bw, ty * bh
    return np.ascontiguousarray(np.stack([x0, y0, np.minimum(x0 + bw - 1, W - 1), np.minimum(y0 + bh - 1, H - 1)], 1),
                                dtype=F32), gx, gy


def rect_keep(lib, x, y, r, rects):
    keep = np.zeros(rects.shape[0], np.int32)
    lib.host_rect_keep_many(F32(x), F32(y), r["A"], r["B"], r["C"], r["qthr"], rects.shape[0],
                            rects.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
                            keep.ctypes.data_as(ctypes.POINTER(ctypes.c_int)))
    return keep.astype(bool)


def tightened_rect(lib, x, y, r, W, H):
    """k_preprocess's tightening of the whole frame's tile rect: (rx0, ry0, rx1, ry1)."""
    rect = np.array([0, 0, (W + BLOCK - 1) // BLOCK, (H + BLOCK - 1) // BLOCK], np.int32)
    lib.host_tighten_cull_rect(F32(x), F32(y), r["A"], r["B"], r["C"], r["qthr"],
                               rect.ctypes.data_as(ctypes.POINTER(ctypes.c_int)))
    return tuple(int(v) for v in rect)


def row_keep(lib, x, y, r, W, H):
    """Kept tiles [gy, gx] of row_keep_range over the whole frame, or None when it falls back to the per-tile test."""
    gx, gy = (W + BLOCK - 1) // BLOCK, (H + BLOCK - 1) // BLOCK
    ta, tb = np.zeros(gy, np.int32), np.zeros(gy, np.int32)
    ok = lib.host_row_ranges(F32(x), F32(y), r["A"], r["B"], r["C"], r["qthr"], H, 0, 0, gx, gy,
                             ta.ctypes.data_as(ctypes.POINTER(ctypes.c_int)),
                             tb.ctypes.data_as(ctypes.POINTER(ctypes.c_int)))
    if not ok:
        return None
    t = np.arange(gx)[None, :]
    return (t >= ta[:, None]) & (t <= tb[:, None])
