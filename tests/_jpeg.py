"""Test helpers for the GPU JPEG decoder (instantsplat_b200/jpeg.py, DESIGN.md 4.24): a seeded corpus written by
Pillow's encoder, the entropy segment's unstuffing restated in numpy, the shared arithmetic of gs_jpeg.cuh built for
the host by g++ (tests/host_jpeg.cpp), a sequential decoder restated in Python and numpy, and a tiny baseline
encoder that writes given coefficient blocks with given tables (4:4:0, and the streams the kernels must flag)."""
from __future__ import annotations

import ctypes
import io
import os
import subprocess
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from instantsplat_b200 import jpeg as J
from instantsplat_b200._lib import GsbJpegFile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ----------------------------------------------------------------------------------------------
# corpus
# ----------------------------------------------------------------------------------------------
def image(h: int, w: int, seed: int) -> np.ndarray:
    """A smooth gradient plus noise and a few hard edges: every coefficient band and both clamps get exercised."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    base = np.stack([128 + 100 * np.sin(x / (3 + w / 7) + c) * np.cos(y / (4 + h / 9) - c) for c in range(3)], -1)
    base += rng.normal(0, 25, base.shape)
    base[(x.astype(int) // 5 + y.astype(int) // 7) % 3 == 0] = [255, 0, 255]
    return np.clip(base, 0, 255).astype(np.uint8)


def pil_jpeg(arr: np.ndarray, **kw) -> bytes:
    from PIL import Image
    buf = io.BytesIO()
    Image.fromarray(arr).save(buf, "JPEG", **kw)
    return buf.getvalue()


def pil_decode(data: bytes) -> np.ndarray:
    from PIL import Image
    with Image.open(io.BytesIO(data)) as im:
        return np.array(im)


# ----------------------------------------------------------------------------------------------
# the unstuffing pass, restated: kept bytes and the first bit of every restart interval
# ----------------------------------------------------------------------------------------------
def unstuff(seg: bytes, n_intervals: int) -> Tuple[np.ndarray, np.ndarray, bool]:
    """(the kept bytes, ibits [n_intervals + 1] with the end last, whether the RSTn count and numbers are right)."""
    d = np.frombuffer(seg, np.uint8).astype(np.int32)
    prev = np.concatenate([[0], d[:-1]])
    nxt = np.concatenate([d[1:], [0]])
    rst = (prev == 0xFF) & ((d & 0xF8) == 0xD0)
    keep = ~(rst | ((prev == 0xFF) & (d == 0)) | ((d == 0xFF) & (nxt != 0)))
    pos = np.cumsum(keep) - keep
    starts = pos[rst] * 8
    nums = d[rst] & 7
    ok = len(starts) == n_intervals - 1 and all(int(v) == i % 8 for i, v in enumerate(nums))
    ibits = np.zeros(n_intervals + 1, np.uint32)
    k = min(len(starts), n_intervals - 1)
    ibits[1:1 + k] = starts[:k]
    ibits[n_intervals] = int(keep.sum()) * 8
    return d[keep].astype(np.uint8), ibits, ok


def n_intervals(p: J.Parsed) -> int:
    mcus = -(-p.width // (8 * p.h)) * -(-p.height // (8 * p.v))
    ri = p.restart_interval or mcus
    return -(-mcus // ri)


def descriptor(p: J.Parsed) -> GsbJpegFile:
    f = GsbJpegFile()
    J._descriptor(p, f, 0, 0)
    return f


# ----------------------------------------------------------------------------------------------
# gs_jpeg.cuh on the host
# ----------------------------------------------------------------------------------------------
_HOST = None


def host_lib(tmpdir: str) -> ctypes.CDLL:
    global _HOST
    if _HOST is None:
        out = os.path.join(tmpdir, "libhostjpeg.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++",
                               os.path.join(ROOT, "tests", "host_jpeg.cpp"), "-o", out])
        L = ctypes.CDLL(out)
        fp, vp, i32 = ctypes.POINTER(GsbJpegFile), ctypes.c_void_p, ctypes.c_int
        L.hj_blocks.restype = ctypes.c_int64
        L.hj_blocks.argtypes = [fp]
        L.hj_decode_seq.argtypes = [fp, vp, vp, i32, vp]
        L.hj_decode_sync.argtypes = [fp, vp, vp, i32, i32, vp, ctypes.POINTER(i32)]
        L.hj_pixels.argtypes = [fp, vp, vp]
        _HOST = L
    return _HOST


def host_coefs(L, data: bytes, subseq_bits: Optional[int] = None):
    """(raster coefficient blocks [blocks, 64] int16 with predicted DC, status bits, sync rounds) of one file from
    the host build: the sequential decode, or the subsequence synchronisation at subseq_bits."""
    p = J.parse(data)
    f = descriptor(p)
    kept, ibits, ok = unstuff(data[p.scan_begin:p.scan_end], n_intervals(p))
    kept = np.concatenate([kept, np.zeros(8, np.uint8)])
    coef = np.zeros((L.hj_blocks(ctypes.byref(f)), 64), np.int16)
    rounds = ctypes.c_int(0)
    if subseq_bits is None:
        st = L.hj_decode_seq(ctypes.byref(f), kept.ctypes.data, ibits.ctypes.data, len(ibits) - 1, coef.ctypes.data)
    else:
        st = L.hj_decode_sync(ctypes.byref(f), kept.ctypes.data, ibits.ctypes.data, len(ibits) - 1, subseq_bits,
                              coef.ctypes.data, ctypes.byref(rounds))
    return coef, st | (0 if ok else 8), rounds.value


def host_decode(L, data: bytes) -> Tuple[np.ndarray, int]:
    """(rgb [H, W, 3], status bits) from the host build's sequential decode and per-pixel stages."""
    p = J.parse(data)
    f = descriptor(p)
    coef, st, _ = host_coefs(L, data)
    rgb = np.zeros((p.height, p.width, 3), np.uint8)
    st |= L.hj_pixels(ctypes.byref(f), coef.ctypes.data, rgb.ctypes.data)
    return rgb, st


# ----------------------------------------------------------------------------------------------
# a tiny baseline encoder: given quantised coefficient blocks, fixed-length Huffman tables
# ----------------------------------------------------------------------------------------------
# DC: 12 symbols of 4 bits (codes 0..11); AC: the 162 baseline run/size symbols of 8 bits (codes 0..161), so the
# 8-bit pattern 11111111 (and everything after it) is no code.
DC_BITS = (0, 0, 0, 12) + (0,) * 12
DC_VALS = bytes(range(12))
AC_VALS = bytes([0x00, 0xF0] + [(r << 4) | s for r in range(16) for s in range(1, 11)])
AC_BITS = (0,) * 7 + (len(AC_VALS),) + (0,) * 8


class _Bits:
    def __init__(self):
        self.out, self.acc, self.n = bytearray(), 0, 0

    def put(self, value: int, n: int) -> None:
        for i in range(n - 1, -1, -1):
            self.acc = (self.acc << 1) | ((value >> i) & 1)
            self.n += 1
            if self.n == 8:
                self.out.append(self.acc)
                if self.acc == 0xFF:
                    self.out.append(0)
                self.acc, self.n = 0, 0

    def flush(self) -> None:                   # pad with 1 bits to the byte boundary
        if self.n:
            self.put((1 << (8 - self.n)) - 1, 8 - self.n)


def _category(v: int) -> int:
    return int(abs(v)).bit_length()


def _put_value(b: _Bits, v: int, s: int) -> None:
    if s:
        b.put(v if v >= 0 else v + (1 << s) - 1, s)


def encode(blocks: Sequence[np.ndarray], width: int, height: int, h: int, v: int, quant: np.ndarray,
           restart: int = 0, rst_numbers: Optional[Sequence[int]] = None, drop_mcus: int = 0, truncate: int = 0,
           bad_code_mcu: int = -1, run_past_63_mcu: int = -1, jfif: bool = True) -> bytes:
    """A baseline JPEG of three components (luma sampling h x v, chroma 1x1) from quantised coefficient blocks
    blocks[c] [by, bx, 64] (natural order; at least the MCU-padded grid), quantisation tables quant [3, 64] (natural
    order), an optional restart interval with the RSTn numbers written (rst_numbers, default 0, 1, ..., 7, 0, ...)
    and the stream faults the decoder must flag: drop_mcus (stop early), truncate (drop the segment's last bytes),
    bad_code_mcu (an AC pattern with no code in that MCU's first block), run_past_63_mcu (a run that takes the
    coefficient index to 64 in that MCU's first block)."""
    from instantsplat_b200.jpeg import ZIGZAG
    mx, my = -(-width // (8 * h)), -(-height // (8 * v))
    mcus = mx * my
    hdr = bytearray(b"\xff\xd8")
    if jfif:
        hdr += b"\xff\xe0\x00\x10JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00"
    for c in range(3):
        hdr += b"\xff\xdb\x00\x43" + bytes([c]) + bytes(int(x) for x in np.asarray(quant[c])[ZIGZAG])
    hdr += b"\xff\xc0\x00\x11\x08" + height.to_bytes(2, "big") + width.to_bytes(2, "big") + b"\x03"
    hdr += bytes([1, (h << 4) | v, 0, 2, 0x11, 1, 3, 0x11, 2])
    for tc, bits, vals in ((0, DC_BITS, DC_VALS), (1, AC_BITS, AC_VALS)):
        body = bytes([tc << 4]) + bytes(bits) + vals
        hdr += b"\xff\xc4" + (len(body) + 2).to_bytes(2, "big") + body
    if restart:
        hdr += b"\xff\xdd\x00\x04" + restart.to_bytes(2, "big")
    hdr += b"\xff\xda\x00\x0c\x03\x01\x00\x02\x00\x03\x00\x00\x3f\x00"
    ac_code = {s: i for i, s in enumerate(AC_VALS)}
    seg = bytearray()
    b = _Bits()
    pred = [0, 0, 0]
    n_rst = 0
    for m in range(mcus - drop_mcus):
        if restart and m and m % restart == 0:
            b.flush()
            seg += b.out
            b = _Bits()
            num = (rst_numbers[n_rst] if rst_numbers is not None and n_rst < len(rst_numbers) else n_rst % 8)
            if num is not None:
                seg += bytes([0xFF, 0xD0 + num])
            n_rst += 1
            pred = [0, 0, 0]
        bxm, bym = m % mx, m // mx
        first = True
        for c in range(3):
            hc, vc = (h, v) if c == 0 else (1, 1)
            for j in range(hc * vc):
                blk = blocks[c][bym * vc + j // hc, bxm * hc + j % hc]
                zz = [int(blk[ZIGZAG[k]]) for k in range(64)]
                diff = zz[0] - pred[c]
                pred[c] = zz[0]
                s = _category(diff)
                b.put(s, 4)
                _put_value(b, diff, s)
                if first and m == bad_code_mcu:
                    b.put(0xFF, 8)
                    b.put(0xFF, 8)
                if first and m == run_past_63_mcu:
                    for _ in range(3):
                        b.put(ac_code[0xF0], 8)          # k = 49
                    b.put(ac_code[0xF1], 8)              # run 15 then a value at k = 64
                    b.put(1, 1)
                    zz = [0] * 64
                first = False
                run = 0
                last = max([k for k in range(1, 64) if zz[k]], default=0)
                for k in range(1, last + 1):
                    if zz[k] == 0:
                        run += 1
                        continue
                    while run > 15:
                        b.put(ac_code[0xF0], 8)
                        run -= 16
                    s = _category(zz[k])
                    b.put(ac_code[(run << 4) | s], 8)
                    _put_value(b, zz[k], s)
                    run = 0
                if last < 63:
                    b.put(ac_code[0x00], 8)
    b.flush()
    seg += b.out
    if truncate:
        seg = seg[:-truncate]
    return bytes(hdr + seg + b"\xff\xd9")


def random_blocks(width: int, height: int, h: int, v: int, seed: int, scale: float = 6.0) -> List[np.ndarray]:
    """Quantised coefficient blocks for encode(): a DC walk and sparse, decaying AC terms."""
    rng = np.random.default_rng(seed)
    mx, my = -(-width // (8 * h)), -(-height // (8 * v))
    out = []
    for c in range(3):
        hc, vc = (h, v) if c == 0 else (1, 1)
        n = (my * vc, mx * hc)
        blk = np.zeros(n + (64,), np.int32)
        blk[..., 0] = np.cumsum(rng.integers(-6, 7, n), axis=1) % 40 - 20
        decay = np.exp(-np.arange(64) / 10.0) * scale
        mask = rng.random(n + (64,)) < 0.3
        blk[..., 1:] = (rng.normal(0, 1, n + (64,)) * decay * mask).astype(np.int32)[..., 1:]
        out.append(blk)
    return out


def flagged_corpus() -> List[Tuple[str, bytes, bool]]:
    """(name, file, whether the kernels must flag it): 4:4:0 files that decode, and one file per flagged stream."""
    q = np.full((3, 64), 4, np.uint16)
    q[:, 0] = 8
    W, H = 53, 37
    out = []
    for h, v in ((1, 2), (2, 2), (1, 1), (2, 1)):
        blocks = random_blocks(W, H, h, v, 10 * h + v)
        out.append((f"clean_{h}{v}", encode(blocks, W, H, h, v, q), False))
        out.append((f"clean_rst_{h}{v}", encode(blocks, W, H, h, v, q, restart=2), False))
    blocks = random_blocks(W, H, 1, 2, 5)
    out.append(("bad_code", encode(blocks, W, H, 1, 2, q, bad_code_mcu=7), True))
    out.append(("run_past_63", encode(blocks, W, H, 1, 2, q, run_past_63_mcu=3), True))
    out.append(("truncated", encode(blocks, W, H, 1, 2, q, truncate=40), True))
    out.append(("mcus_left", encode(blocks, W, H, 1, 2, q, drop_mcus=2), True))
    out.append(("rst_out_of_order", encode(blocks, W, H, 1, 2, q, restart=3, rst_numbers=[0, 2, 1, 3, 4, 5, 6, 7] * 8),
                True))
    out.append(("rst_missing", encode(blocks, W, H, 1, 2, q, restart=3, rst_numbers=[0, None] + list(range(2, 8)) * 8),
                True))
    big = [b.copy() for b in blocks]
    big[0][1, 1, 5] = 1000                              # 1000 * 40 is outside int16
    q40 = q.copy()
    q40[0, 5] = 40
    out.append(("coef_range", encode(big, W, H, 1, 2, q40), True))
    return out


# ----------------------------------------------------------------------------------------------
# a sequential decoder restated in Python and numpy (jdhuff.c, jidctint.c, jdsample.c, jdcolor.c)
# ----------------------------------------------------------------------------------------------
def _idct_pass(x: np.ndarray) -> np.ndarray:
    """The 1-D islow transform of jidctint.c over the last axis of x [..., 8] (int64); returns the 8 sums before
    descaling."""
    i = [x[..., k] for k in range(8)]
    z1 = (i[2] + i[6]) * 4433
    tmp2 = z1 + i[6] * -15137
    tmp3 = z1 + i[2] * 6270
    tmp0 = (i[0] + i[4]) << 13
    tmp1 = (i[0] - i[4]) << 13
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    a0, a1, a2, a3 = i[7], i[5], i[3], i[1]
    z1, z2, z3, z4 = a0 + a3, a1 + a2, a0 + a2, a1 + a3
    z5 = (z3 + z4) * 9633
    a0, a1, a2, a3 = a0 * 2446, a1 * 16819, a2 * 25172, a3 * 12299
    z1, z2, z3, z4 = z1 * -7373, z2 * -20995, z3 * -16069 + z5, z4 * -3196 + z5
    a0, a1, a2, a3 = a0 + z1 + z3, a1 + z2 + z4, a2 + z2 + z3, a3 + z1 + z4
    return np.stack([t10 + a3, t11 + a2, t12 + a1, t13 + a0, t13 - a0, t12 - a1, t11 - a2, t10 - a3], -1)


def py_idct(deq: np.ndarray) -> np.ndarray:
    """jpeg_idct_islow of dequantised blocks [..., 8, 8] (natural order, int) -> uint8 samples [..., 8, 8]."""
    x = deq.astype(np.int64)
    ws = _idct_pass(np.swapaxes(x, -1, -2))                  # columns: [..., col, row]
    ws = (ws + (1 << 10)) >> 11
    ws = ws.astype(np.int32).astype(np.int64)
    out = _idct_pass(np.swapaxes(ws, -1, -2))               # rows: [..., row, col]
    v = ((out + (1 << 17)) >> 18) & 1023
    v = np.where(v >= 512, v - 1024, v) + 128
    return np.clip(v, 0, 255).astype(np.uint8)


def _upsample(pl: np.ndarray, w: int, h: int, H: int, V: int, W_out: int, H_out: int) -> np.ndarray:
    """The chroma plane pl [>=h, >=w] at full resolution [H_out, W_out], as jdsample.c and jdmainct.c make it."""
    c = pl[:h, :w].astype(np.int32)
    if (H, V) == (1, 1):
        return c[:H_out, :W_out]
    if V == 2:
        rows = np.arange(H_out)
        i, odd = rows >> 1, rows & 1
        j = np.clip(np.where(odd == 1, i + 1, i - 1), 0, h - 1)
        near, far = c[i], c[j]
        if H == 1:
            return ((near * 3 + far + np.where(odd == 1, 2, 1)[:, None]) >> 2)[:, :W_out]
        if w <= 2:
            return np.repeat(near, 2, axis=1)[:, :W_out]
        t = near * 3 + far                                          # column sums
        left = np.concatenate([t[:, :1], t[:, :-1]], 1)
        right = np.concatenate([t[:, 1:], t[:, -1:]], 1)
        even = (t * 3 + left + 8) >> 4
        even[:, 0] = (t[:, 0] * 4 + 8) >> 4
        oddc = (t * 3 + right + 7) >> 4
        oddc[:, -1] = (t[:, -1] * 4 + 7) >> 4
        return np.stack([even, oddc], 2).reshape(H_out, 2 * w)[:, :W_out]
    # 2h1v
    if w <= 2:
        return np.repeat(c, 2, axis=1)[:H_out, :W_out]
    left = np.concatenate([c[:, :1], c[:, :-1]], 1)
    right = np.concatenate([c[:, 1:], c[:, -1:]], 1)
    even = (c * 3 + left + 1) >> 2
    even[:, 0] = c[:, 0]
    oddc = (c * 3 + right + 2) >> 2
    oddc[:, -1] = c[:, -1]
    return np.stack([even, oddc], 2).reshape(c.shape[0], 2 * w)[:H_out, :W_out]


def py_decode(data: bytes) -> np.ndarray:
    """np.array(Image.open(...)) of a file in the GPU subset, restated sequentially in Python and numpy."""
    p = J.parse(data)
    H, V = p.h, p.v
    mx, my = -(-p.width // (8 * H)), -(-p.height // (8 * V))
    n_int = n_intervals(p)
    kept, ibits, ok = unstuff(data[p.scan_begin:p.scan_end], n_int)
    assert ok, "restart markers out of sequence"
    bits = np.concatenate([np.unpackbits(kept), np.zeros(64, np.uint8)]).tolist()
    maps = []
    for c in range(3):
        mc = []
        for t in (p.dc[c], p.ac[c]):
            mc.append({(length, code): int(t.huffval[k]) for k, (code, length) in enumerate(t.codes)})
        maps.append(mc)
    coef = [np.zeros((my * (V if c == 0 else 1), mx * (H if c == 0 else 1), 64), np.int64) for c in range(3)]
    ri = p.restart_interval or mx * my
    pos = 0

    def symbol(m):
        nonlocal pos
        code = 0
        for length in range(1, 17):
            code = (code << 1) | bits[pos]
            pos += 1
            if (length, code) in m:
                return m[(length, code)]
        raise ValueError("bad Huffman code")

    def value(s):
        nonlocal pos
        r = 0
        for _ in range(s):
            r = (r << 1) | bits[pos]
            pos += 1
        return r - (1 << s) + 1 if s and r < (1 << (s - 1)) else r

    for m in range(mx * my):
        if m % ri == 0:
            pos = int(ibits[m // ri])
            pred = [0, 0, 0]
        for c in range(3):
            hc, vc = (H, V) if c == 0 else (1, 1)
            for j in range(hc * vc):
                blk = coef[c][(m // mx) * vc + j // hc, (m % mx) * hc + j % hc]
                pred[c] += value(symbol(maps[c][0]))
                blk[0] = np.int16(np.int32(pred[c]))
                k = 1
                while k < 64:
                    rs = symbol(maps[c][1])
                    r, s = rs >> 4, rs & 15
                    if s:
                        k += r
                        assert k <= 63, "run past 63"
                        blk[J.ZIGZAG[k]] = value(s)
                    elif r != 15:
                        break
                    else:
                        k += 15
                    k += 1
    planes = []
    for c in range(3):
        deq = coef[c] * p.quant[c].astype(np.int64)
        assert np.all((deq >= -32768) & (deq <= 32767)), "a dequantised coefficient outside int16"
        s = py_idct(deq.reshape(deq.shape[:2] + (8, 8)))
        planes.append(s.transpose(0, 2, 1, 3).reshape(s.shape[0] * 8, s.shape[1] * 8))
    Y = planes[0][:p.height, :p.width].astype(np.int64)
    cw, ch = -(-p.width // H), -(-p.height // V)
    cb = _upsample(planes[1], cw, ch, H, V, p.width, p.height).astype(np.int64) - 128
    cr = _upsample(planes[2], cw, ch, H, V, p.width, p.height).astype(np.int64) - 128
    r = Y + ((91881 * cr + 32768) >> 16)
    g = Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16)
    b = Y + ((116130 * cb + 32768) >> 16)
    return np.clip(np.stack([r, g, b], -1), 0, 255).astype(np.uint8)
