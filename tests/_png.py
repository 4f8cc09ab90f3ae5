"""Reference restatements for the PNG tests: Pillow's scanline filter choice in numpy, PNG chunk parsing, and the
Adler-32 combine that gsb_png_encode_batch's pack kernel computes."""
import struct
import zlib

import numpy as np

FILTER_TYPES = (0, 1, 2, 4)       # the order Pillow's ZipEncode tries them in; Average (3) is never tried


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    return np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))


def filter_rows(img: np.ndarray):
    """Pillow's adaptive filter of an 8-bit RGB image [H, W, 3]: (filtered stream of H (3W + 1) bytes, row types).
    Per row, the type of None, Sub, Up, Paeth whose filtered bytes have the least sum of |int8| wins, the first on a
    tie; row 0 filters against a zero row and the first pixel's left neighbours are zero (3 bytes per pixel)."""
    H, W, C = img.shape
    a = img.reshape(H, W * C).astype(np.int32)
    prev = np.zeros(W * C, np.int32)
    rows, types = [], []
    for y in range(H):
        r = a[y]
        left = np.concatenate([np.zeros(C, np.int32), r[:-C]])
        ul = np.concatenate([np.zeros(C, np.int32), prev[:-C]])
        cands = [r, r - left, r - prev, r - _paeth(left, prev, ul)]
        cands = [(c & 255).astype(np.uint8) for c in cands]
        cost = [int(np.minimum(c, 256 - c.astype(np.int32)).sum()) for c in cands]
        k = int(np.argmin(cost))                     # argmin takes the first of equal minima
        types.append(FILTER_TYPES[k])
        rows.append(bytes([FILTER_TYPES[k]]) + cands[k].tobytes())
        prev = r
    return b"".join(rows), np.array(types, np.uint8)


def chunks(data: bytes):
    """[(type, payload)] of a PNG file; asserts the signature and every chunk's CRC-32."""
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    out, i = [], 8
    while i < len(data):
        (n,) = struct.unpack(">I", data[i:i + 4])
        kind, payload = data[i + 4:i + 8], data[i + 8:i + 8 + n]
        (crc,) = struct.unpack(">I", data[i + 8 + n:i + 12 + n])
        assert crc == zlib.crc32(payload, zlib.crc32(kind)), kind
        out.append((kind, payload))
        i += 12 + n
    assert i == len(data)
    return out


def idat(data: bytes) -> bytes:
    """The concatenated IDAT data of a PNG file (its zlib stream)."""
    return b"".join(p for k, p in chunks(data) if k == b"IDAT")


ADLER_MOD = 65521
SEGMENT = 32768


def adler_parts(data: bytes, seg: int = SEGMENT):
    """Per segment of seg bytes, the Adler-32 sums from (0, 0): a = sum x_j, b = sum (n - j) x_j, mod 65521."""
    out = []
    for s in range(0, len(data), seg):
        x = np.frombuffer(data[s:s + seg], np.uint8).astype(np.int64)
        n = len(x)
        out.append((int(x.sum()) % ADLER_MOD, int(((n - np.arange(n)) * x).sum()) % ADLER_MOD))
    return out


def adler_combine(parts, N: int, seg: int = SEGMENT) -> int:
    """Adler-32 of the whole stream from the segments' sums: byte i weighs N - i, its weight inside its segment plus N
    minus the segment's end."""
    s1, s2 = 1, N % ADLER_MOD
    for r, (a, b) in enumerate(parts):
        end = min(N, (r + 1) * seg)
        s1 += a
        s2 += b + (N - end) % ADLER_MOD * a
    return ((s2 % ADLER_MOD) << 16) | (s1 % ADLER_MOD)
