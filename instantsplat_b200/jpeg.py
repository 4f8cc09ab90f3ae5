"""JPEG source images decoded on the GPU (gsb_jpeg_decode_batch, DESIGN.md section 4.24): the bytes
`np.array(Image.open(path))` gives (Pillow on libjpeg-turbo, default settings: islow IDCT, fancy upsampling, no draft
or scale, no EXIF orientation), opt-in with `--jpeg_decoder gpu` on the train, render_views and pipeline command lines.

The host parses the marker segments only (`parse`): the frame, the quantisation tables, jpeg_make_d_derived_tbl's
derived Huffman tables with its checks, DRI and the one scan.  The entropy-coded bytes go to the device as stored.
`route` names the supported subset: SOF0/SOF1, 8-bit, three components libjpeg reads as YCbCr, chroma 1x1 and luma
1x1, 2x1, 1x2 or 2x2, one scan of all three components (Ss 0, Se 63, Ah Al 0) followed by EOI, every table defined.
Every other file, and every file whose stream the kernels flag (a bad code, a run past 63, bits past a segment's end,
MCUs left over, RSTn out of sequence, a dequantised coefficient outside int16), is decoded by Pillow: that path is not
a second implementation but the only one for those inputs, so a flagged file costs one Pillow decode, never a wrong
pixel.
"""
from __future__ import annotations

import argparse
import ctypes
import functools
import re
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from ._lib import GsbJpegFile as JpegFile, GsbJpegHuff as JpegHuff, check

SUBSEQ_BITS = 1024              # bits per self-synchronising subsequence (a multiple of 8 in 32..2^20)
MIN_SUBSEQ_BITS = 32
SCRATCH_BUDGET = 1 << 30        # device scratch one decode call may take; larger splits go in sub-batches
MAX_FILES = 65535               # files in one decode call

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20,
                   13, 6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52,
                   45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])       # jpeg_natural_order
LOOKAHEAD = _lib.JPEG_LOOKAHEAD
_SEGMENT_END = re.compile(rb"\xff[^\x00\xd0-\xd7]")   # the first marker that is not RSTn ends the entropy segment


class Unsupported(ValueError):
    """A file outside the GPU decoder's subset (the reason is the message); Pillow decodes it."""


class Derived:
    """jpeg_make_d_derived_tbl's tables of one DHT entry: maxcode [18], valoffset [18], huffval [256] and the 9-bit
    lookahead ((length << 8) | symbol, 0 for a longer code), plus the code table (code, length) per symbol index."""

    def __init__(self, bits: Tuple[int, ...], vals: bytes, is_dc: bool):
        if sum(bits) > 256:
            raise Unsupported("a Huffman table with more than 256 symbols")
        huffsize = [l + 1 for l in range(16) for _ in range(bits[l])]
        codes, code, si, p = [], 0, huffsize[0] if huffsize else 0, 0
        while p < len(huffsize):
            while p < len(huffsize) and huffsize[p] == si:
                codes.append(code)
                code += 1
                p += 1
            if code >= (1 << si):
                raise Unsupported("a Huffman table whose codes overflow their length (bad Huffman table)")
            code <<= 1
            si += 1
        self.maxcode = np.full(18, -1, np.int32)
        self.valoffset = np.zeros(18, np.int32)
        p = 0
        for l in range(1, 17):
            if bits[l - 1]:
                self.valoffset[l] = p - codes[p]
                p += bits[l - 1]
                self.maxcode[l] = codes[p - 1]
        self.maxcode[17] = 0xFFFFF
        self.huffval = np.zeros(256, np.uint8)
        self.huffval[:len(vals)] = np.frombuffer(vals, np.uint8)
        if is_dc and any(v > 15 for v in vals):
            raise Unsupported("a DC Huffman table with a symbol above 15 (bad Huffman table)")
        self.look = np.zeros(1 << LOOKAHEAD, np.uint16)
        self.codes = [(c, s) for c, s in zip(codes, huffsize)]
        for i, (c, s) in enumerate(self.codes):
            if s <= LOOKAHEAD:
                lo = c << (LOOKAHEAD - s)
                self.look[lo:lo + (1 << (LOOKAHEAD - s))] = (s << 8) | vals[i]

    def fill(self, h: JpegHuff) -> None:
        ctypes.memmove(h.look, self.look.ctypes.data, self.look.nbytes)
        ctypes.memmove(h.maxcode, self.maxcode.ctypes.data, 72)
        ctypes.memmove(h.valoffset, self.valoffset.ctypes.data, 72)
        ctypes.memmove(h.huffval, self.huffval.ctypes.data, 256)


@functools.lru_cache(maxsize=256)
def derived(bits: Tuple[int, ...], vals: bytes, is_dc: bool) -> Derived:
    return Derived(bits, vals, is_dc)


class Parsed:
    """The marker segments of a supported file: width, height, luma sampling (h, v), restart_interval (MCUs, 0 for
    none), quant [3, 64] (natural order, per component) and the DQT slot each came from (qt_ids), dc / ac (Derived,
    per component), the entropy-coded segment data[scan_begin:scan_end], and component ids."""
    __slots__ = ("width", "height", "h", "v", "restart_interval", "quant", "qt_ids", "dc", "ac", "scan_begin",
                 "scan_end", "ids")


def parse(data: bytes) -> Parsed:
    """The marker segments of a JPEG file; raises Unsupported for anything outside the GPU subset."""
    if data[:2] != b"\xff\xd8":
        raise Unsupported("not a JPEG file")
    n = len(data)
    pos = 2
    qt, dht_dc, dht_ac = {}, {}, {}
    frame = None
    jfif, adobe = False, None
    ri = 0

    def u16(at: int) -> int:
        if at + 2 > n:
            raise Unsupported("truncated marker segment")
        return (data[at] << 8) | data[at + 1]

    while True:
        if pos + 2 > n or data[pos] != 0xFF:
            raise Unsupported("no marker where one is expected")
        while pos < n and data[pos] == 0xFF:
            pos += 1
        if pos >= n:
            raise Unsupported("truncated file")
        m = data[pos]
        pos += 1
        if m in (0xD8, 0xD9) or 0xD0 <= m <= 0xD7 or m == 0x01:
            raise Unsupported(f"marker {m:#04x} before the scan")
        length = u16(pos)
        if length < 2 or pos + length > n:
            raise Unsupported("truncated marker segment")
        seg = data[pos + 2:pos + length]
        pos += length
        if 0xE0 <= m <= 0xEF or m == 0xFE:
            if m == 0xE0 and len(seg) >= 14 and seg[:5] == b"JFIF\x00":
                jfif = True
            elif m == 0xEE and len(seg) >= 12 and seg[:5] == b"Adobe":
                adobe = seg[11]
            elif m == 0xE2 and seg[:4] == b"MPF\x00":
                raise Unsupported("an MPO file (Pillow opens its first frame)")
        elif m == 0xDB:
            i = 0
            while i < len(seg):
                pq, tq = seg[i] >> 4, seg[i] & 15
                if tq > 3 or pq > 1:
                    raise Unsupported("a bad quantisation table")
                size = 64 * (pq + 1)
                if i + 1 + size > len(seg):
                    raise Unsupported("a truncated quantisation table")
                raw = np.frombuffer(seg, ">u2" if pq else np.uint8, 64, i + 1).astype(np.uint16)
                nat = np.zeros(64, np.uint16)
                nat[ZIGZAG] = raw
                qt[tq] = nat
                i += 1 + size
        elif m == 0xC4:
            i = 0
            while i < len(seg):
                if i + 17 > len(seg):
                    raise Unsupported("a truncated Huffman table")
                tc, th = seg[i] >> 4, seg[i] & 15
                bits = tuple(seg[i + 1:i + 17])
                count = sum(bits)
                if tc > 1 or th > 3 or count > 256 or i + 17 + count > len(seg):
                    raise Unsupported("a bad Huffman table")
                (dht_dc if tc == 0 else dht_ac)[th] = (bits, bytes(seg[i + 17:i + 17 + count]))
                i += 17 + count
        elif m == 0xDD:
            if len(seg) != 2:
                raise Unsupported("a bad DRI segment")
            ri = (seg[0] << 8) | seg[1]
        elif m in (0xC0, 0xC1):
            if frame is not None:
                raise Unsupported("two frame headers")
            if len(seg) < 6:
                raise Unsupported("a truncated frame header")
            prec, height, width, nf = seg[0], (seg[1] << 8) | seg[2], (seg[3] << 8) | seg[4], seg[5]
            if prec != 8:
                raise Unsupported(f"{prec}-bit samples")
            if nf != 3:
                raise Unsupported(f"{nf} components")
            if len(seg) != 6 + 3 * nf:
                raise Unsupported("a bad frame header")
            if height == 0 or width == 0:
                raise Unsupported("a frame height set by DNL, or an empty frame")
            comps = [(seg[6 + 3 * c], seg[7 + 3 * c] >> 4, seg[7 + 3 * c] & 15, seg[8 + 3 * c]) for c in range(3)]
            frame = (width, height, comps)
        elif 0xC0 <= m <= 0xCF:
            raise Unsupported(f"SOF{m - 0xC0} (progressive, lossless or arithmetic-coded)")
        elif m == 0xDA:
            break
        else:
            raise Unsupported(f"marker {m:#04x}")
    if frame is None:
        raise Unsupported("a scan before the frame header")
    width, height, comps = frame
    ids = tuple(c[0] for c in comps)
    if not jfif:
        if adobe is not None and adobe != 1:
            raise Unsupported(f"Adobe transform {adobe} (not YCbCr)")
        if adobe is None and ids == (82, 71, 66):
            raise Unsupported("RGB component ids")
    (_, h, v, _), (_, h1, v1, _), (_, h2, v2, _) = comps
    if (h, v) not in ((1, 1), (2, 1), (1, 2), (2, 2)) or (h1, v1, h2, v2) != (1, 1, 1, 1):
        raise Unsupported(f"sampling {[(c[1], c[2]) for c in comps]}")
    if len(seg) < 1 or seg[0] != 3 or len(seg) != 1 + 2 * 3 + 3:
        raise Unsupported("a scan that does not interleave all three components")
    tabs = [(seg[1 + 2 * c], seg[2 + 2 * c] >> 4, seg[2 + 2 * c] & 15) for c in range(3)]
    if tuple(t[0] for t in tabs) != ids:
        raise Unsupported("scan components not in frame order")
    if tuple(seg[7:10]) != (0, 63, 0):
        raise Unsupported("a scan other than Ss 0, Se 63, Ah Al 0")
    p = Parsed()
    p.width, p.height, p.h, p.v, p.restart_interval, p.ids = width, height, h, v, ri, ids
    try:
        p.qt_ids = tuple(c[3] for c in comps)
        p.quant = np.stack([qt[c[3]] for c in comps])
        p.dc = [derived(*dht_dc[t[1]], True) for t in tabs]
        p.ac = [derived(*dht_ac[t[2]], False) for t in tabs]
    except KeyError:
        raise Unsupported("a table the scan uses is not defined") from None
    p.scan_begin = pos
    mt = _SEGMENT_END.search(data, pos)
    if mt is None:
        raise Unsupported("no marker after the scan (truncated file)")
    if data[mt.start() + 1] != 0xD9:
        raise Unsupported("a marker other than EOI after the scan (DNL, more scans or fill bytes)")
    p.scan_end = mt.start()
    return p


def route(data: bytes) -> str:
    """"gpu" for a file in the GPU decoder's subset, "pil" otherwise (before any stream check)."""
    try:
        parse(data)
        return "gpu"
    except Unsupported:
        return "pil"


def _descriptor(p: Parsed, out: JpegFile, data_offset: int, out_offset: int) -> None:
    out.width, out.height, out.h, out.v = p.width, p.height, p.h, p.v
    out.restart_interval = p.restart_interval
    out.data_offset, out.data_bytes, out.out_offset = data_offset, p.scan_end - p.scan_begin, out_offset
    q = np.ascontiguousarray(p.quant, np.uint16)
    ctypes.memmove(out.quant, q.ctypes.data, q.nbytes)
    for c in range(3):
        p.dc[c].fill(out.dc[c])
        p.ac[c].fill(out.ac[c])


def _pil(path: str) -> np.ndarray:
    from PIL import Image
    with Image.open(path) as im:
        return np.array(im)


def decode_u8(paths: Sequence[str], device, subseq_bits: int = SUBSEQ_BITS, budget: int = SCRATCH_BUDGET,
              return_routes: bool = False):
    """np.array(Image.open(path)) of every path, as uint8 tensors on the CUDA device: [H, W, 3] for the files the GPU
    decodes, Pillow's array for the others (whatever its shape).  Files are decoded in as few calls as the scratch
    budget allows, each with one status read; files outside the subset or flagged by the kernels are decoded by
    Pillow, whose exception, if it raises, propagates.  When every image has the same size the tensors are views of
    one [N, H, W, 3] buffer (`stack` returns it).  return_routes: also the list of "gpu" / "pil" per file."""
    dev = torch.device(device)
    if dev.type != "cuda":
        raise ValueError(f"jpeg.decode_u8: device {device!r}: the decoder runs on a CUDA device only")
    if subseq_bits < MIN_SUBSEQ_BITS or subseq_bits % 8 or subseq_bits > (1 << 20):
        raise ValueError(f"jpeg.decode_u8: subseq_bits {subseq_bits} is not a multiple of 8 in 32..2^20")
    datas, parsed = [], []
    for path in paths:
        with open(path, "rb") as f:
            data = f.read()
        try:
            p = parse(data)
        except Unsupported:
            p = None
        datas.append(data)
        parsed.append(p)
    out: List[Optional[torch.Tensor]] = [None] * len(paths)
    routes = ["gpu" if p is not None else "pil" for p in parsed]
    gpu = [i for i, p in enumerate(parsed) if p is not None]
    sizes = {(p.height, p.width) for p in parsed if p is not None}
    with torch.cuda.device(dev):
        base = None
        if len(gpu) == len(paths) and len(sizes) == 1:
            Hs, Ws = sizes.pop()
            base = torch.empty(len(paths), Hs, Ws, 3, dtype=torch.uint8, device=dev)
        for batch in _batches(gpu, parsed, subseq_bits, budget):
            images, st = _decode_batch(batch, datas, parsed, dev, subseq_bits, base)
            for i, im, s in zip(batch, images, st):
                if s:
                    routes[i] = "pil"
                else:
                    out[i] = im
        for i, r in enumerate(routes):
            if r == "pil":
                arr = torch.from_numpy(_pil(paths[i])).to(dev)
                if base is not None and tuple(arr.shape) == tuple(base.shape[1:]):
                    base[i].copy_(arr)
                    arr = base[i]
                out[i] = arr
    return (out, routes) if return_routes else out


def stack(images: List[torch.Tensor]) -> torch.Tensor:
    """[N, H, W, 3] of decode_u8's images (no copy when they are views of its one buffer)."""
    if images and images[0]._base is not None and all(im._base is images[0]._base for im in images) \
            and images[0]._base.dim() == 4 and images[0]._base.shape[0] == len(images) \
            and all(im.data_ptr() == images[0]._base[i].data_ptr() for i, im in enumerate(images)):
        return images[0]._base
    return torch.stack(images)


def _table(batch: List[int], parsed) -> Tuple["ctypes.Array", int]:
    """The descriptors of the files batch, their entropy segments packed in order: (table, total bytes)."""
    files = (JpegFile * max(len(batch), 1))()
    off = 0
    for k, i in enumerate(batch):
        p = parsed[i]
        _descriptor(p, files[k], off, 0)
        off += p.scan_end - p.scan_begin
    return files, off


def _batches(gpu: List[int], parsed, subseq_bits: int, budget: int):
    """Splits the files in order so that each call's scratch stays under budget (a file larger than the budget goes
    alone)."""
    L = _lib.lib()
    cur: List[int] = []
    for i in gpu:
        trial = cur + [i]
        files, _ = _table(trial, parsed)
        if cur and (len(trial) > MAX_FILES or L.gsb_jpeg_scratch_bytes(len(trial), files, subseq_bits) > budget):
            yield cur
            cur = [i]
        else:
            cur = trial
    if cur:
        yield cur


def _decode_batch(batch: List[int], datas, parsed, dev, subseq_bits: int, base=None):
    """One gsb_jpeg_decode_batch call for the files batch (indices into datas / parsed): (their images, [H, W, 3]
    views of base when given, else of one new buffer; their status words)."""
    L = _lib.lib()
    files, total = _table(batch, parsed)
    stream = np.empty(max(total, 1), np.uint8)
    o = 0
    for i in batch:
        p = parsed[i]
        m = p.scan_end - p.scan_begin
        stream[o:o + m] = np.frombuffer(datas[i], np.uint8, m, p.scan_begin)
        o += m
    shapes = [(parsed[i].height, parsed[i].width, 3) for i in batch]
    if base is not None:
        target, offs = base, [i * base[0].numel() for i in batch]
    else:
        sizes = [h * w * 3 for h, w, _ in shapes]
        target = torch.empty(max(sum(sizes), 1), dtype=torch.uint8, device=dev)
        offs = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64).tolist()
    for k in range(len(batch)):
        files[k].out_offset = int(offs[k])
    d_stream = torch.from_numpy(stream).to(dev)
    nb = L.gsb_jpeg_scratch_bytes(len(batch), files, subseq_bits)
    scratch = torch.empty(nb + 256, dtype=torch.uint8, device=dev)
    status = torch.empty(len(batch), dtype=torch.int32, device=dev)
    check(L.gsb_jpeg_decode_batch(len(batch), files, d_stream.data_ptr(), subseq_bits,
                                  (scratch.data_ptr() + 255) & ~255, nb, target.data_ptr(), status.data_ptr(),
                                  _lib.stream_ptr()), "gsb_jpeg_decode_batch")
    flat = target.view(-1)
    images = [flat[o:o + h * w * 3].view(h, w, 3) for o, (h, w, _) in zip(offs, shapes)]
    return images, status.cpu().tolist()


def status_of(paths: Sequence[str], device, subseq_bits: int = SUBSEQ_BITS) -> List[Optional[int]]:
    """The kernels' status word of each file, all in one call (None for a file outside the subset): 0 decoded
    exactly, else GSB_JPEG_* bits.  For the tests and the cost script."""
    datas, parsed = [], []
    for path in paths:
        with open(path, "rb") as f:
            datas.append(f.read())
        try:
            parsed.append(parse(datas[-1]))
        except Unsupported:
            parsed.append(None)
    gpu = [i for i, p in enumerate(parsed) if p is not None]
    res: List[Optional[int]] = [None] * len(paths)
    if gpu:
        dev = torch.device(device)
        with torch.cuda.device(dev):
            _, st = _decode_batch(gpu, datas, parsed, dev, subseq_bits)
        for i, s in zip(gpu, st):
            res[i] = s
    return res


def add_arg(ap: argparse.ArgumentParser) -> None:
    """--jpeg_decoder {pil,gpu}, left out of the namespace unless it is given, so a command line without it parses to
    the namespace it parsed to before the flag existed; read it with decoder(args)."""
    ap.add_argument("--jpeg_decoder", choices=("pil", "gpu"), default=argparse.SUPPRESS,
                    help="how JPEG source images are decoded: pil (default) or gpu (Pillow's pixels byte for byte; "
                         "files outside the GPU subset and flagged streams go to Pillow)")


def decoder(args: argparse.Namespace) -> Optional[str]:
    """The --jpeg_decoder given, or None."""
    return getattr(args, "jpeg_decoder", None)


def requested(args: argparse.Namespace) -> bool:
    """Whether --jpeg_decoder gpu was given."""
    return decoder(args) == "gpu"


def argv(value: Optional[str]) -> List[str]:
    """The flag as a stage's command line carries it: [] for None."""
    return [] if value is None else ["--jpeg_decoder", value]
