"""PNG files of 8-bit RGB frames encoded on the GPU (gsb_png_encode_batch, DESIGN.md section 4.19): the opt-in
`--png_encoder gpu` of the freeview, render_views and pipeline command lines.

The kernels filter every scanline as Pillow does (so the files inflate to the very scanlines save_image's files
hold) and deflate 32 KiB segments of a frame in parallel, so the zlib stream differs from Pillow's: the files decode to
the same pixels but are not byte-identical to save_image's.  A frame's bytes depend on its pixels alone.  Only the
compressed bytes cross to the host, which frames them into chunks (IHDR as Pillow writes it, one IDAT, IEND, a CRC-32
each) and writes the files.
"""
from __future__ import annotations

import os
import struct
import zlib
from collections import deque
from concurrent.futures import ThreadPoolExecutor
from typing import Iterable, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from ._lib import check

SIGNATURE = b"\x89PNG\r\n\x1a\n"
MAX_BATCH = 8                 # frames per gsb_png_encode_batch call of encode_host: bounds the device scratch
_IDAT_MAX = (1 << 31) - 1     # a chunk's length field is 31 bits


def bound(H: int, W: int) -> int:
    """gsb_png_bound: the largest zlib stream an H x W frame can need."""
    return int(_lib.lib().gsb_png_bound(int(H), int(W)))


def chunk(kind: bytes, data: bytes) -> bytes:
    """One PNG chunk: big-endian length, type, data, CRC-32 of type and data."""
    return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", zlib.crc32(data, zlib.crc32(kind)))


def ihdr(H: int, W: int) -> bytes:
    """The IHDR data Pillow writes for an 8-bit RGB image: no interlace."""
    return struct.pack(">IIBBBBB", int(W), int(H), 8, 2, 0, 0, 0)


def png_file(H: int, W: int, stream: bytes) -> bytes:
    """A complete PNG file of an 8-bit RGB H x W image around its zlib stream."""
    idat = [chunk(b"IDAT", stream[i:i + _IDAT_MAX]) for i in range(0, max(len(stream), 1), _IDAT_MAX)]
    return b"".join([SIGNATURE, chunk(b"IHDR", ihdr(H, W))] + idat + [chunk(b"IEND", b"")])


def encode(frames: torch.Tensor) -> List[bytes]:
    """frames: contiguous uint8 CUDA [V, H, W, 3] (freeview.quantise's output) -> V complete PNG files, encoded on the
    current stream.  Only each frame's used bytes are copied to the host."""
    if not isinstance(frames, torch.Tensor) or frames.dim() != 4 or frames.shape[3] != 3 \
            or frames.dtype != torch.uint8 or not frames.is_cuda or not frames.is_contiguous():
        raise ValueError(f"png.encode: expected a contiguous uint8 CUDA [V, H, W, 3] tensor, got "
                         f"{tuple(getattr(frames, 'shape', ()))} {getattr(frames, 'dtype', type(frames))}")
    V, H, W, _ = frames.shape
    if V == 0:
        return []
    L = _lib.lib()
    nb = L.gsb_png_bound(H, W)
    if nb == 0:
        raise ValueError(f"png.encode: a {H} x {W} frame is too large to encode")
    dev = frames.device
    with torch.cuda.device(dev):
        scratch = torch.empty(L.gsb_png_scratch_bytes(V, H, W), dtype=torch.uint8, device=dev)
        out = torch.empty(V, nb, dtype=torch.uint8, device=dev)
        sizes = torch.empty(V, dtype=torch.int64, device=dev)
        check(L.gsb_png_encode_batch(V, H, W, frames.data_ptr(), scratch.data_ptr(), scratch.numel(), out.data_ptr(),
                                     sizes.data_ptr(), _lib.stream_ptr()), "gsb_png_encode_batch")
        n = sizes.cpu().tolist()
        return [png_file(H, W, out[v, :n[v]].cpu().numpy().tobytes()) for v in range(V)]


def encode_host(chunk_u8: np.ndarray, device=None) -> List[bytes]:
    """encode for a host uint8 [B, H, W, 3] array: uploaded and encoded MAX_BATCH frames at a time on device (None:
    the current CUDA device)."""
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    out = []
    for i in range(0, chunk_u8.shape[0], MAX_BATCH):
        out += encode(torch.from_numpy(np.ascontiguousarray(chunk_u8[i:i + MAX_BATCH])).to(dev))
    return out


def write_file(data: bytes, path: str) -> None:
    with open(path, "wb") as f:
        f.write(data)


def write_pngs(frames: Iterable[Tuple[int, np.ndarray]], folder: str, workers: Optional[int] = None,
               names: Optional[Sequence[str]] = None) -> int:
    """freeview.write_pngs' files, names and arguments, encoded on the GPU: each host chunk is uploaded and encoded on
    the current device, and the files are written on a pool of `workers` threads (None: up to 8), at most 4 x workers
    files waiting.  Returns the number of files."""
    os.makedirs(folder, exist_ok=True)
    workers = min(8, os.cpu_count() or 1) if workers is None else int(workers)
    if workers < 1:
        raise ValueError("write_pngs: workers must be >= 1")
    count, pending = 0, deque()
    with ThreadPoolExecutor(max_workers=workers) as pool:
        for first, frames_u8 in frames:
            for i, data in enumerate(encode_host(frames_u8)):
                name = f"{first + i:05d}.png" if names is None else names[first + i]
                pending.append(pool.submit(write_file, data, os.path.join(folder, name)))
                count += 1
                while len(pending) > 4 * workers:
                    pending.popleft().result()
        for f in pending:
            f.result()
    return count
