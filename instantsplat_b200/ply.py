"""point_cloud.ply written and read on the GPU (gsb_ply_pack / gsb_ply_unpack, DESIGN.md section 4.23), opt-in with
`--ply_io gpu` on the train, render_views, freeview and pipeline command lines.

The file is byte for byte what scene_io.save_gaussians_ply writes: the header comes from scene_io.gaussian_ply_header
(the same _ply_header the numpy writer uses), and the vertex records are construct_list_of_attributes' layout, raw
little-endian fp32 words packed by one kernel straight from the device tensors.  Records move through at most
CHUNK_BYTES of pinned host memory (and as much device memory) at a time: per chunk, one pack, one device-to-host copy
and one file write; reading is the reverse.

The reader takes the GPU path only for the exact layout save_gaussians_ply writes (SH degree 0-3, with or without
filter_3D: `layout`).  Any other header, property list, format or element set goes to scene_io.load_gaussians_ply, so
--ply_io gpu reads every file the default reads, with the same result.
"""
from __future__ import annotations

import argparse
import os
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch

from . import _lib
from ._lib import GsbPlySegment, check
from .scene_io import gaussian_ply_header, load_gaussians_ply

CHUNK_BYTES = 64 << 20          # pinned host bytes one save or load holds at a time (and device staging bytes)
REST_WIDTHS = (0, 9, 24, 45)    # f_rest_* properties at SH degree 0..3
_HEADER_MAX = 8192              # a 62-property header is about 1.1 KB


def _segments(n_rest: int, has_filter: bool) -> List[Tuple[Optional[str], int, int]]:
    """(tensor name or None for the zero normals, width, inner) in record order; f_rest [P, M-1, 3] is stored
    channel-major (inner 3), an empty f_rest has no segment."""
    segs = [("xyz", 3, 3), (None, 3, 3), ("f_dc", 3, 3), ("f_rest", n_rest, 3), ("opacity", 1, 1),
            ("scaling", 3, 3), ("rotation", 4, 4), ("filter_3D", 1, 1)]
    return [s for s in segs if not (s[0] == "f_rest" and n_rest == 0) and not (s[0] == "filter_3D" and not has_filter)]


def _table(segs, tensors: Dict[str, torch.Tensor], first: int) -> "ctypes.Array":
    """The GsbPlySegment table of records first.. of the tensors."""
    arr = (GsbPlySegment * len(segs))()
    for i, (name, width, inner) in enumerate(segs):
        ptr = None if name is None else tensors[name].data_ptr() + 4 * first * width
        arr[i] = GsbPlySegment(ptr, width, inner)
    return arr


def pack(tensors: Dict[str, torch.Tensor], out: torch.Tensor, first: int = 0, count: Optional[int] = None,
         byte_offset: int = 0) -> None:
    """Records first..first+count of tensors (save_gaussians_ply's inputs by name, contiguous fp32 on one CUDA device:
    xyz, f_dc, f_rest, opacity, scaling, rotation and optionally filter_3D, each with P rows) into out, a uint8 tensor
    on that device or in pinned host memory, from byte byte_offset (a multiple of 4), on the current stream."""
    P, n_rest, has_filter = _check(tensors)
    count = P - first if count is None else count
    segs = _segments(n_rest, has_filter)
    rec = 4 * sum(w for _, w, _ in segs)
    if not (0 <= first and 0 <= count and first + count <= P) or byte_offset % 4 or \
            out.dtype != torch.uint8 or byte_offset + count * rec > out.numel():
        raise ValueError(f"ply.pack: records {first}..{first + count} of {P} do not fit {out.numel()} bytes from "
                         f"offset {byte_offset}")
    check(_lib.lib().gsb_ply_pack(count, len(segs), _table(segs, tensors, first), out.data_ptr() + byte_offset,
                                  _lib.stream_ptr()), "gsb_ply_pack")


def unpack(src: torch.Tensor, tensors: Dict[str, torch.Tensor], first: int = 0, count: Optional[int] = None,
           byte_offset: int = 0) -> None:
    """The reverse of pack: records from src (device or pinned host uint8, from byte byte_offset) into records
    first..first+count of tensors, on the current stream."""
    P, n_rest, has_filter = _check(tensors)
    count = P - first if count is None else count
    segs = _segments(n_rest, has_filter)
    rec = 4 * sum(w for _, w, _ in segs)
    if not (0 <= first and 0 <= count and first + count <= P) or byte_offset % 4 or \
            src.dtype != torch.uint8 or byte_offset + count * rec > src.numel():
        raise ValueError(f"ply.unpack: records {first}..{first + count} of {P} do not fit {src.numel()} bytes from "
                         f"offset {byte_offset}")
    check(_lib.lib().gsb_ply_unpack(count, src.data_ptr() + byte_offset, len(segs), _table(segs, tensors, first),
                                    _lib.stream_ptr()), "gsb_ply_unpack")


def _check(tensors: Dict[str, torch.Tensor]) -> Tuple[int, int, bool]:
    """(P, f_rest width, whether filter_3D is there) of save_gaussians_ply's tensors; ValueError for anything the
    kernels cannot read as they are."""
    P = tensors["xyz"].shape[0]
    n_rest = int(np.prod(tensors["f_rest"].shape[1:]))
    has_filter = tensors.get("filter_3D") is not None
    want = dict(xyz=3, f_dc=3, f_rest=n_rest, opacity=1, scaling=3, rotation=4, **({"filter_3D": 1} if has_filter else {}))
    if n_rest not in REST_WIDTHS:
        raise ValueError(f"ply: f_rest has {n_rest} values per Gaussian; SH degrees 0-3 store {REST_WIDTHS}")
    dev = tensors["xyz"].device
    for name, w in want.items():
        t = tensors[name]
        if t.dtype != torch.float32 or not t.is_contiguous() or t.device != dev or dev.type != "cuda" or \
                t.dim() < 1 or t.shape[0] != P or int(np.prod(t.shape[1:])) != w:
            raise ValueError(f"ply: {name} must be a contiguous fp32 CUDA tensor of {P} x {w} values on {dev}, got "
                             f"{tuple(t.shape)} {t.dtype} on {t.device}")
    return P, n_rest, has_filter


def _pinned(nbytes: int) -> torch.Tensor:
    """The pinned host staging buffer of one save or load (at most CHUNK_BYTES)."""
    return torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)


def save(path: str, tensors: Dict[str, torch.Tensor], chunk_bytes: int = CHUNK_BYTES) -> None:
    """save_gaussians_ply(path, **tensors) from CUDA tensors (pack's): the same file, byte for byte, with the
    records packed on the GPU and copied to the host chunk by chunk, chunk_bytes of pinned memory at most."""
    P, n_rest, has_filter = _check(tensors)
    rec = 4 * sum(w for _, w, _ in _segments(n_rest, has_filter))
    if chunk_bytes < rec:
        raise ValueError(f"ply.save: chunk_bytes {chunk_bytes} is smaller than one {rec}-byte record")
    per = min(chunk_bytes // rec, max(P, 1))
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with torch.cuda.device(tensors["xyz"].device):
        stage = torch.empty(per * rec, dtype=torch.uint8, device=tensors["xyz"].device)
        host = _pinned(per * rec)
        view = memoryview(host.numpy())
        stream = torch.cuda.current_stream()
        with open(path, "wb") as f:
            f.write(gaussian_ply_header(P, n_rest, has_filter))
            for first in range(0, P, per):
                k = min(per, P - first)
                pack(tensors, stage, first, k)
                host[:k * rec].copy_(stage[:k * rec], non_blocking=True)
                stream.synchronize()
                f.write(view[:k * rec])


def layout(path: str) -> Optional[Tuple[int, int, bool, int]]:
    """(P, f_rest width, filter_3D present, header bytes) when path's header is byte for byte the one
    save_gaussians_ply writes for some SH degree 0-3, with or without filter_3D, and the file holds all P records;
    None otherwise (load then uses scene_io.load_gaussians_ply)."""
    with open(path, "rb") as f:
        head = f.read(_HEADER_MAX)
        size = os.fstat(f.fileno()).st_size
    end = head.find(b"\nend_header\n")
    if end < 0:
        return None
    end += len(b"\nend_header\n")
    lines = head[:end].split(b"\n")[:-1]
    if len(lines) < 4 or not lines[2].startswith(b"element vertex "):
        return None
    try:
        P = int(lines[2][len(b"element vertex "):])
    except ValueError:
        return None
    n_props = len(lines) - 4
    for n_rest in REST_WIDTHS:
        for has_filter in (False, True):
            if 17 + n_rest + has_filter != n_props or P < 0:
                continue
            if head[:end] == gaussian_ply_header(P, n_rest, has_filter) and size >= end + 4 * n_props * P:
                return P, n_rest, has_filter, end
    return None


def load(path: str, device="cuda", chunk_bytes: int = CHUNK_BYTES) -> Dict[str, torch.Tensor]:
    """load_gaussians_ply(path) as contiguous fp32 tensors on a CUDA device, bit for bit: the records of a file in
    save_gaussians_ply's exact layout (`layout`) read chunk by chunk into pinned memory (chunk_bytes at most), copied
    to the device and unpacked there; any other file read by load_gaussians_ply and copied to the device."""
    dev = torch.device(device)
    if dev.type != "cuda":
        raise ValueError(f"ply.load: device {device!r}; the GPU reader needs a CUDA device")
    lay = layout(path)
    if lay is None:
        return {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in load_gaussians_ply(path).items()}
    P, n_rest, has_filter, offset = lay
    rec = 4 * sum(w for _, w, _ in _segments(n_rest, has_filter))
    if chunk_bytes < rec:
        raise ValueError(f"ply.load: chunk_bytes {chunk_bytes} is smaller than one {rec}-byte record")
    shapes = dict(xyz=(3,), f_dc=(1, 3), f_rest=(n_rest // 3, 3), opacity=(1,), scaling=(3,), rotation=(4,))
    if has_filter:
        shapes["filter_3D"] = (1,)
    out = {k: torch.empty(P, *s, dtype=torch.float32, device=dev) for k, s in shapes.items()}
    per = min(chunk_bytes // rec, max(P, 1))
    with torch.cuda.device(dev):
        stage = torch.empty(per * rec, dtype=torch.uint8, device=dev)
        host = _pinned(per * rec)
        view = memoryview(host.numpy())
        copied = torch.cuda.Event()
        with open(path, "rb") as f:
            f.seek(offset)
            for first in range(0, P, per):
                k = min(per, P - first)
                copied.synchronize()                   # the previous chunk's copy has left the pinned buffer
                if f.readinto(view[:k * rec]) != k * rec:
                    raise ValueError(f"{path}: truncated while reading its vertex records")
                stage[:k * rec].copy_(host[:k * rec], non_blocking=True)
                copied.record()
                unpack(stage, out, first, k)
        torch.cuda.current_stream().synchronize()
    return out


# ---- the command line ----------------------------------------------------------------------------------------
def add_arg(ap: argparse.ArgumentParser) -> None:
    """--ply_io {numpy,gpu}, left out of the namespace unless it is given, so a command line without it parses to the
    namespace it parsed to before the flag existed; read it with io(args)."""
    ap.add_argument("--ply_io", choices=("numpy", "gpu"), default=argparse.SUPPRESS,
                    help="how point_cloud.ply is written and read: numpy (default) or gpu (records packed and unpacked "
                         "by one kernel; the same bytes)")


def io(args: argparse.Namespace) -> Optional[str]:
    """The --ply_io given, or None."""
    return getattr(args, "ply_io", None)


def argv(value: Optional[str]) -> List[str]:
    """The flag as a stage's command line carries it: [] for None."""
    return [] if value is None else ["--ply_io", value]


def kwargs(args: argparse.Namespace) -> Dict[str, str]:
    """{"ply_io": value} when --ply_io is given, else {}: a loader called without the flag gets what it got before."""
    v = io(args)
    return {} if v is None else {"ply_io": v}
