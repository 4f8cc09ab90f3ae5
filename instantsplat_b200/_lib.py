"""ctypes binding of libgsb200.so (C ABI: include/gsb200.h).

The product path has NO fallback: if the CUDA library is missing or fails, every entry point
raises.  (The CPU oracle under oracle/ is test infrastructure and is never imported from here.)
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libgsb200.so")
CSRC = os.path.join(_HERE, "csrc")

c_float_p = ctypes.POINTER(ctypes.c_float)


class GsbCamera(ctypes.Structure):
    _fields_ = [("width", ctypes.c_int32), ("height", ctypes.c_int32),
                ("tanfovx", ctypes.c_float), ("tanfovy", ctypes.c_float),
                ("scale_modifier", ctypes.c_float), ("sh_degree", ctypes.c_int32),
                ("sh_coeffs", ctypes.c_int32), ("exact_cull", ctypes.c_int32),
                ("bg", ctypes.c_void_p), ("viewmatrix", ctypes.c_void_p),
                ("projmatrix", ctypes.c_void_p), ("campos", ctypes.c_void_p)]


class GsbGaussians(ctypes.Structure):
    _fields_ = [("P", ctypes.c_int32), ("sh_packed", ctypes.c_int32), ("raw_params", ctypes.c_int32),
                ("reserved", ctypes.c_int32),
                ("means3D", ctypes.c_void_p), ("scales", ctypes.c_void_p), ("rotations", ctypes.c_void_p),
                ("opacities", ctypes.c_void_p), ("sh_dc", ctypes.c_void_p), ("sh_rest", ctypes.c_void_p),
                ("colors_precomp", ctypes.c_void_p), ("cov3D_precomp", ctypes.c_void_p),
                ("pose", ctypes.c_void_p)]


class GsbGrads(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in (
        "dL_dmeans3D", "dL_dmeans2D", "dL_dscales", "dL_drotations", "dL_dopacities", "dL_dsh_dc",
        "dL_dsh_rest", "dL_dcolors", "dL_dcov3D", "dL_dpose")]


class GsbFilter(ctypes.Structure):
    _fields_ = [("kernel_size", ctypes.c_float), ("flags", ctypes.c_int32), ("filter3D", ctypes.c_void_p)]


FILTER_MIP2D = 1


class GsbDensifyStats(ctypes.Structure):
    _fields_ = [("radii", ctypes.c_void_p), ("grad_accum", ctypes.c_void_p), ("denom", ctypes.c_void_p),
                ("max_radii2D", ctypes.c_void_p)]


class GsbAdamTensor(ctypes.Structure):
    _fields_ = [("param", ctypes.c_void_p), ("grad", ctypes.c_void_p), ("exp_avg", ctypes.c_void_p),
                ("exp_avg_sq", ctypes.c_void_p), ("per_point_lr", ctypes.c_void_p),
                ("numel", ctypes.c_int64), ("row_len", ctypes.c_int32), ("grad_scale", ctypes.c_float),
                ("step_size", ctypes.c_double), ("beta1", ctypes.c_double), ("beta2", ctypes.c_double),
                ("eps", ctypes.c_double), ("weight_decay", ctypes.c_double)]


class GsbPlySegment(ctypes.Structure):
    _fields_ = [("data", ctypes.c_void_p), ("width", ctypes.c_int32), ("inner", ctypes.c_int32)]


PLY_MAX_SEGMENTS = 8
JPEG_LOOKAHEAD = 9


class GsbJpegHuff(ctypes.Structure):
    _fields_ = [("look", ctypes.c_uint16 * (1 << JPEG_LOOKAHEAD)), ("maxcode", ctypes.c_int32 * 18),
                ("valoffset", ctypes.c_int32 * 18), ("huffval", ctypes.c_uint8 * 256)]


class GsbJpegFile(ctypes.Structure):
    _fields_ = [("width", ctypes.c_int32), ("height", ctypes.c_int32), ("h", ctypes.c_int32), ("v", ctypes.c_int32),
                ("restart_interval", ctypes.c_int32), ("reserved", ctypes.c_int32),
                ("data_offset", ctypes.c_int64), ("data_bytes", ctypes.c_int64), ("out_offset", ctypes.c_int64),
                ("quant", (ctypes.c_uint16 * 64) * 3), ("dc", GsbJpegHuff * 3), ("ac", GsbJpegHuff * 3)]


class GsbShardPiece(ctypes.Structure):
    _fields_ = [("begin", ctypes.c_int64), ("end", ctypes.c_int64), ("seg_begin", ctypes.c_int64),
                ("per_point_lr", ctypes.c_void_p), ("row_len", ctypes.c_int32), ("flag_index", ctypes.c_int32),
                ("step_size", ctypes.c_double), ("beta1", ctypes.c_double), ("beta2", ctypes.c_double),
                ("eps", ctypes.c_double)]


ADAM_MAX_TENSORS = 8
EXPORTS = ("gsb_geom_bytes", "gsb_binning_bytes", "gsb_image_bytes", "gsb_preprocess", "gsb_render",
           "gsb_backward", "gsb_mark_visible", "gsb_ssim_forward", "gsb_ssim_backward",
           "gsb_loss_forward", "gsb_loss_backward", "gsb_adam_step", "gsb_last_error",
           "gsb_abi_version", "gsb_profile_enable", "gsb_profile_collect", "gsb_launch_count", "gsb_set_option", "gsb_adam_gate",
           "gsb_ipc_alloc", "gsb_ipc_open", "gsb_ipc_close", "gsb_ipc_free", "gsb_fused_rs_adam_ag",
           "gsb_knn_scratch_bytes", "gsb_knn_mean_dist2", "gsb_status_device", "gsb_adam_step_gated", "gsb_blend_stats", "gsb_l1_mask_fwd_bwd", "gsb_track_step", "gsb_peer_signal_bytes", "gsb_peer_barrier", "gsb_peer_exchange", "gsb_adam_step_ex",
           "gsb_preprocess_ex", "gsb_backward_ex", "gsb_mip_filter3d", "gsb_backward_stats",
           "gsb_geom_bytes_batch", "gsb_binning_bytes_batch", "gsb_image_bytes_batch", "gsb_status_device_batch",
           "gsb_preprocess_batch", "gsb_render_batch", "gsb_backward_pose_batch", "gsb_l1_mask_fwd_bwd_batch",
           "gsb_track_step_batch", "gsb_backward_batch", "gsb_loss_forward_batch", "gsb_loss_backward_batch",
           "gsb_backward_batch_stats", "gsb_image_metrics_scratch_bytes", "gsb_image_metrics_batch",
           "gsb_frames_u8_batch", "gsb_lpips_scratch_bytes", "gsb_lpips_prepare", "gsb_lpips_conv3x3_relu",
           "gsb_lpips_maxpool2", "gsb_lpips_head", "gsb_render_batch_bg", "gsb_backward_batch_stats_bg",
           "gsb_png_bound", "gsb_png_scratch_bytes", "gsb_png_encode_batch", "gsb_resample_u8_batch",
           "gsb_ply_pack", "gsb_ply_unpack", "gsb_jpeg_scratch_bytes", "gsb_jpeg_decode_batch")
KERNEL_IDS = ("preprocess", "sort_depth", "scan", "duplicate", "sort_tile", "gather", "blend_fwd", "blend_bwd",
              "preprocess_bwd", "loss_fwd", "loss_bwd", "adam")

_lib = None


class GsbError(RuntimeError):
    pass


def build(verbose: bool = False) -> str:
    """Compile libgsb200.so for sm_90a with nvcc (cross-compiles without a GPU)."""
    out = subprocess.run(["make", "-C", CSRC, "-j4"], capture_output=True, text=True)
    if out.returncode != 0:
        raise GsbError("building libgsb200.so failed:\n" + out.stdout + out.stderr)
    if verbose:
        print(out.stdout)
    return LIB_PATH


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise GsbError(f"{LIB_PATH} not found -- run `python -c 'import __graft_entry__ as g; g.build()'` "
                       "(there is no CPU fallback)")
    L = ctypes.CDLL(LIB_PATH)
    vp, i32, i64, sz = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_size_t
    L.gsb_geom_bytes.restype = sz
    L.gsb_geom_bytes.argtypes = [i32]
    L.gsb_binning_bytes.restype = sz
    L.gsb_binning_bytes.argtypes = [i64, i32, i32]
    L.gsb_image_bytes.restype = sz
    L.gsb_image_bytes.argtypes = [i32, i32]
    L.gsb_preprocess.argtypes = [ctypes.POINTER(GsbCamera), ctypes.POINTER(GsbGaussians), vp, sz, vp, vp, vp]
    L.gsb_preprocess_ex.argtypes = [ctypes.POINTER(GsbCamera), ctypes.POINTER(GsbGaussians), ctypes.POINTER(GsbFilter),
                                    vp, sz, vp, vp, vp]
    L.gsb_backward_ex.argtypes = [ctypes.POINTER(GsbCamera), ctypes.POINTER(GsbGaussians), ctypes.POINTER(GsbFilter),
                                  vp, vp, i64, vp, vp, ctypes.POINTER(GsbGrads), vp]
    L.gsb_backward_stats.argtypes = [ctypes.POINTER(GsbCamera), ctypes.POINTER(GsbGaussians), ctypes.POINTER(GsbFilter),
                                     ctypes.POINTER(GsbDensifyStats), vp, vp, i64, vp, vp, ctypes.POINTER(GsbGrads), vp]
    L.gsb_mip_filter3d.argtypes = [i32, vp, i32, vp, i32, i32, ctypes.c_float, ctypes.c_float, vp, vp]
    L.gsb_render.argtypes = [ctypes.POINTER(GsbCamera), i32, vp, vp, sz, i64, vp, vp, vp, vp]
    L.gsb_blend_stats.argtypes = [ctypes.POINTER(GsbCamera), i32, vp, vp, i64, vp, vp, vp, vp, vp]
    L.gsb_blend_stats.restype = ctypes.c_int
    fl = ctypes.c_float
    L.gsb_l1_mask_fwd_bwd.argtypes = [i32, i32, i32, vp, vp, fl, vp, vp, vp]
    L.gsb_l1_mask_fwd_bwd.restype = ctypes.c_int
    L.gsb_track_step.argtypes = [vp, vp, vp, vp, vp, vp, vp, i32, fl, fl, fl, fl, fl, fl, vp]
    L.gsb_track_step.restype = ctypes.c_int
    L.gsb_peer_signal_bytes.restype = sz
    L.gsb_peer_barrier.argtypes = [i32, i32, ctypes.POINTER(vp), ctypes.c_uint32, i32, vp]
    L.gsb_peer_barrier.restype = ctypes.c_int
    L.gsb_peer_exchange.argtypes = [i32, i32, ctypes.POINTER(vp), ctypes.c_uint32, vp, vp, vp, i32, vp]
    L.gsb_peer_exchange.restype = ctypes.c_int
    L.gsb_adam_step_ex.argtypes = [i32, ctypes.POINTER(GsbAdamTensor), vp, vp, vp, vp]
    L.gsb_adam_step_ex.restype = ctypes.c_int
    L.gsb_status_device.argtypes = [vp, i32]
    L.gsb_status_device.restype = vp
    L.gsb_geom_bytes_batch.restype = sz
    L.gsb_geom_bytes_batch.argtypes = [i32, i32, i32, i32]
    L.gsb_binning_bytes_batch.restype = sz
    L.gsb_binning_bytes_batch.argtypes = [i64, i32, i32, i32]
    L.gsb_image_bytes_batch.restype = sz
    L.gsb_image_bytes_batch.argtypes = [i32, i32, i32]
    L.gsb_status_device_batch.argtypes = [vp, i32, i32]
    L.gsb_status_device_batch.restype = vp
    L.gsb_preprocess_batch.argtypes = [ctypes.POINTER(GsbCamera), ctypes.POINTER(GsbGaussians),
                                       ctypes.POINTER(GsbFilter), i32, vp, vp, sz, vp, vp, vp]
    L.gsb_render_batch.argtypes = [ctypes.POINTER(GsbCamera), i32, i32, vp, vp, sz, i64, vp, vp, vp, vp]
    L.gsb_backward_pose_batch.argtypes = [ctypes.POINTER(GsbCamera), ctypes.POINTER(GsbGaussians),
                                          ctypes.POINTER(GsbFilter), i32, vp, vp, vp, i64, vp, vp, vp, vp]
    L.gsb_l1_mask_fwd_bwd_batch.argtypes = [i32, i32, i32, i32, vp, vp, ctypes.c_float, vp, vp, vp]
    L.gsb_track_step_batch.argtypes = [i32, vp, vp, vp, vp, vp, vp, vp, i64, i32] + [ctypes.c_float] * 6 + [vp]
    L.gsb_backward_batch.argtypes = [ctypes.POINTER(GsbCamera), ctypes.POINTER(GsbGaussians), ctypes.POINTER(GsbFilter),
                                     i32, vp, vp, vp, i64, vp, vp, ctypes.POINTER(GsbGrads), vp, vp]
    L.gsb_backward_batch_stats.argtypes = [ctypes.POINTER(GsbCamera), ctypes.POINTER(GsbGaussians),
                                           ctypes.POINTER(GsbFilter), i32, i32, ctypes.POINTER(GsbDensifyStats), vp, vp,
                                           vp, i64, vp, vp, ctypes.POINTER(GsbGrads), vp, vp]
    L.gsb_render_batch_bg.argtypes = [ctypes.POINTER(GsbCamera), i32, i32, vp, vp, vp, sz, i64, vp, vp, vp, vp]
    L.gsb_backward_batch_stats_bg.argtypes = [ctypes.POINTER(GsbCamera), ctypes.POINTER(GsbGaussians),
                                              ctypes.POINTER(GsbFilter), i32, vp, i32, ctypes.POINTER(GsbDensifyStats),
                                              vp, vp, vp, i64, vp, vp, ctypes.POINTER(GsbGrads), vp, vp]
    L.gsb_loss_forward_batch.argtypes = [i32, i32, i32, i32, vp, vp, vp, vp, vp, vp]
    L.gsb_loss_backward_batch.argtypes = [i32, i32, i32, i32, vp, vp, vp, vp, ctypes.c_float, vp, vp]
    L.gsb_image_metrics_scratch_bytes.restype = sz
    L.gsb_image_metrics_scratch_bytes.argtypes = [i32, i32, i32, i32]
    L.gsb_image_metrics_batch.argtypes = [i32, i32, i32, i32, vp, vp, vp, i32, vp, vp, sz, vp]
    L.gsb_frames_u8_batch.argtypes = [i32, i32, i32, vp, vp, vp]
    L.gsb_lpips_scratch_bytes.restype = sz
    L.gsb_lpips_scratch_bytes.argtypes = [i32, i32, i32]
    L.gsb_lpips_prepare.argtypes = [i32, i32, i32, vp, vp, vp, vp]
    L.gsb_lpips_conv3x3_relu.argtypes = [i32, i32, i32, i32, i32, vp, vp, vp, vp, vp]
    L.gsb_lpips_maxpool2.argtypes = [i32, i32, i32, i32, vp, vp, vp]
    L.gsb_lpips_head.argtypes = [i32, i32, i32, i32, vp, vp, i32, vp, vp, vp]
    L.gsb_png_bound.restype = sz
    L.gsb_png_bound.argtypes = [i32, i32]
    L.gsb_png_scratch_bytes.restype = sz
    L.gsb_png_scratch_bytes.argtypes = [i32, i32, i32]
    L.gsb_png_encode_batch.argtypes = [i32, i32, i32, vp, vp, sz, vp, vp, vp]
    L.gsb_resample_u8_batch.argtypes = [i32, i32, i32, i32, i32, vp, vp, vp, vp, i32, vp, vp, i32, vp, sz, vp]
    L.gsb_ply_pack.argtypes = [i64, i32, ctypes.POINTER(GsbPlySegment), vp, vp]
    L.gsb_ply_unpack.argtypes = [i64, vp, i32, ctypes.POINTER(GsbPlySegment), vp]
    L.gsb_jpeg_scratch_bytes.restype = sz
    L.gsb_jpeg_scratch_bytes.argtypes = [i32, ctypes.POINTER(GsbJpegFile), i32]
    L.gsb_jpeg_decode_batch.argtypes = [i32, ctypes.POINTER(GsbJpegFile), vp, i32, vp, sz, vp, vp, vp]
    for f in ("gsb_preprocess_batch", "gsb_render_batch", "gsb_backward_pose_batch", "gsb_l1_mask_fwd_bwd_batch",
              "gsb_track_step_batch", "gsb_backward_batch", "gsb_loss_forward_batch", "gsb_loss_backward_batch",
              "gsb_backward_batch_stats", "gsb_image_metrics_batch", "gsb_frames_u8_batch", "gsb_lpips_prepare",
              "gsb_lpips_conv3x3_relu", "gsb_lpips_maxpool2", "gsb_lpips_head", "gsb_render_batch_bg",
              "gsb_backward_batch_stats_bg", "gsb_png_encode_batch", "gsb_resample_u8_batch", "gsb_ply_pack",
              "gsb_ply_unpack", "gsb_jpeg_decode_batch"):
        getattr(L, f).restype = ctypes.c_int
    L.gsb_adam_step_gated.argtypes = [i32, ctypes.POINTER(GsbAdamTensor), vp, vp, vp]
    L.gsb_adam_step_gated.restype = ctypes.c_int
    L.gsb_backward.argtypes = [ctypes.POINTER(GsbCamera), ctypes.POINTER(GsbGaussians), vp, vp, i64, vp, vp,
                               ctypes.POINTER(GsbGrads), vp]
    L.gsb_mark_visible.argtypes = [i32, vp, vp, vp, vp, vp]
    L.gsb_ssim_forward.argtypes = [i32, i32, i32, vp, vp, vp, vp, vp]
    L.gsb_ssim_backward.argtypes = [i32, i32, i32, vp, vp, vp, ctypes.c_float, vp, vp, vp]
    L.gsb_loss_forward.argtypes = [i32, i32, i32, vp, vp, vp, vp, vp]
    L.gsb_loss_backward.argtypes = [i32, i32, i32, vp, vp, vp, ctypes.c_float, vp, vp]
    L.gsb_adam_step.argtypes = [i32, ctypes.POINTER(GsbAdamTensor), vp, vp]
    L.gsb_last_error.restype = ctypes.c_char_p
    L.gsb_abi_version.restype = ctypes.c_int
    L.gsb_profile_enable.argtypes = [ctypes.c_int]
    L.gsb_profile_enable.restype = None
    L.gsb_profile_collect.argtypes = [vp, vp, ctypes.c_int]
    L.gsb_profile_collect.restype = ctypes.c_int
    L.gsb_launch_count.restype = ctypes.c_uint64
    L.gsb_set_option.argtypes = [ctypes.c_char_p, ctypes.c_int]
    L.gsb_set_option.restype = ctypes.c_int
    L.gsb_adam_gate.argtypes = [i32, ctypes.POINTER(GsbAdamTensor), vp, vp]
    L.gsb_ipc_alloc.argtypes = [sz, ctypes.POINTER(vp), ctypes.c_char_p]
    L.gsb_ipc_open.argtypes = [ctypes.c_char_p, ctypes.POINTER(vp)]
    L.gsb_ipc_close.argtypes = [vp]
    L.gsb_ipc_free.argtypes = [vp]
    L.gsb_fused_rs_adam_ag.argtypes = [i32, i32, ctypes.POINTER(vp), ctypes.POINTER(vp), vp, vp, i64, i32,
                                       ctypes.POINTER(GsbShardPiece), vp, vp, ctypes.c_float, vp, vp]
    L.gsb_knn_scratch_bytes.argtypes = [i32]
    L.gsb_knn_scratch_bytes.restype = sz
    L.gsb_knn_mean_dist2.argtypes = [i32, vp, vp, vp, sz, vp]
    L.gsb_knn_mean_dist2.restype = ctypes.c_int
    for f in ("gsb_adam_gate", "gsb_ipc_alloc", "gsb_ipc_open", "gsb_ipc_close", "gsb_ipc_free",
              "gsb_fused_rs_adam_ag"):
        getattr(L, f).restype = ctypes.c_int
    for f in ("gsb_preprocess", "gsb_preprocess_ex", "gsb_backward_ex", "gsb_backward_stats", "gsb_mip_filter3d", "gsb_render", "gsb_backward", "gsb_mark_visible", "gsb_ssim_forward",
              "gsb_ssim_backward", "gsb_loss_forward", "gsb_loss_backward", "gsb_adam_step"):
        getattr(L, f).restype = ctypes.c_int
    _lib = L
    return L


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = lib().gsb_last_error().decode(errors="replace")
        kind = {-1: "invalid argument", -2: "CUDA error", -3: "buffer too small"}.get(rc, str(rc))
        raise GsbError(f"{what}: {kind}: {msg}")


def stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


def ptr(t):
    """Device pointer of a contiguous fp32/int CUDA tensor (or None)."""
    if t is None:
        return None
    if not t.is_cuda:
        raise GsbError("expected a CUDA tensor (there is no CPU path)")
    if not t.is_contiguous():
        raise GsbError("expected a contiguous tensor")
    return t.data_ptr()


def f32c(t):
    """Return t as a contiguous fp32 CUDA tensor (no copy when it already is)."""
    if t is None:
        return None
    if not t.is_cuda:
        raise GsbError("expected a CUDA tensor (there is no CPU path)")
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()
