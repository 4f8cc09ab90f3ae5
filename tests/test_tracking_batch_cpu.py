"""Batched tracking, host side (no GPU): the batched entry points are exported and declared, and the batched sizing
helpers grow with the view count as include/gsb200.h documents, never below the single-view sizes at V = 1."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BATCH = ("gsb_geom_bytes_batch", "gsb_binning_bytes_batch", "gsb_image_bytes_batch", "gsb_status_device_batch",
         "gsb_preprocess_batch", "gsb_render_batch", "gsb_backward_pose_batch", "gsb_l1_mask_fwd_bwd_batch",
         "gsb_track_step_batch")


def _lib():
    import __graft_entry__ as G
    G.build()
    import instantsplat_b200 as I
    return I, I.lib()


def test_batched_symbols_exported_and_declared():
    I, L = _lib()
    hdr = open(os.path.join(ROOT, "include", "gsb200.h")).read()
    declared = set(re.findall(r"GSB_API [^;(]*?\b(gsb_\w+)\(", hdr))
    for name in BATCH:
        assert name in declared and name in I._lib.EXPORTS and hasattr(L, name), name
    assert L.gsb_abi_version() == 2


def test_batched_sizes_grow_with_views():
    _, L = _lib()
    for P, W, H in ((1000, 1920, 1080), (450_000, 512, 288), (1, 17, 9)):
        T = ((W + 15) // 16) * ((H + 15) // 16)
        assert L.gsb_geom_bytes_batch(P, 1, W, H) >= L.gsb_geom_bytes(P)
        assert L.gsb_image_bytes_batch(W, H, 1) >= L.gsb_image_bytes(W, H)
        assert L.gsb_binning_bytes_batch(5000, W, H, 1) >= L.gsb_binning_bytes(5000, W, H)
        for V in (2, 5, 12):
            # ~145 bytes per (view, Gaussian): record 48, binning record 16, tile count 4, clamp flag 1, moments 72,
            # big-rect queue 4 (plus 64 bytes of pose partials per 128); the per-tile arrays (5 x 4 bytes) grow once
            # V * T exceeds 65536
            g1, gV = L.gsb_geom_bytes_batch(P, 1, W, H), L.gsb_geom_bytes_batch(P, V, W, H)
            assert gV - g1 >= (V - 1) * 145 * P
            assert gV - g1 <= (V - 1) * (146 * P + 4096) + 5 * 4 * max(0, V * T - 65536) + 8192
            assert L.gsb_image_bytes_batch(W, H, V) >= V * 2 * 4 * W * H
            assert (L.gsb_binning_bytes_batch(5000, W, H, V) - L.gsb_binning_bytes_batch(5000, W, H, 1)
                    >= (V - 1) * T * 8 - 256)            # 8 bytes per tile range, arrays 256-byte aligned
    # the status words lie before the per-tile arrays, at the same offset as the single-view buffer's when V = 1
    assert L.gsb_status_device_batch(4096, 1000, 1) == L.gsb_status_device(4096, 1000)
    assert L.gsb_status_device_batch(4096, 1000, 3) > L.gsb_status_device(4096, 1000)
