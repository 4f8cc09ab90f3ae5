"""Random background, host side (no GPU): the new entry points are exported, declared and bound with the argument
types of their C declarations; the option is off by default and outside the train CLI's configuration; several ranks
are refused before anything is allocated; the checkpoint field is optional and checked; a malformed background table
is refused before the library is called."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("gsb_render_batch_bg", "gsb_backward_batch_stats_bg")


def test_entry_points_exported_declared_and_typed():
    import __graft_entry__ as G
    G.build()
    import instantsplat_b200 as I
    from instantsplat_b200._lib import GsbCamera, GsbDensifyStats, GsbFilter, GsbGaussians, GsbGrads
    L = I.lib()
    hdr = open(os.path.join(ROOT, "include", "gsb200.h")).read()
    declared = set(re.findall(r"GSB_API [^;(]*?\b(gsb_\w+)\(", hdr))
    for name in NEW:
        assert name in declared and name in I._lib.EXPORTS and hasattr(L, name), name
        assert getattr(L, name).restype is ctypes.c_int
    vp, i32, i64, sz = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_size_t
    P = ctypes.POINTER
    # the existing entry point with the table inserted after V
    assert L.gsb_render_batch_bg.argtypes == [P(GsbCamera), i32, i32, vp, vp, vp, sz, i64, vp, vp, vp, vp]
    assert L.gsb_render_batch_bg.argtypes[:3] + L.gsb_render_batch_bg.argtypes[4:] == L.gsb_render_batch.argtypes
    want = [P(GsbCamera), P(GsbGaussians), P(GsbFilter), i32, vp, i32, P(GsbDensifyStats), vp, vp, vp, i64, vp, vp,
            P(GsbGrads), vp, vp]
    assert L.gsb_backward_batch_stats_bg.argtypes == want
    old = L.gsb_backward_batch_stats.argtypes
    assert want[:4] + want[5:] == old
    # the C declarations take the same parameters in the same order
    for name, params, at in (("gsb_render_batch_bg", 12, 3), ("gsb_backward_batch_stats_bg", 16, 4)):
        decl = re.search(name + r"\(([^)]*)\)", hdr).group(1)
        args = [a.strip() for a in decl.split(",")]
        assert len(args) == params and args[at - 1] == "int32_t V" and args[at] == "const float* bg", (name, args)
    assert L.gsb_abi_version() == 2


def test_defaults_leave_the_option_off():
    from instantsplat_b200 import train as T
    from instantsplat_b200.trainer import OptimConfig
    c = OptimConfig()
    assert c.random_background is False and c.background_seed == 0
    assert "random_background" not in T.LOOP_FIELDS and "background_seed" not in T.LOOP_FIELDS
    args = T.parse_args(["-s", "src", "-m", "out", "--n_views", "3"])
    assert T.optim_config(args, 1.0).random_background is False


def test_several_ranks_are_refused_with_the_reason():
    import instantsplat_b200 as I
    cfg = I.OptimConfig()
    cfg.random_background = True
    with pytest.raises(I.GsbError, match=r"random_background=True needs world_size == 1: the ranks' views"):
        I.JointTrainer(None, "cpu", cfg=cfg, world_size=2, rank=0)


def test_checkpoint_generator_field_is_optional_and_checked():
    from instantsplat_b200 import trainer as TR
    from test_checkpoint_cpu import trainer_format
    import numpy as np
    z = np.load(os.path.join(ROOT, "tests", "golden", "checkpoint.npz"))
    cap, it = trainer_format(z)
    assert "background_generator" not in TR._EXTRA_KEYS
    assert TR._parse_capture(cap, it)["extra"].get("background_generator") is None
    extra = cap[10][TR.CHECKPOINT_KEY]
    extra["background_generator"] = torch.Generator().manual_seed(0).get_state()
    TR._parse_capture(cap, it)
    extra["background_generator"] = [1, 2, 3]
    with pytest.raises(TR._lib.GsbError, match="background_generator must be a generator state"):
        TR._parse_capture(cap, it)


@pytest.mark.parametrize("bad", ["cpu", "shape", "dtype", "list"])
def test_malformed_background_table_is_refused(bad):
    from instantsplat_b200 import _lib
    from instantsplat_b200.frame import _bg_table
    t = {"cpu": torch.zeros(2, 3), "shape": torch.zeros(3), "dtype": torch.zeros(2, 3, dtype=torch.float64),
         "list": [[0.0] * 3] * 2}[bad]
    with pytest.raises(_lib.GsbError, match=r"background table: expected a contiguous float32 \[2, 3\] CUDA tensor"):
        _bg_table(t, 2)
