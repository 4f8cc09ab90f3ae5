"""Batched training, host side (no GPU): the batched training entry points are exported and declared, and the
schedule accounting of one optimizer step over V views (SH-degree steps, 3D-filter recomputes, learning rates, the
last-iteration rule) is that of step() on V ranks."""
import os
import re

from instantsplat_b200.trainer import OptimConfig, adam_step_sizes, batch_events, group_lrs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BATCH = ("gsb_backward_batch", "gsb_loss_forward_batch", "gsb_loss_backward_batch")


def test_batched_training_symbols_exported_and_declared():
    import __graft_entry__ as G
    G.build()
    import instantsplat_b200 as I
    L = I.lib()
    hdr = open(os.path.join(ROOT, "include", "gsb200.h")).read()
    declared = set(re.findall(r"GSB_API [^;(]*?\b(gsb_\w+)\(", hdr))
    for name in BATCH:
        assert name in declared and name in I._lib.EXPORTS and hasattr(L, name), name
    assert L.gsb_abi_version() == 2


def _run(cfg, V, n):
    """Restatement of train.py's per-view schedules for n steps of V views: the events of each step are those of its
    last view, as on V ranks."""
    it, out = 0, []
    for _ in range(n):
        views = range(it + 1, it + V + 1)
        out.append(dict(iteration=it + V,
                        sh_up=any(i % cfg.sh_increase_interval == 0 for i in views),
                        mip=any(i % cfg.mip_filter3d_interval == 0 for i in views) and it + V < cfg.iterations - 100,
                        do_opt=it + V < cfg.iterations))
        it += V
    return out


def test_schedule_events_with_v_views_per_step():
    cfg = OptimConfig()
    cfg.sh_increase_interval, cfg.mip_filter3d_interval, cfg.iterations = 4, 5, 130
    for V in (1, 2, 3, 5, 12):
        it = 0
        for k, want in enumerate(_run(cfg, V, 140 // V)):
            ev = batch_events(cfg, it, V)
            assert ev == want, (V, k, ev, want)
            it = ev["iteration"]
    # V = 3 from 0: iterations 3, 6, 9, 12, ...; SH steps cross 4, 8, 12; recomputes cross 5, 10, 15
    cfg.iterations = 30_000
    evs = [batch_events(cfg, 3 * k, 3) for k in range(5)]
    assert [e["sh_up"] for e in evs] == [False, True, True, True, False]
    assert [e["mip"] for e in evs] == [False, True, False, True, True]
    # no recompute within the last 100 iterations, no Adam step at the last one
    cfg.iterations = 120
    assert not batch_events(cfg, 18, 3)["mip"] and batch_events(cfg, 3, 3)["mip"]
    assert batch_events(cfg, 117, 3)["do_opt"] is False and batch_events(cfg, 114, 3)["do_opt"] is True


def test_learning_rates_follow_the_iteration_not_the_step():
    cfg = OptimConfig()
    lag = {}
    # after k steps of V views the rates are those of iteration k V, the bias correction that of step k
    for V, k in ((3, 1), (3, 7), (12, 5)):
        sizes = adam_step_sizes(cfg, k * V, k, lag)
        lrs = group_lrs(cfg, cfg.spatial_lr_scale, k * V)
        b1, b2 = 0.9, 0.999
        for name, lr in lrs.items():
            assert sizes[name] == lr * ((1 - b2 ** k) ** 0.5 / (1 - b1 ** k)), (V, k, name)
