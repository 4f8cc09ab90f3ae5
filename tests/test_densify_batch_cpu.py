"""Densify with batched training, host side (no GPU): batch_densify_events, which step() and step_batch both run,
against a per-iteration restatement of train.py's densify / reset rules, and the batched statistics entry point is
exported and declared."""
import os
import re

from instantsplat_b200.trainer import OptimConfig, batch_densify_events

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_batched_statistics_symbol_exported_and_declared():
    import __graft_entry__ as G
    G.build()
    import instantsplat_b200 as I
    L = I.lib()
    hdr = open(os.path.join(ROOT, "include", "gsb200.h")).read()
    declared = set(re.findall(r"GSB_API [^;(]*?\b(gsb_\w+)\(", hdr))
    name = "gsb_backward_batch_stats"
    assert name in declared and name in I._lib.EXPORTS and hasattr(L, name)
    assert L.gsb_abi_version() == 2


def _per_iteration(cfg, before, V, white):
    """train.py's rules applied to each iteration j the step covers, then merged: the statistics views, whether
    any j densifies or resets, and the size threshold of the last densify point."""
    stats, dens, reset = [], [], False
    for j in range(before + 1, before + V + 1):
        s = j < cfg.densify_until_iter
        stats.append(s)
        if s and j > cfg.densify_from_iter and j % cfg.densification_interval == 0:
            dens.append(j)
        reset |= s and (j % cfg.opacity_reset_interval == 0 or (white and j == cfg.densify_from_iter))
    n = sum(stats)
    assert stats == [True] * n + [False] * (V - n)                    # the counted views are a prefix
    size = None
    if dens:
        size = cfg.size_threshold if dens[-1] > cfg.opacity_reset_interval else None
    return dict(n_stats=n, densify=bool(dens), reset=reset, size_threshold=size), len(dens)


def _cfg(**kw):
    c = OptimConfig()
    for k, v in kw.items():
        setattr(c, k, v)
    return c


CONFIGS = [
    _cfg(densify_from_iter=5, densification_interval=5, opacity_reset_interval=20, densify_until_iter=150),
    _cfg(densify_from_iter=4, densification_interval=3, opacity_reset_interval=10, densify_until_iter=97),
    _cfg(densify_from_iter=0, densification_interval=2, opacity_reset_interval=7, densify_until_iter=61),
    _cfg(densify_from_iter=30, densification_interval=100, opacity_reset_interval=50, densify_until_iter=180),
]


def test_batch_events_equal_the_per_iteration_rules():
    seen = dict(two_densify=0, until=0, size_none_and_set=set(), reset_white_only=0)
    for cfg in CONFIGS:
        for white in (False, True):
            for V in (1, 2, 3, 5, 12):
                for before in range(200):
                    want, n_dens = _per_iteration(cfg, before, V, white)
                    got = batch_densify_events(cfg, before, V, white)
                    assert got == want, (vars(cfg), white, V, before, got, want)
                    seen["two_densify"] += n_dens >= 2
                    seen["until"] += 0 < got["n_stats"] < V
                    if got["densify"]:
                        seen["size_none_and_set"].add(got["size_threshold"])
                    if white and got["reset"] and not _per_iteration(cfg, before, V, False)[0]["reset"]:
                        seen["reset_white_only"] += 1
    assert seen["two_densify"] > 0 and seen["until"] > 0 and seen["reset_white_only"] > 0
    assert seen["size_none_and_set"] == {None, 20}


def test_one_view_is_step():
    """V = 1, step()'s case, is train.py's rule: statistics while iteration < densify_until_iter, the densify and reset
    iterations themselves, and size_threshold past the first reset interval."""
    c = CONFIGS[0]
    assert batch_densify_events(c, 9, 1, False) == dict(n_stats=1, densify=True, reset=False, size_threshold=None)
    assert batch_densify_events(c, 19, 1, False) == dict(n_stats=1, densify=True, reset=True, size_threshold=None)
    assert batch_densify_events(c, 24, 1, False) == dict(n_stats=1, densify=True, reset=False, size_threshold=20)
    assert batch_densify_events(c, 4, 1, True)["reset"] and not batch_densify_events(c, 4, 1, False)["reset"]
    assert batch_densify_events(c, 149, 1, False)["n_stats"] == 0
    assert batch_densify_events(c, 148, 1, False)["n_stats"] == 1


def test_a_batch_fires_each_event_once_at_its_end():
    c = CONFIGS[0]
    # 18..24 covers 20 (densify + reset): one densify, one reset; size from the last point (20 is not past 20)
    assert batch_densify_events(c, 17, 7, False) == dict(n_stats=7, densify=True, reset=True, size_threshold=None)
    # 19..30 covers densify points 20, 25 and 30: size from 30
    assert batch_densify_events(c, 18, 12, False)["size_threshold"] == 20
    # across densify_until_iter = 150: views of iterations 147..149 count, 150 and 151 do not
    assert batch_densify_events(c, 146, 5, False)["n_stats"] == 3
    assert batch_densify_events(c, 160, 5, False) == dict(n_stats=0, densify=False, reset=False, size_threshold=None)
