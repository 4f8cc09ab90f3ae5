"""Adaptive density control on the CPU: the mirror's densify_and_prune (through the shared densify_plan) against what
the reference's own densify_and_clone / densify_and_split / densify_and_prune computed (tests/golden/densify.npz,
oracle/make_golden_densify.py), the scene extent against getNerfppNorm, and the new C entry point."""
import os

import numpy as np
import pytest
import torch

from instantsplat_b200.densify import cameras_extent, densify_plan
from instantsplat_b200.model import GaussianModel, optimization_defaults

KEYS = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")
CASES = (("prune", False, 20), ("prune_nosize", False, None), ("cs", True, 20), ("cs_nosize", True, None))


@pytest.fixture(scope="module")
def z(golden_dir):
    return np.load(os.path.join(golden_dir, "densify.npz"))


def _mirror(z):
    T = lambda a: torch.from_numpy(np.array(a))
    m = GaussianModel(3, "cpu")
    m._set_params({k: T(z["init_" + k]) for k in KEYS})
    m.init_RT_seq(T(z["poses0"]))
    m.spatial_lr_scale = 1.0
    m.training_setup_pp(optimization_defaults(iterations=1000), T(z["ppl0"]))
    for k in KEYS:
        p = getattr(m, m._ATTR[k])
        m.optimizer.state[p] = dict(step=3, exp_avg=T(z["m_" + k]), exp_avg_sq=T(z["v_" + k]))
    m.xyz_gradient_accum, m.denom, m.max_radii2D = T(z["grad_accum"]), T(z["denom"]), T(z["max_radii2D"])
    return m


@pytest.mark.parametrize("tag,clone_and_split,size", CASES)
def test_mirror_densify_and_prune_matches_reference(z, tag, clone_and_split, size):
    m = _mirror(z)
    gen = torch.Generator().manual_seed(int(z["split_seed"]))
    plan = m.densify_and_prune(float(z["max_grad"]), float(z["min_opacity"]), float(z["extent"]), size,
                               clone_and_split=clone_and_split, generator=gen)
    P = int(z[f"{tag}_P"])
    assert m._xyz.shape[0] == P == plan.P
    np.testing.assert_array_equal(plan.src.numpy(), z[f"{tag}_src"])
    if clone_and_split:
        assert int(plan.clone.sum()) == int(z[f"{tag}_n_clone"]) > 0
        np.testing.assert_array_equal(plan.split_sel.numpy(), z[f"{tag}_split_mask"])
        assert int(plan.split_sel.sum()) > 0
    np.testing.assert_array_equal(plan.keep.numpy(), ~z[f"{tag}_prune_mask"])
    assert 0 < int((~plan.keep).sum()) < plan.keep.numel()
    for k in KEYS:
        p = getattr(m, m._ATTR[k])
        st = m.optimizer.state[p]
        np.testing.assert_array_equal(p.detach().numpy(), z[f"{tag}_p_{k}"], err_msg=k)
        np.testing.assert_array_equal(st["exp_avg"].numpy(), z[f"{tag}_m_{k}"], err_msg=k)
        np.testing.assert_array_equal(st["exp_avg_sq"].numpy(), z[f"{tag}_v_{k}"], err_msg=k)
        assert st["step"] == 3
    np.testing.assert_array_equal(m.xyz_gradient_accum.numpy(), z[f"{tag}_grad_accum"])
    np.testing.assert_array_equal(m.denom.numpy(), z[f"{tag}_denom"])
    np.testing.assert_array_equal(m.max_radii2D.numpy(), z[f"{tag}_max_radii2D"])
    np.testing.assert_array_equal(m.per_point_lr.numpy(), z[f"{tag}_ppl"])
    assert m.optimizer.param_groups[0]["per_point_lr"] is m.per_point_lr


def test_plan_equals_the_three_reference_steps_in_sequence(z):
    """The mirror's own densify_and_clone + densify_and_split + prune (the sequence the plan composes) give the same
    rows as the one-rebuild plan."""
    a, b = _mirror(z), _mirror(z)
    args = float(z["max_grad"]), float(z["min_opacity"]), float(z["extent"]), 20
    a.densify_and_prune(*args, clone_and_split=True, generator=torch.Generator().manual_seed(5))
    grads = b.xyz_gradient_accum / b.denom
    grads[grads.isnan()] = 0.0
    b.densify_and_clone(grads, args[0], args[2])
    b.densify_and_split(grads, args[0], args[2], generator=torch.Generator().manual_seed(5))
    b.densify_and_prune(*args, clone_and_split=False)
    for k in KEYS:
        pa, pb = getattr(a, a._ATTR[k]), getattr(b, b._ATTR[k])
        assert torch.equal(pa.detach(), pb.detach()), k
        for s in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(a.optimizer.state[pa][s], b.optimizer.state[pb][s]), (k, s)
    assert torch.equal(a.per_point_lr, b.per_point_lr)
    assert torch.equal(a.max_radii2D, b.max_radii2D) and torch.equal(a.denom, b.denom)


def test_plan_without_selection_is_identity():
    P = 50
    g = torch.Generator().manual_seed(3)
    xyz, sc, rot = torch.randn(P, 3, generator=g), torch.full((P, 3), -4.0), torch.randn(P, 4, generator=g)
    op = torch.full((P, 1), 2.0)
    plan = densify_plan(xyz, sc, rot, op, torch.zeros(P, 1), torch.zeros(P, 1), torch.zeros(P), 2e-4, 0.005, 1.0,
                        20, 0.01, clone_and_split=True)
    assert torch.equal(plan.src, torch.arange(P)) and not bool(plan.new.any()) and plan.split.numel() == 0
    assert plan.reset_stats


def test_cameras_extent_matches_getNerfppNorm(z):
    # getWorld2View2 works in fp32, cameras_extent in fp64
    r = cameras_extent(torch.from_numpy(z["cam_poses7"]))
    assert abs(r - float(z["cam_radius"])) <= 1e-6 * float(z["cam_radius"])


def test_build_exports_backward_stats():
    from instantsplat_b200 import _lib
    assert "gsb_backward_stats" in _lib.EXPORTS
    so = _lib.LIB_PATH
    if not os.path.exists(so):
        pytest.skip("libgsb200.so not built")
    assert hasattr(_lib.lib(), "gsb_backward_stats")
    assert _lib.lib().gsb_abi_version() == 2
