"""JointTrainer's learning-rate table and Adam step sizes against the mirror GaussianModel's optimizer, on the CPU:
the group learning rates of training_setup_pp / update_learning_rate, and the step size PerPointAdam derives from a
group's `lr` and its tensor's step count (scene/per_point_adam.py:76-81)."""
import pytest
import torch

from instantsplat_b200.model import GaussianModel, optimization_defaults
from instantsplat_b200.trainer import SEGMENTS, OptimConfig, adam_step_sizes, group_lrs

NAMES = tuple(name for name, _ in SEGMENTS) + ("pose",)
SCALE = 2.5          # spatial_lr_scale: not 1, so that a missing factor shows


def mirror(args):
    g = torch.Generator().manual_seed(0)
    m = GaussianModel(3, "cpu")
    m._set_params({name: torch.randn(4, k, generator=g) for name, k in SEGMENTS})
    m.init_RT_seq(torch.randn(2, 7, generator=g))
    m.spatial_lr_scale = SCALE
    m.training_setup_pp(args)
    return m


def config(args):
    cfg = OptimConfig()
    for k, v in vars(args).items():
        setattr(cfg, k, v)
    cfg.spatial_lr_scale = SCALE
    return cfg


def lrs_of(m):
    return {g["name"]: g["lr"] for g in m.optimizer.param_groups}


# (iteration, opt_step, lag): lags are the optimizer steps a tensor skipped (densify / opacity reset iterations)
@pytest.mark.parametrize("iteration,opt_step,lag", [
    (0, 1, {}),
    (1, 1, {}),
    (7, 7, {}),
    (300, 299, {"opacity": 1}),
    (600, 600, dict({name: 1 for name, _ in SEGMENTS}, opacity=2)),
    (999, 40, {"xyz": 39, "f_rest": 5}),
])
def test_step_sizes_follow_per_point_adam(iteration, opt_step, lag):
    args = optimization_defaults(iterations=1000)
    m = mirror(args)
    m.update_learning_rate(iteration)
    sizes = adam_step_sizes(config(args), iteration, opt_step, lag)
    assert tuple(sizes) == NAMES
    for g in m.optimizer.param_groups:
        assert g["betas"] == (0.9, 0.999) and g["eps"] == 1e-15
        t = opt_step - lag.get(g["name"], 0)
        assert sizes[g["name"]] == g["lr"] * ((1 - 0.999 ** t) ** 0.5 / (1 - 0.9 ** t)), g["name"]
        # what the kernels read: the same float32 either way
        assert torch.tensor(sizes[g["name"]], dtype=torch.float32) == \
            torch.tensor(g["lr"] * ((1 - 0.999 ** t) ** 0.5 / (1 - 0.9 ** t)), dtype=torch.float32)


@pytest.mark.parametrize("iteration", [None, 0, 1, 250, 1000])
def test_group_lrs_are_training_setup_pp_s(iteration):
    args = optimization_defaults(iterations=1000)
    m = mirror(args)
    if iteration is not None:
        m.update_learning_rate(iteration)
    assert group_lrs(args, SCALE, iteration) == lrs_of(m)
    assert tuple(group_lrs(config(args), SCALE, iteration)) == NAMES
    # training_setup (torch.optim.Adam) starts from the same groups and rates
    m.training_setup(args)
    assert lrs_of(m) == group_lrs(args, SCALE)
    assert all(g["eps"] == 1e-15 for g in m.optimizer.param_groups)


def test_optimization_defaults_are_unchanged():
    assert vars(optimization_defaults()) == dict(
        iterations=30_000, position_lr_init=0.00016, position_lr_final=0.0000016, position_lr_delay_mult=0.01,
        position_lr_max_steps=30_000, feature_lr=0.0025, opacity_lr=0.05, scaling_lr=0.005, rotation_lr=0.001,
        percent_dense=0.01, lambda_dssim=0.2, densification_interval=100, opacity_reset_interval=3000,
        densify_from_iter=500, densify_until_iter=15_000, densify_grad_threshold=0.0002,
        random_background=False, pp_optimizer=True, optim_pose=True)
    over = optimization_defaults(iterations=1000, random_background=True)
    assert over.iterations == 1000 and over.random_background is True
