"""Checkpoints on the CPU (DESIGN.md section 4.9): the mirror's capture / restore / training_setup against what the
reference's own functions computed (tests/golden/checkpoint.npz, oracle/make_golden_checkpoint.py), and the file
layout JointTrainer writes, read back by torch.load's default weights_only=True, the mirror's restore and
torch.optim.Adam."""
import copy
import os

import numpy as np
import pytest
import torch
from torch import nn

import instantsplat_b200 as I
from cpu_standins.per_point_adam_cpu import PerPointAdam as CpuPerPointAdam
from instantsplat_b200.model import GaussianModel, optimization_defaults
from instantsplat_b200.trainer import _EXTRA_KEYS, _parse_capture

KEYS = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")
CAP = ("xyz", "f_dc", "f_rest", "scaling", "rotation", "opacity", "max_radii2D", "xyz_gradient_accum", "denom")


@pytest.fixture(scope="module")
def z(golden_dir):
    return np.load(os.path.join(golden_dir, "checkpoint.npz"))


T = lambda a: torch.from_numpy(np.array(a))


def mirror_run(z):
    """The generator's script on the mirror: create_from_pcd, training_setup_pp, the seeded steps (the reference's
    update through the CPU stand-in of PerPointAdam) with the prune, then the statistics the golden captured."""
    m = GaussianModel(3, "cpu")
    m.create_from_pcd(z["points"], z["colors"], float(z["spatial_lr_scale"]))
    for k in KEYS:
        np.testing.assert_array_equal(getattr(m, m._ATTR[k]).detach().numpy(), z["init_" + k], err_msg=k)
    m.init_RT_seq(T(z["poses0"]))
    m.training_setup_pp(optimization_defaults(iterations=1000), T(z["ppl0"]))
    for it in range(1, int(z["n_steps"]) + 1):
        m.update_learning_rate(it)
        for k in KEYS + ("pose",):
            p = m.P if k == "pose" else getattr(m, m._ATTR[k])
            p.grad = T(z[f"g{it}_{k}"]) if f"g{it}_{k}" in z else None
        CpuPerPointAdam.step(m.optimizer)
        for k in KEYS:
            getattr(m, m._ATTR[k]).grad = None
        m.P.grad = None
        if it == int(z["prune_after"]):
            m.prune_points(T(z["prune_mask"]))
    m.oneupSHdegree()
    m.oneupSHdegree()
    m.max_radii2D = T(z["cap_max_radii2D"])
    m.xyz_gradient_accum, m.denom = T(z["cap_xyz_gradient_accum"]), T(z["cap_denom"])
    return m


def check_groups(prefix, opt, z, exact_keys=True):
    """An optimizer's state dict against the golden's record of the reference's (make_golden_checkpoint.group_record)."""
    sd = opt.state_dict()
    gs = sd["param_groups"]
    assert [g["name"] for g in gs] == z[prefix + "names"].tolist()
    assert [float(g["lr"]) for g in gs] == z[prefix + "lr"].tolist()
    assert [list(g["betas"]) for g in gs] == z[prefix + "betas"].tolist()
    assert [float(g["eps"]) for g in gs] == z[prefix + "eps"].tolist()
    assert [float(g["weight_decay"]) for g in gs] == z[prefix + "weight_decay"].tolist()
    assert [g["params"] for g in gs] == z[prefix + "params"].tolist()
    if exact_keys:
        assert [",".join(sorted(g)) for g in gs] == z[prefix + "keys"].tolist()
    assert [g.get("per_point_lr") is not None for g in gs] == z[prefix + "has_ppl"].tolist()
    np.testing.assert_array_equal(gs[0]["per_point_lr"].numpy(), z[prefix + "per_point_lr"])
    assert sorted(sd["state"]) == z[prefix + "state_ids"].tolist()
    for i, st in sd["state"].items():
        assert float(st["step"]) == float(z[f"{prefix}step_{i}"]), i
        assert torch.is_tensor(st["step"]) == bool(z[f"{prefix}step_is_tensor_{i}"]), i
        np.testing.assert_array_equal(st["exp_avg"].numpy(), z[f"{prefix}m_{i}"], err_msg=str(i))
        np.testing.assert_array_equal(st["exp_avg_sq"].numpy(), z[f"{prefix}v_{i}"], err_msg=str(i))


def test_mirror_capture_matches_reference(z):
    cap = mirror_run(z).capture()
    assert len(cap) == 13
    assert cap[0] == int(z["cap_active_sh_degree"])
    for i, k in enumerate(CAP):
        t = cap[1 + i]
        np.testing.assert_array_equal(t.detach().numpy(), z["cap_" + k], err_msg=k)
        assert isinstance(t, nn.Parameter) == bool(z["cap_is_param_" + k]), k
    assert cap[11] == float(z["cap_spatial_lr_scale"])
    np.testing.assert_array_equal(cap[12].detach().numpy(), z["cap_P"])
    assert cap[12].requires_grad
    assert len(set(float(z[f"sd_step_{i}"]) for i in z["sd_state_ids"])) == 2     # the opacity lags one step
    check_groups("sd_", _Packed(cap[10]), z)


class _Packed:
    """A state dict where check_groups expects an optimizer."""
    def __init__(self, sd):
        self.sd = sd

    def state_dict(self):
        return self.sd


def test_mirror_restore_matches_reference(z):
    cap = mirror_run(z).capture()
    r = GaussianModel(3, "cpu")
    r.restore(cap, optimization_defaults(iterations=1000))
    cls = type(r.optimizer)
    assert cls.__module__ + "." + cls.__name__ == str(z["rs_class"])
    assert r.active_sh_degree == int(z["rs_active_sh_degree"])
    params = [g["params"][0] for g in r.optimizer.param_groups]
    assert [p is getattr(r, a) for p, a in zip(params, [r._ATTR[k] for k in KEYS] + ["P"])] == \
        z["rs_param_is_model"].tolist()
    check_groups("rs_", r.optimizer, z)
    assert r.xyz_gradient_accum is cap[8] and r.denom is cap[9]


def test_training_setup_matches_training_setup_pp_groups(z):
    m = GaussianModel(3, "cpu")
    m.create_from_pcd(z["points"], z["colors"], float(z["spatial_lr_scale"]))
    m.init_RT_seq(T(z["poses0"]))
    a = optimization_defaults(iterations=1000)
    pp = [(g["name"], g["lr"]) for g in m.training_setup_pp(a, T(z["ppl0"])).param_groups]
    opt = m.training_setup(a)
    assert type(opt) is torch.optim.Adam and opt.defaults["eps"] == 1e-15 and opt.defaults["lr"] == 0.0
    assert [(g["name"], g["lr"]) for g in opt.param_groups] == pp
    assert all("per_point_lr" not in g for g in opt.param_groups)


# ---- the file JointTrainer writes ----------------------------------------------------------------------------------
def trainer_format(z):
    """A capture() tuple in JointTrainer's layout, from CPU tensors: the mirror's tuple plus the extra state."""
    cap = list(mirror_run(z).capture())
    P = cap[1].shape[0]
    sd = cap[10]
    for g in sd["param_groups"]:
        g["lr"] = float(g["lr"])             # JointTrainer writes Python floats; the schedules return numpy float64
    steps = {g["name"]: int(sd["state"][g["params"][0]]["step"]) for g in sd["param_groups"]}
    extra = dict(iteration=5, opt_step=steps["pose"], lag={k: steps["pose"] - steps[k] for k in KEYS},
                 densify_generator=torch.Generator().manual_seed(3).get_state(), scene_extent=1.25,
                 filter_3D=torch.rand(P), mip_recomputed_at=[], densified_at=[3], reset_at=[],
                 cfg={k: getattr(I.OptimConfig, k) for k in dir(I.OptimConfig) if not k.startswith("_")},
                 frame=dict(W=32, H=32, fovx=1.0, fovy=0.8, bg=[0.0, 0.0, 0.0], n_views=3, sh_degree=3))
    assert sorted(extra) == sorted(_EXTRA_KEYS)
    sd[I.CHECKPOINT_KEY] = extra
    return tuple(cap), 5


def test_trainer_format_loads_weights_only(z, tmp_path):
    cap, it = trainer_format(z)
    path = str(tmp_path / "chkpnt5.pth")
    torch.save((cap, it), path)
    (model_params, first_iter) = torch.load(path)                  # train.py:104, torch's default weights_only=True
    assert first_iter == 5
    (model_params2, _) = torch.load(path, weights_only=True)
    for a, b in zip(model_params, cap):
        if torch.is_tensor(b):
            assert type(a) is type(b) and torch.equal(a, b)
    assert isinstance(model_params[1], nn.Parameter) and model_params[1].requires_grad
    extra = model_params[10][I.CHECKPOINT_KEY]
    assert torch.equal(extra["densify_generator"], cap[10][I.CHECKPOINT_KEY]["densify_generator"])
    assert extra["cfg"] == cap[10][I.CHECKPOINT_KEY]["cfg"] and extra["frame"] == cap[10][I.CHECKPOINT_KEY]["frame"]
    # the mirror's restore (torch.optim.Adam.load_state_dict), extra key included
    r = GaussianModel(3, "cpu")
    r.restore(model_params, optimization_defaults(iterations=1000))
    assert type(r.optimizer) is torch.optim.Adam
    check_groups("rs_", r.optimizer, z)
    assert I.CHECKPOINT_KEY not in r.optimizer.state_dict()
    # a bare Adam over parameters of the same shapes
    ps = [nn.Parameter(torch.zeros_like(model_params2[i])) for i in (1, 2, 3, 6, 4, 5, 12)]
    opt = torch.optim.Adam([{"params": [p]} for p in ps], lr=0.0)
    opt.load_state_dict(model_params2[10])
    assert float(opt.state[ps[3]]["step"]) == float(z["sd_step_3"])
    # and JointTrainer's own parser
    t = _parse_capture(model_params, first_iter)
    assert t["P"] == cap[1].shape[0] and t["steps"]["opacity"] == t["steps"]["pose"] - 1
    assert t["extra"]["lag"]["opacity"] == 1


def test_mirror_checkpoint_parses_without_extra_state(z):
    cap = mirror_run(z).capture()
    t = _parse_capture(cap, 5)
    assert t["extra"] is None and t["steps"] == {k: int(z[f"sd_step_{i}"]) for i, k in
                                                 enumerate(KEYS + ("pose",))}
    assert torch.equal(t["per_point_lr"], cap[10]["param_groups"][0]["per_point_lr"].reshape(-1))


@pytest.mark.parametrize("case", ["length", "first_iter", "sh_type", "shape", "f_rest", "pose", "groups", "state",
                                  "ppl", "extra_missing", "extra_iteration", "filter"])
def test_malformed_checkpoints_are_refused(z, case):
    cap, it = trainer_format(z)
    cap = list(copy.deepcopy(cap))
    sd = cap[10]
    P = cap[1].shape[0]
    if case == "length":
        cap = cap[:12]
    elif case == "first_iter":
        it = -1
    elif case == "sh_type":
        cap[0] = 1.0
    elif case == "shape":
        cap[5] = cap[5][:, :3]
    elif case == "f_rest":
        cap[3] = cap[3].reshape(P, 3, 15)
    elif case == "pose":
        cap[12] = cap[12][:, :6]
    elif case == "groups":
        sd["param_groups"] = sd["param_groups"][:6]
    elif case == "state":
        del sd["state"][2]["exp_avg_sq"]
    elif case == "ppl":
        sd["param_groups"][0]["per_point_lr"] = torch.ones(P - 1, 1)
    elif case == "extra_missing":
        del sd[I.CHECKPOINT_KEY]["lag"]
    elif case == "extra_iteration":
        it = 6
    elif case == "filter":
        sd[I.CHECKPOINT_KEY]["filter_3D"] = torch.zeros(P + 1)
    with pytest.raises(I.GsbError, match="checkpoint"):
        _parse_capture(tuple(cap) if case != "length" else cap, it)


def test_mirror_checkpoint_file_reads_back(z, tmp_path):
    """The reference's (and the mirror's) state dict holds numpy float64 learning rates; read_checkpoint allows them."""
    cap = mirror_run(z).capture()
    assert any(isinstance(g["lr"], np.floating) for g in cap[10]["param_groups"])
    path = str(tmp_path / "chkpnt5.pth")
    torch.save((cap, 5), path)
    model_params, first_iter = I.read_checkpoint(path)
    assert first_iter == 5 and _parse_capture(model_params, first_iter)["extra"] is None
    assert [g["lr"] for g in model_params[10]["param_groups"]] == [g["lr"] for g in cap[10]["param_groups"]]


def test_read_checkpoint_refuses_other_objects(tmp_path):
    path = str(tmp_path / "x.pth")
    torch.save({"a": torch.zeros(1)}, path)
    with pytest.raises(I.GsbError, match="model_params, first_iter"):
        I.read_checkpoint(path)
