"""Generate tests/golden/checkpoint.npz from the REFERENCE's own checkpoint surface (scene/gaussian_model.py):
`create_from_pcd` (:146-172) -> `training_setup_pp` (:203-232) -> a few `update_learning_rate` (:234-243) +
`PerPointAdam.step` on seeded gradients, with one `prune_points` (:359-374) in between, -> `capture` (:65-80) ->
`restore` (:82-99) into a fresh model (which calls `training_setup`, :174-200).

Run like make_golden_surgery.py (CPU; `.cuda()` / device="cuda" are neutralised, `distCUDA2` is the stand-in of
tests/cpu_standins).  The reference's _prune_optimizer cannot index the [n_views,7] pose group, so the pose group is
taken out of the optimizer around the prune and put back; its state stays keyed by the pose table.  One step leaves
the opacity without a gradient (what a reset iteration does), so the per-tensor step counts differ.

    python oracle/make_golden_checkpoint.py <path to the InstantSplat checkout>
"""
import importlib.abc
import importlib.util
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if len(sys.argv) != 2:
    sys.exit(__doc__)
REF = sys.argv[1]
for p in (os.path.join(ROOT, "tests", "cpu_standins"), os.path.join(ROOT, "tests", "stubs"), ROOT):
    sys.path.insert(0, p)
sys.path.append(REF)


class _Stub(importlib.abc.MetaPathFinder, importlib.abc.Loader):
    def find_spec(self, name, path, target=None):
        if name.split(".")[0] == "matplotlib":
            return importlib.util.spec_from_loader(name, self, is_package=True)

    def create_module(self, spec):
        m = types.ModuleType(spec.name)
        m.__path__ = []
        return m

    def exec_module(self, m):
        pass


sys.meta_path.insert(0, _Stub())
import numpy as np  # noqa: E402
import torch  # noqa: E402

torch.Tensor.cuda = lambda self, *a, **k: self


class _TorchNoCuda:
    def __getattr__(self, name):
        obj = getattr(torch, name)
        if callable(obj) and not isinstance(obj, type):
            def call(*a, **k):
                if k.get("device") == "cuda":
                    k.pop("device")
                return obj(*a, **k)
            return call
        return obj


import scene.gaussian_model as ref_gm  # noqa: E402
from utils.graphics_utils import BasicPointCloud  # noqa: E402

ref_gm.torch = _TorchNoCuda()
from instantsplat_b200.model import optimization_defaults  # noqa: E402
from instantsplat_b200.scenes import surface_scene  # noqa: E402

KEYS = (("_xyz", "xyz"), ("_features_dc", "f_dc"), ("_features_rest", "f_rest"), ("_opacity", "opacity"),
        ("_scaling", "scaling"), ("_rotation", "rotation"))
GROUPS = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation", "pose")
N_STEPS, PRUNE_AFTER, NO_OPACITY_GRAD_AT = 5, 2, 4
SPATIAL_LR_SCALE = 2.5


def opt_args():
    return optimization_defaults(iterations=1000)


def group_record(prefix, opt, out):
    """Structure of an optimizer's state dict: group order, names, hyper-parameters, per-parameter state."""
    sd = opt.state_dict()
    gs = sd["param_groups"]
    out[prefix + "names"] = np.array([g["name"] for g in gs])
    out[prefix + "lr"] = np.array([float(g["lr"]) for g in gs])
    out[prefix + "betas"] = np.array([list(g["betas"]) for g in gs], dtype=np.float64)
    out[prefix + "eps"] = np.array([float(g["eps"]) for g in gs])
    out[prefix + "weight_decay"] = np.array([float(g["weight_decay"]) for g in gs])
    out[prefix + "params"] = np.array([g["params"] for g in gs])
    out[prefix + "keys"] = np.array([",".join(sorted(g)) for g in gs])
    out[prefix + "has_ppl"] = np.array([g.get("per_point_lr") is not None for g in gs])
    ppl = gs[0].get("per_point_lr")
    if ppl is not None:
        out[prefix + "per_point_lr"] = ppl.detach().numpy().copy()
    out[prefix + "state_ids"] = np.array(sorted(sd["state"]), dtype=np.int64)
    for i, st in sd["state"].items():
        s = st["step"]
        out[f"{prefix}step_{i}"] = np.float64(float(s))
        out[f"{prefix}step_is_tensor_{i}"] = np.bool_(torch.is_tensor(s))
        out[f"{prefix}m_{i}"] = st["exp_avg"].numpy().copy()
        out[f"{prefix}v_{i}"] = st["exp_avg_sq"].numpy().copy()


def main():
    sc = surface_scene(240, 3, 32, 32, seed=31, sh_degree=3)
    g = torch.Generator().manual_seed(17)
    P0 = sc.P
    points = sc.params["xyz"].numpy().astype(np.float32)
    colors = torch.rand(P0, 3, generator=g).numpy()
    ppl0 = 1.0 + torch.rand(P0, 1, generator=g)
    out = dict(points=points, colors=colors, ppl0=ppl0.numpy(), poses0=sc.poses.numpy(),
               spatial_lr_scale=np.float64(SPATIAL_LR_SCALE), n_steps=np.int64(N_STEPS),
               prune_after=np.int64(PRUNE_AFTER), no_opacity_grad_at=np.int64(NO_OPACITY_GRAD_AT))
    m = ref_gm.GaussianModel(3)
    m.create_from_pcd(BasicPointCloud(points=points, colors=colors, normals=np.zeros_like(points)), SPATIAL_LR_SCALE)
    for attr, key in KEYS:
        out["init_" + key] = getattr(m, attr).detach().numpy().copy()
    m.P = sc.poses.clone().requires_grad_(True)
    m.training_setup_pp(opt_args(), ppl0.clone())
    for it in range(1, N_STEPS + 1):
        m.update_learning_rate(it)
        for attr, key in KEYS + (("P", "pose"),):
            p = getattr(m, attr)
            if it == NO_OPACITY_GRAD_AT and key == "opacity":
                p.grad = None
                continue
            gr = torch.randn(p.shape, generator=g) * 1e-2
            p.grad = gr
            out[f"g{it}_{key}"] = gr.numpy().copy()
        m.optimizer.step()
        for attr, _ in KEYS + (("P", "pose"),):
            getattr(m, attr).grad = None
        if it == PRUNE_AFTER:
            mask = torch.rand(m._xyz.shape[0], generator=g) < 0.25
            out["prune_mask"] = mask.numpy()
            pose_group = m.optimizer.param_groups.pop()
            assert pose_group["name"] == "pose"
            m.prune_points(mask)
            m.optimizer.param_groups.append(pose_group)
            # the reference keeps per_point_lr un-pruned (it would fail its own shape check); prune it as a caller must
            m.per_point_lr = m.per_point_lr[~mask]
            m.optimizer.param_groups[0]["per_point_lr"] = m.per_point_lr
    m.oneupSHdegree()
    m.oneupSHdegree()
    P = m._xyz.shape[0]
    m.max_radii2D = torch.rand(P, generator=g) * 30.0
    m.denom = torch.randint(0, 6, (P, 1), generator=g).float()
    m.xyz_gradient_accum = m.denom * torch.rand(P, 1, generator=g) * 1e-3
    cap = m.capture()
    assert len(cap) == 13
    out["cap_active_sh_degree"] = np.int64(cap[0])
    for i, key in enumerate(("xyz", "f_dc", "f_rest", "scaling", "rotation", "opacity", "max_radii2D",
                             "xyz_gradient_accum", "denom")):
        out["cap_" + key] = cap[1 + i].detach().numpy().copy()
        out["cap_is_param_" + key] = np.bool_(isinstance(cap[1 + i], torch.nn.Parameter))
    out["cap_spatial_lr_scale"] = np.float64(cap[11])
    out["cap_P"] = cap[12].detach().numpy().copy()
    group_record("sd_", m.optimizer, out)
    # ---- restore into a fresh model
    r = ref_gm.GaussianModel(3)
    r.restore(cap, opt_args())
    out["rs_class"] = np.array(type(r.optimizer).__module__ + "." + type(r.optimizer).__name__)
    out["rs_active_sh_degree"] = np.int64(r.active_sh_degree)
    out["rs_param_is_model"] = np.array([r.optimizer.param_groups[i]["params"][0] is getattr(r, a)
                                         for i, a in enumerate([a for a, _ in KEYS] + ["P"])])
    group_record("rs_", r.optimizer, out)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "checkpoint.npz"), **out)
    print("wrote tests/golden/checkpoint.npz:", len(out), "arrays; P", P0, "->", P, "; optimizer after restore",
          out["rs_class"], "; steps", [out[f"sd_step_{i}"] for i in out["sd_state_ids"]])


if __name__ == "__main__":
    main()
