"""Generate tests/golden/surgery.npz from the REFERENCE's own GaussianModel (scene/gaussian_model.py): the
optimizer-state surgery behind densify / prune / opacity reset (SURVEY.md section 8 row f4) --
`prune_points` (:359-374), `densification_postfix` (:399-418), `reset_opacity` (:280-283) -- interleaved with
`update_learning_rate` + `PerPointAdam.step` on seeded gradients.

Needs an InstantSplat checkout (CPU; `.cuda()` / device="cuda" are neutralised, the native packages are the
oracle-backed stand-ins of tests/cpu_standins).  The GPU tests replay the same script on `JointTrainer` and on the
mirror `instantsplat_b200.model.GaussianModel` and must land on these vectors.

    python oracle/make_golden_surgery.py <path to the InstantSplat checkout>
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

ref_gm.torch = _TorchNoCuda()
from instantsplat_b200.model import optimization_defaults  # noqa: E402
from instantsplat_b200.scenes import surface_scene  # noqa: E402

KEYS = (("_xyz", "xyz"), ("_features_dc", "f_dc"), ("_features_rest", "f_rest"), ("_opacity", "opacity"),
        ("_scaling", "scaling"), ("_rotation", "rotation"))


def main():
    sc = surface_scene(60, 2, 32, 32, seed=13, sh_degree=3)
    g = torch.Generator().manual_seed(99)
    m = ref_gm.GaussianModel(3)
    for attr, key in KEYS:
        setattr(m, attr, torch.nn.Parameter(sc.params[key].clone().requires_grad_(True)))
    m.P = sc.poses.clone().requires_grad_(True)
    m.spatial_lr_scale = 1.0
    m.max_radii2D = torch.zeros(sc.P)
    ppl = sc.per_point_lr.clone()
    m.training_setup_pp(optimization_defaults(iterations=1000), ppl)
    # The reference's _prune_optimizer / cat_tensors_to_optimizer walk EVERY param group and index it with the
    # per-Gaussian mask, which raises on the [n_views,7] pose group (densification is dormant in InstantSplat,
    # train.py:195-206).  Drop the pose group so the reference functions can run on the six Gaussian groups.
    assert m.optimizer.param_groups[-1]["name"] == "pose"
    m.optimizer.param_groups.pop()
    out = {"ppl0": ppl.numpy(), "poses0": sc.poses.numpy()}
    for attr, key in KEYS:
        out["init_" + key] = getattr(m, attr).detach().numpy().copy()
    it = [0]

    def adam_step(tag):
        it[0] += 1
        m.update_learning_rate(it[0])
        for attr, key in KEYS:
            p = getattr(m, attr)
            gr = torch.randn(p.shape, generator=g) * 1e-2
            p.grad = gr
            out[f"{tag}_g_{key}"] = gr.numpy().copy()
        m.optimizer.step()
        for attr, key in KEYS:
            p = getattr(m, attr)
            st = m.optimizer.state[p]
            out[f"{tag}_p_{key}"] = p.detach().numpy().copy()
            out[f"{tag}_m_{key}"] = st["exp_avg"].numpy().copy()
            out[f"{tag}_v_{key}"] = st["exp_avg_sq"].numpy().copy()
        out[f"{tag}_iteration"] = np.int64(it[0])

    adam_step("s1")
    adam_step("s2")
    # ---- prune
    mask = torch.rand(sc.P, generator=g) < 0.3
    out["prune_mask"] = mask.numpy()
    m.prune_points(mask)
    # the reference keeps per_point_lr un-pruned (it would fail its own shape check); prune it the way a caller must
    m.per_point_lr = ppl[~mask]
    m.optimizer.param_groups[0]["per_point_lr"] = m.per_point_lr
    adam_step("s3")
    # ---- append
    n_new = 17
    new = dict(xyz=torch.randn(n_new, 3, generator=g), f_dc=torch.randn(n_new, 1, 3, generator=g),
               f_rest=0.1 * torch.randn(n_new, 15, 3, generator=g), opacity=torch.randn(n_new, 1, generator=g),
               scaling=torch.randn(n_new, 3, generator=g) - 3.0, rotation=torch.randn(n_new, 4, generator=g))
    for k, v in new.items():
        out["new_" + k] = v.numpy().copy()
    m.densification_postfix(new["xyz"], new["f_dc"], new["f_rest"], new["opacity"], new["scaling"], new["rotation"])
    new_ppl = 1.0 + torch.rand(n_new, 1, generator=g)
    out["new_ppl"] = new_ppl.numpy()
    m.per_point_lr = torch.cat((m.per_point_lr, new_ppl))
    m.optimizer.param_groups[0]["per_point_lr"] = m.per_point_lr
    adam_step("s4")
    # ---- opacity reset
    m.reset_opacity()
    out["reset_opacity"] = m._opacity.detach().numpy().copy()
    adam_step("s5")
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "surgery.npz"), **out)
    print("wrote tests/golden/surgery.npz:", len(out), "arrays; final P =", m._xyz.shape[0])


if __name__ == "__main__":
    main()
