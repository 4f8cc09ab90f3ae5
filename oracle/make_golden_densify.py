"""Generate tests/golden/densify.npz from the REFERENCE's own adaptive density control (scene/gaussian_model.py):
`densify_and_clone` (:448-459), `densify_and_split` (:420-446) and the prune of `densify_and_prune` (:461-474), run
on CPU from seeded parameters, Adam moments and densification statistics, plus `getNerfppNorm`
(scene/dataset_readers.py:50-71) on seeded camera infos.

Run like make_golden_surgery.py (CPU; `.cuda()` / device="cuda" are neutralised, the pose group is dropped because
the reference's optimizer surgery cannot index it).  `torch.normal` inside the reference module draws from a
generator seeded with SPLIT_SEED, so the split samples are reproducible; tests/test_densify_cpu.py hands the mirror a
generator with the same seed.

    python oracle/make_golden_densify.py <path to the InstantSplat checkout>
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
SPLIT_SEED = 1234


class _TorchNoCuda:
    """The torch module without device="cuda"; torch.normal draws from `gen` when it is set."""
    gen = None

    def __getattr__(self, name):
        obj = getattr(torch, name)
        if callable(obj) and not isinstance(obj, type):
            def call(*a, **k):
                if k.get("device") == "cuda":
                    k.pop("device")
                if name == "normal" and _TorchNoCuda.gen is not None:
                    k["generator"] = _TorchNoCuda.gen
                return obj(*a, **k)
            return call
        return obj


import scene.gaussian_model as ref_gm  # noqa: E402
import scene.dataset_readers as ref_dr  # noqa: E402
import utils.general_utils as ref_gu  # noqa: E402

ref_gm.torch = _TorchNoCuda()
ref_gu.torch = _TorchNoCuda()
from instantsplat_b200.model import optimization_defaults  # noqa: E402
from instantsplat_b200.scenes import surface_scene  # noqa: E402

KEYS = (("_xyz", "xyz"), ("_features_dc", "f_dc"), ("_features_rest", "f_rest"), ("_opacity", "opacity"),
        ("_scaling", "scaling"), ("_rotation", "rotation"))
# (tag, clone and split, max_screen_size)
CASES = (("prune", False, 20), ("prune_nosize", False, None), ("cs", True, 20), ("cs_nosize", True, None))
MAX_GRAD, MIN_OPACITY, EXTENT = 0.0002, 0.05, 1.5


def inputs():
    """Seeded parameters, Adam moments and statistics, shared by every case."""
    sc = surface_scene(300, 2, 32, 32, seed=21, sh_degree=3)
    g = torch.Generator().manual_seed(7)
    P = sc.P
    prm = {k: v.clone() for k, v in sc.params.items()}
    prm["opacity"] = torch.randn(P, 1, generator=g) * 2.0 - 1.0             # some below MIN_OPACITY
    prm["scaling"] = torch.log(0.03 * torch.rand(P, 3, generator=g) + 1e-3)   # around percent_dense * EXTENT
    prm["rotation"] = torch.randn(P, 4, generator=g)                        # unique rows, unnormalised
    d = dict(ppl0=(1.0 + torch.rand(P, 1, generator=g)), poses0=sc.poses.clone())
    for _, key in KEYS:
        d["m_" + key] = torch.randn(prm[key].shape, generator=g) * 1e-3
        d["v_" + key] = torch.rand(prm[key].shape, generator=g) * 1e-6
        d["init_" + key] = prm[key]
    denom = torch.randint(0, 5, (P, 1), generator=g).float()                 # zeros give NaN -> 0
    d["denom"] = denom
    d["grad_accum"] = denom * torch.rand(P, 1, generator=g) * 4e-4
    d["max_radii2D"] = torch.rand(P, generator=g) * 40.0
    return d


def run_case(d, clone_and_split, max_screen_size):
    m = ref_gm.GaussianModel(3)
    for attr, key in KEYS:
        setattr(m, attr, torch.nn.Parameter(d["init_" + key].clone().requires_grad_(True)))
    m.P = d["poses0"].clone().requires_grad_(True)
    m.spatial_lr_scale = 1.0
    m.training_setup_pp(optimization_defaults(iterations=1000), d["ppl0"].clone())
    assert m.optimizer.param_groups[-1]["name"] == "pose"
    m.optimizer.param_groups.pop()
    for attr, key in KEYS:
        m.optimizer.state[getattr(m, attr)] = dict(step=torch.tensor(3.0), exp_avg=d["m_" + key].clone(),
                                                   exp_avg_sq=d["v_" + key].clone())
    m.xyz_gradient_accum = d["grad_accum"].clone()
    m.denom = d["denom"].clone()
    m.max_radii2D = d["max_radii2D"].clone()
    masks = []
    prune_points = m.prune_points
    m.prune_points = lambda mask: (masks.append(mask.clone()), prune_points(mask))[1]
    out = {}
    if clone_and_split:
        grads = m.xyz_gradient_accum / m.denom
        grads[grads.isnan()] = 0.0
        _TorchNoCuda.gen = torch.Generator().manual_seed(SPLIT_SEED)
        n0 = m._xyz.shape[0]
        m.densify_and_clone(grads, MAX_GRAD, EXTENT)
        out["n_clone"] = np.int64(m._xyz.shape[0] - n0)
        m.densify_and_split(grads, MAX_GRAD, EXTENT)
        _TorchNoCuda.gen = None
        out["split_mask"] = masks[-1][:n0 + int(out["n_clone"])].numpy()
    m.densify_and_prune(MAX_GRAD, MIN_OPACITY, EXTENT, max_screen_size)      # InstantSplat's body: the prune
    out["prune_mask"] = masks[-1].numpy()
    for attr, key in KEYS:
        p = getattr(m, attr)
        st = m.optimizer.state[p]
        out["p_" + key] = p.detach().numpy().copy()
        out["m_" + key] = st["exp_avg"].numpy().copy()
        out["v_" + key] = st["exp_avg_sq"].numpy().copy()
    out["grad_accum"] = m.xyz_gradient_accum.numpy().copy()
    out["denom"] = m.denom.numpy().copy()
    out["max_radii2D"] = m.max_radii2D.numpy().copy()
    # every new row copies its source's rotation (unique random rows): recover the row map and the per-point
    # learning-rate multipliers a caller must carry along (the reference leaves per_point_lr unchanged)
    rot0 = d["init_rotation"]
    eq = (m._rotation.detach()[:, None, :] == rot0[None, :, :]).all(-1)
    assert bool((eq.sum(1) == 1).all())
    src = eq.float().argmax(1)
    out["src"] = src.numpy()
    out["ppl"] = d["ppl0"][src].numpy()
    out["P"] = np.int64(m._xyz.shape[0])
    return out


def cameras():
    """Seeded camera infos of the 3DGS convention (R: camera-to-world rotation, T: world-to-camera translation)."""
    g = np.random.default_rng(5)
    infos = []
    for i in range(6):
        q = g.normal(size=4)
        q /= np.linalg.norm(q)
        w, x, y, z = q
        Rw2c = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                         [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                         [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
        T = g.normal(size=3) * 2.0
        infos.append(ref_dr.CameraInfo(uid=i, R=Rw2c.T, T=T, FovY=1.0, FovX=1.0, image=None, image_path="",
                                       image_name="", width=32, height=32))
    poses7 = np.array([[*ref_q(c.R.T), *c.T] for c in infos])
    return poses7, float(ref_dr.getNerfppNorm(infos)["radius"])


def ref_q(R):
    """Quaternion (w, x, y, z) of a rotation matrix (the reference's utils/pose_utils.rotation2quad)."""
    from utils.pose_utils import rotation2quad
    return rotation2quad(torch.tensor(R[None], dtype=torch.float64))[0].numpy()


def main():
    d = inputs()
    out = {k: v.numpy() for k, v in d.items()}
    out.update(max_grad=np.float64(MAX_GRAD), min_opacity=np.float64(MIN_OPACITY), extent=np.float64(EXTENT),
               split_seed=np.int64(SPLIT_SEED))
    for tag, cs, size in CASES:
        for k, v in run_case(d, cs, size).items():
            out[f"{tag}_{k}"] = v
    out["cam_poses7"], out["cam_radius"] = cameras()
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "densify.npz"), **out)
    print("wrote tests/golden/densify.npz:", {tag: int(out[f"{tag}_P"]) for tag, _, _ in CASES},
          {tag: int(out[f"{tag}_n_clone"]) for tag, cs, _ in CASES if cs})


if __name__ == "__main__":
    main()
