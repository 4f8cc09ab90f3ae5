"""Generate tests/golden/ref_loop.npz by running the REFERENCE's own Python for the hot path on the CPU:
gaussian_renderer.render() (gaussian_renderer/__init__.py:23-144), GaussianModel.training_setup_pp /
update_learning_rate / oneupSHdegree / create_from_pcd (scene/gaussian_model.py), PerPointAdam
(scene/per_point_adam.py), l1_loss (utils/loss_utils.py), get_tensor_from_camera (utils/pose_utils.py) and the loop
body of train.py:140-211, with the three native packages it imports replaced by tests/cpu_standins.

Needs an InstantSplat checkout (NVlabs/InstantSplat); the vectors it writes are committed and
tests/_ref_loop_cpu.py checks the repository's mirror and the oracle against them.

    python oracle/make_golden_ref_loop.py <path to the InstantSplat checkout>
"""
import importlib.abc
import importlib.util
import os
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import _ref_loop_cpu as T  # noqa: E402  (scene, cameras, loop body; puts the stand-ins on sys.path)


class _Stub(importlib.abc.MetaPathFinder, importlib.abc.Loader):
    """Empty modules for third-party packages the reference imports at module load but the path never calls."""
    NAMES = {"matplotlib"}

    def find_spec(self, name, path, target=None):
        if name.split(".")[0] in self.NAMES:
            return importlib.util.spec_from_loader(name, self, is_package=True)

    def create_module(self, spec):
        m = types.ModuleType(spec.name)
        m.__path__ = []
        return m

    def exec_module(self, m):
        pass


class _TorchNoCuda:
    """The reference hard-codes device="cuda"; on this CPU-only run the argument is dropped."""

    def __getattr__(self, name):
        obj = getattr(torch, name)
        if callable(obj) and not isinstance(obj, type):
            def call(*a, **k):
                if k.get("device") == "cuda":
                    k.pop("device")
                return obj(*a, **k)
            return call
        return obj


def main(ref):
    sys.path.append(ref)               # reference LAST: its `utils`/`scene` are found, the stand-ins shadow native pkgs
    sys.meta_path.insert(0, _Stub())
    torch.Tensor.cuda = lambda self, *a, **k: self
    import gaussian_renderer as ref_gr
    import scene.gaussian_model as ref_gm
    from utils.loss_utils import l1_loss as ref_l1
    from utils.pose_utils import get_tensor_from_camera
    ref_gr.torch = _TorchNoCuda()
    ref_gm.torch = _TorchNoCuda()

    model = ref_gm.GaussianModel(3)
    T.fill(model)
    model.training_setup_pp(T.opt_args, T.sc.per_point_lr.clone())
    assert type(model.optimizer).__module__ == "scene.per_point_adam"
    losses = T.loop(model, ref_gr.render, ref_l1, T.fused_ssim)
    tfc = np.stack([get_tensor_from_camera(T.O.pose_to_w2c(T.sc.poses[v])).numpy() for v in range(3)])
    pts, cols = T.pcd()
    m2 = ref_gm.GaussianModel(3)
    m2.create_from_pcd(types.SimpleNamespace(points=pts, colors=cols), 1.5)
    out = os.path.join(ROOT, "tests", "golden", "ref_loop.npz")
    np.savez(out, n_it=T.N_IT, views=np.array(T.views), losses=np.array(losses),
             xyz=model._xyz.detach().numpy(), poses=model.P.detach().numpy(), sh_degree=model.active_sh_degree,
             tensor_from_camera=tfc, **{"pcd" + a: getattr(m2, a).detach().numpy() for a in T.PCD_ATTRS})
    print("wrote", out, "losses", [round(x, 7) for x in losses])


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])
