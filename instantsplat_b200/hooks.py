"""No-edit installation into an unchanged InstantSplat checkout (SURVEY.md section 8b, boundaries B1 / B4).

The native packages (`diff_gaussian_rasterization`, `fused_ssim`, `simple_knn`) are replaced simply by putting
<repo>/shims on PYTHONPATH.  Two replacements live INSIDE the reference's own packages and cannot be shadowed by a
path entry:

  * `scene.per_point_adam`  (imported by scene/gaussian_model.py:26) -> the fused sm_90a optimizer;
  * `gaussian_renderer.render` (imported by train.py:24, render.py:27) -> the fused render body.

`install()` registers a meta-path finder that serves `scene.per_point_adam` from `instantsplat_b200.per_point_adam`
and, when GSB_FUSED_RENDER=1 (default), swaps `gaussian_renderer.render` for `instantsplat_b200.renderer.render` right
after the reference's module has been executed (its other exports -- `network_gui`, `GaussianModel` -- stay).
<repo>/shims/sitecustomize.py calls it at interpreter start-up, so

    PYTHONPATH=<repo>/shims:<repo> python train.py -s <scene> -m <out> --pp_optimizer --optim_pose ...

runs the unchanged train.py on the H100 kernels.  GSB_HOOKS=0 disables the hook, GSB_FUSED_RENDER=0 keeps the
reference's own render() body (PyTorch pose pre-transform -> GaussianRasterizer shim).
"""
import importlib
import importlib.abc
import importlib.util
import os
import sys

_TARGET_OPT = "scene.per_point_adam"
_TARGET_RENDER = "gaussian_renderer"


class _AliasLoader(importlib.abc.Loader):
    def __init__(self, real_name):
        self.real_name = real_name

    def create_module(self, spec):
        return importlib.import_module(self.real_name)

    def exec_module(self, module):
        pass


class _PatchRenderLoader(importlib.abc.Loader):
    def __init__(self, inner):
        self.inner = inner

    def create_module(self, spec):
        return self.inner.create_module(spec)

    def exec_module(self, module):
        self.inner.exec_module(module)
        from instantsplat_b200.renderer import render as fused_render
        module.reference_render = getattr(module, "render", None)
        module.render = fused_render


class GsbFinder(importlib.abc.MetaPathFinder):
    def find_spec(self, fullname, path, target=None):
        if fullname == _TARGET_OPT:
            return importlib.util.spec_from_loader(fullname, _AliasLoader("instantsplat_b200.per_point_adam"))
        if fullname == _TARGET_RENDER and os.environ.get("GSB_FUSED_RENDER", "1") != "0":
            for f in sys.meta_path:
                if f is self or not hasattr(f, "find_spec"):
                    continue
                spec = f.find_spec(fullname, path, target)
                if spec is not None and spec.loader is not None:
                    spec.loader = _PatchRenderLoader(spec.loader)
                    return spec
        return None


_installed = None


def install():
    global _installed
    if _installed is None and os.environ.get("GSB_HOOKS", "1") != "0":
        _installed = GsbFinder()
        sys.meta_path.insert(0, _installed)
    return _installed


def uninstall():
    global _installed
    if _installed is not None:
        try:
            sys.meta_path.remove(_installed)
        except ValueError:
            pass
        _installed = None
