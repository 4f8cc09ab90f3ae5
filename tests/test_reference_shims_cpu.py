"""CPU tests of this repo's drop-in interfaces against the reference (InstantSplat) on the CPU.
See tests/test_reference_loop.py for the GPU side.

1. `test_reference_loop_body_runs_on_the_shim_interfaces`: the train.py:140-211 loop body on CPU stand-ins with the
   shims' surface: the repo's GaussianModel mirror and the oracle reproduce exactly what the reference's own render(),
   GaussianModel and PerPointAdam computed on the same inputs (tests/_ref_loop_cpu.py, tests/golden/ref_loop.npz).
2. `test_no_edit_install_hook`: with <repo>/shims on PYTHONPATH (sitecustomize -> instantsplat_b200/hooks.py) an
   unchanged checkout with the reference's package layout imports `scene.per_point_adam.PerPointAdam` and
   `gaussian_renderer.render` from this repo.
"""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_loop_body_runs_on_the_shim_interfaces(tmp_path):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "_ref_loop_cpu.py")], capture_output=True,
                         text=True, timeout=600, cwd=str(tmp_path))
    assert out.returncode == 0 and "REF_LOOP_OK" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]


# The module-level imports the hook has to intercept, laid out like the reference tree: scene/gaussian_model.py:26
# imports the optimizer from its own package, train.py:24 imports render and network_gui from gaussian_renderer,
# whose __init__ imports GaussianModel.  The bodies are placeholders: only the import wiring is under test.
_CHECKOUT = {
    "scene/__init__.py": "",
    "scene/per_point_adam.py": "class PerPointAdam:\n    pass\n",
    "scene/gaussian_model.py": "from scene.per_point_adam import PerPointAdam\n\n\nclass GaussianModel:\n    pass\n",
    "gaussian_renderer/__init__.py": ("from scene.gaussian_model import GaussianModel\n\n\n"
                                      "def render(viewpoint_camera, pc, pipe, bg_color, scaling_modifier=1.0, "
                                      "override_color=None, camera_pose=None):\n    raise NotImplementedError\n"),
    "gaussian_renderer/network_gui.py": "",
}

_HOOK_PROBE = r'''
import sys
assert type(sys.meta_path[0]).__name__ == "GsbFinder", sys.meta_path
import scene.gaussian_model as g
import gaussian_renderer as gr
print("OPT", g.PerPointAdam.__module__)
from gaussian_renderer import render, network_gui            # what train.py:24 does
ref_body = getattr(gr, "reference_render", gr.render)
print("RENDER", render.__module__, ref_body.__module__, network_gui.__name__, hasattr(gr, "GaussianModel"))
'''


@pytest.mark.parametrize("fused", ["1", "0"])
def test_no_edit_install_hook(fused, tmp_path):
    checkout = tmp_path / "checkout"
    for rel, src in _CHECKOUT.items():
        (checkout / rel).parent.mkdir(parents=True, exist_ok=True)
        (checkout / rel).write_text(src)
    env = dict(os.environ, GSB_FUSED_RENDER=fused,
               PYTHONPATH=os.pathsep.join([os.path.join(ROOT, "shims"), ROOT, str(checkout)]))
    out = subprocess.run([sys.executable, "-c", _HOOK_PROBE], capture_output=True, text=True, timeout=300,
                         cwd=str(tmp_path), env=env)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
    assert "OPT instantsplat_b200.per_point_adam" in out.stdout
    if fused == "1":
        assert "RENDER instantsplat_b200.renderer gaussian_renderer gaussian_renderer.network_gui True" in out.stdout, out.stdout
    else:
        assert "RENDER gaussian_renderer gaussian_renderer gaussian_renderer.network_gui True" in out.stdout, out.stdout
