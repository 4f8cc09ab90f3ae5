"""Picked up automatically by Python when <repo>/shims is on PYTHONPATH: installs the import hook that swaps the
reference's in-package pieces (`scene.per_point_adam`, `gaussian_renderer.render`) for the fused ones without editing
the reference (instantsplat_b200/hooks.py).  The hook module is loaded by file path so that start-up does not import
torch; the heavy imports happen only when the reference actually imports the hooked modules."""
import importlib.util
import os
import sys

_repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if _repo not in sys.path:
    sys.path.append(_repo)
try:
    _spec = importlib.util.spec_from_file_location("instantsplat_b200_hooks",
                                                   os.path.join(_repo, "instantsplat_b200", "hooks.py"))
    _hooks = importlib.util.module_from_spec(_spec)
    _spec.loader.exec_module(_hooks)
    sys.modules["instantsplat_b200_hooks"] = _hooks
    _hooks.install()
except Exception:      # never break an interpreter that merely has shims/ on its path
    pass
