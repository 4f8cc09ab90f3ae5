import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


def pytest_sessionfinish(session, exitstatus):
    """Parity numbers recorded by the GPU tests (tests/_parity.py REPORT) -> gpurun_out/parity_r02.json."""
    try:
        import json
        import _parity
        if not _parity.REPORT:
            return
        import torch
        out = os.path.join(ROOT, "gpurun_out")
        os.makedirs(out, exist_ok=True)
        doc = {"tolerances": {"image_max_abs": _parity.IMG_TOL, "grad_rel": _parity.GRAD_TOL,
                              "flip_budget": "max(2, 5e-5 * pixels compared), every such pixel oracle-flagged"},
               "device": torch.cuda.get_device_name(0) if torch.cuda.is_available() else None,
               "exit_status": int(exitstatus), "cases": _parity.REPORT}
        with open(os.path.join(out, "parity_r02.json"), "w") as f:
            json.dump(doc, f, indent=1)
    except Exception as e:   # never fail the session over the report
        print("parity report not written:", e)
