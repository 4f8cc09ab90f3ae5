"""Test-only stand-in for the `plyfile` PyPI package (not installed in this image): lets
scene/gaussian_model.py be IMPORTED by tests/test_reference_shims_cpu.py.  Nothing on the tested path
reads or writes PLY files through it."""


class PlyData:
    def __init__(self, *a, **k):
        raise NotImplementedError("plyfile stub (tests only)")

    @staticmethod
    def read(*a, **k):
        raise NotImplementedError("plyfile stub (tests only)")


class PlyElement:
    @staticmethod
    def describe(*a, **k):
        raise NotImplementedError("plyfile stub (tests only)")
