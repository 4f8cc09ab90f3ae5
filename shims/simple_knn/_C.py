"""`simple_knn._C` drop-in so scene/gaussian_model.py:20 imports and :156 runs."""
from instantsplat_b200.knn import distCUDA2  # noqa: F401
