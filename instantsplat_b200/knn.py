"""`simple_knn._C.distCUDA2` replacement (scene/gaussian_model.py:20,156; SURVEY.md section 8 row
f1: runs once at initialisation, not on the per-iteration path).

distCUDA2(points [P,3]) -> [P] mean squared distance to the 3 nearest neighbours, computed exactly by the grid-hash
kernel in libgsb200.so (csrc/gs_knn.cu).  CPU tensors are refused, except tiny clouds (<= 20 000 points, used by the
CPU tests of the import shims) which take a brute-force torch path."""
import torch


def distCUDA2(points: torch.Tensor) -> torch.Tensor:
    pts = points.float().contiguous()
    n = pts.shape[0]
    if not pts.is_cuda:
        if n > 20000:
            raise RuntimeError("distCUDA2: CPU input is supported for small test clouds only")
        d = torch.cdist(pts, pts)
        d2 = (d * d).topk(min(4, n), dim=1, largest=False).values[:, 1:]
        return d2.sum(dim=1) / 3.0
    from . import _lib
    L = _lib.lib()
    with torch.cuda.device(pts.device):
        out = torch.empty(n, dtype=torch.float32, device=pts.device)
        nbytes = L.gsb_knn_scratch_bytes(n)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=pts.device)
        _lib.check(L.gsb_knn_mean_dist2(n, pts.data_ptr(), out.data_ptr(), scratch.data_ptr(), nbytes,
                                        _lib.stream_ptr()), "gsb_knn_mean_dist2")
    return out
