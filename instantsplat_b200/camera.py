"""Host-side camera helpers (tiny, fp32 torch on CPU then moved by the caller)."""
import math

import torch


def projection_matrix(znear: float, zfar: float, fovx: float, fovy: float) -> torch.Tensor:
    """utils/graphics_utils.py:71-91 (NOT transposed; callers store P^T like
    scene/cameras.py:55)."""
    ty, tx = math.tan(fovy / 2), math.tan(fovx / 2)
    top, right = ty * znear, tx * znear
    P = torch.zeros(4, 4)
    P[0, 0] = 2.0 * znear / (2 * right)
    P[1, 1] = 2.0 * znear / (2 * top)
    P[3, 2] = 1.0
    P[2, 2] = zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    return P


class SimpleCamera:
    """The attributes `render()` reads from a viewpoint camera
    (gaussian_renderer/__init__.py:51-62)."""

    def __init__(self, width, height, fovx, fovy, device="cuda", znear=0.01, zfar=100.0):
        self.image_width, self.image_height = int(width), int(height)
        self.FoVx, self.FoVy = float(fovx), float(fovy)
        self.projection_matrix = projection_matrix(znear, zfar, fovx, fovy).t().contiguous().to(device)
        self.world_view_transform = torch.eye(4, device=device)
        self.full_proj_transform = self.projection_matrix
        self.camera_center = torch.zeros(3, device=device)
