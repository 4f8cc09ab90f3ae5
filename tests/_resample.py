"""A numpy restatement of Pillow's two integer resampling passes (libImaging Resample.c, 8 bits per channel), fed
resample.coefficients' tables, and the grid of size pairs the resize is tested on."""
import numpy as np

from instantsplat_b200 import resample

# (W, H) -> (W', H'): loaded_size at -r 2 / 4 / 8 of odd sizes, at -r -1 of 1601 and 1920 wide, a numeric -r that
# upscales, one-axis changes, 1-pixel outputs and 4032 x 3024 at -r -1
GRID = [((37, 23), (18, 12)), ((37, 23), (9, 6)), ((101, 75), (13, 9)), ((1601, 5), (1600, 4)), ((1601, 5), (1599, 4)),
        ((1920, 1080), (1600, 900)), ((40, 24), (60, 36)), ((33, 17), (33, 9)), ((33, 17), (20, 17)),
        ((9, 7), (1, 1)), ((9, 7), (3, 1)), ((9, 7), (5, 3)), ((5, 1), (2, 1))]
BIG = ((4032, 3024), (1600, 1200))


def _axis(a: np.ndarray, axis: int, n_out: int) -> np.ndarray:
    n_in = a.shape[axis]
    if n_in == n_out:
        return a
    bounds, coefs = resample.coefficients(n_in, n_out)
    k = np.arange(coefs.shape[1])
    idx = np.minimum(bounds[:, :1] + k, n_in - 1)                       # [out, ksize]; coefs are 0 past each count
    w = np.where(k < bounds[:, 1:], coefs, 0).astype(np.int64)
    taps = np.take(a.astype(np.int64), idx, axis=axis)                    # [..., out, ksize, ...]
    taps = np.moveaxis(taps, (axis, axis + 1), (-2, -1))
    acc = (1 << 21) + (taps * w).sum(-1)
    return np.moveaxis(np.clip(acc >> 22, 0, 255).astype(np.uint8), -1, axis)


def resize(img: np.ndarray, size) -> np.ndarray:
    """Image.fromarray(img).resize(size) for uint8 [H, W, 3] img, size = (width, height): the horizontal pass, then
    the vertical one on its u8 result."""
    return _axis(_axis(img, 1, int(size[0])), 0, int(size[1]))


def image(W: int, H: int, seed: int) -> np.ndarray:
    """A seeded uint8 [H, W, 3] test image: smooth gradients with noise and saturated patches, so that the bicubic
    overshoot clamps at 0 and 255."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W]
    base = 127.5 + 127.5 * np.sin(x[..., None] * np.array([0.05, 0.11, 0.3]) + y[..., None] * np.array([0.07, 0.2, 0.013]))
    img = base + rng.normal(0, 40, (H, W, 3))
    img[(x // 5 + y // 3) % 7 == 0] = 255
    img[(x // 3 + y // 5) % 11 == 0] = 0
    return np.clip(img, 0, 255).astype(np.uint8)
