"""Generate tests/golden/png.npz: two crops of run_infer.sh's input photos (assets/sora/Santorini/images/frame_00.jpg
and assets/sora/Art/images/0.jpg of the InstantSplat checkout), decoded to 8-bit RGB, and what Pillow makes of each
when save_image writes it: the per-row filter types of its PNG and its file size.

The crops are 512 x 384 from the image centre, rounded to even offsets.  The filter types are read from the
decompressed IDAT of Image.fromarray(crop).save(...) (the first byte of each 3W + 1 byte scanline).  The Pillow and
zlib-ng versions that wrote the files are stored beside them, since the sizes depend on them.

    python oracle/make_golden_png.py <path to the InstantSplat checkout>
"""
import io
import os
import sys
import zlib

import numpy as np
import PIL
from PIL import Image, features

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if len(sys.argv) != 2:
    sys.exit(__doc__)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from _png import idat  # noqa: E402

PHOTOS = {"santorini": "assets/sora/Santorini/images/frame_00.jpg", "art": "assets/sora/Art/images/0.jpg"}
CROP_W, CROP_H = 512, 384


def main() -> None:
    out = {"pillow_version": np.array(PIL.__version__), "zlib_ng_version": np.array(str(features.version("zlib_ng")))}
    for name, rel in PHOTOS.items():
        img = np.array(Image.open(os.path.join(sys.argv[1], rel)).convert("RGB"))
        H, W, _ = img.shape
        y0, x0 = (H - CROP_H) // 4 * 2, (W - CROP_W) // 4 * 2
        crop = np.ascontiguousarray(img[y0:y0 + CROP_H, x0:x0 + CROP_W])
        buf = io.BytesIO()
        Image.fromarray(crop).save(buf, "PNG")
        raw = zlib.decompress(idat(buf.getvalue()))
        stride = 3 * CROP_W + 1
        out[f"{name}_crop"] = crop
        out[f"{name}_filters"] = np.frombuffer(raw, np.uint8)[::stride].copy()
        out[f"{name}_pil_bytes"] = np.array(len(buf.getvalue()), np.int64)
        print(name, crop.shape, len(buf.getvalue()), np.bincount(out[f"{name}_filters"], minlength=5))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "png.npz"), **out)


if __name__ == "__main__":
    main()
