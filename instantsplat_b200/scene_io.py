"""On-disk formats either side of the hot path (SURVEY.md section 8 row f3) -- host-side, numpy only.

What the reference's training stage reads and writes, so a scene produced here can drive an unchanged
`train.py` and its outputs can be loaded back:

* `sparse_<n>/0/cameras.txt` (PINHOLE only) and `images.txt` (two lines per image), as parsed by
  scene/colmap_loader.py:159-182,248-275 and written by
  utils/sfm_utils.py:202-315;
* `points3D.ply`: x,y,z f4 | nx,ny,nz f4 | red,green,blue u1 (scene/dataset_readers.py:315-369);
* `confidence_dsp.npy` [P,1] (train.py:63-96);
* the trained model `point_cloud.ply`: x,y,z,nx,ny,nz,f_dc_0..2,f_rest_0..44,opacity,scale_0..2,rot_0..3, all f4
  (f_rest_0..3(M-1)-1 at SH degree D, M = (D+1)^2: none at degree 0), SH stored channel-major (scene/gaussian_model.py:247-278), optionally followed by Mip-Splatting's `filter_3D` f4;
* `pose_optimized.npy` [n,4,4] world-to-camera matrices ordered by COLMAP image id
  (train.py:46-60).

PLY files are written/read directly (binary little endian) -- `plyfile` is not a dependency.
"""
from __future__ import annotations

import os
from typing import Dict, List, Tuple

import numpy as np


# ----------------------------------------------------------------------------------------------
# quaternion <-> rotation (COLMAP convention: qvec = (w, x, y, z) of the world-to-camera rotation)
# ----------------------------------------------------------------------------------------------
def qvec2rotmat(q: np.ndarray) -> np.ndarray:
    w, x, y, z = q
    return np.array([[1 - 2 * y * y - 2 * z * z, 2 * x * y - 2 * w * z, 2 * z * x + 2 * w * y],
                     [2 * x * y + 2 * w * z, 1 - 2 * x * x - 2 * z * z, 2 * y * z - 2 * w * x],
                     [2 * z * x - 2 * w * y, 2 * y * z + 2 * w * x, 1 - 2 * x * x - 2 * y * y]])


def pose7_to_matrix(pose: np.ndarray) -> np.ndarray:
    """[qw,qx,qy,qz,tx,ty,tz] -> 4x4 world-to-camera; the quaternion is normalised first, like
    get_camera_from_tensor (utils/pose_utils.py:57-84)."""
    q = np.asarray(pose[:4], dtype=np.float64)
    q = q / np.linalg.norm(q)
    M = np.eye(4)
    M[:3, :3] = qvec2rotmat(q)
    M[:3, 3] = pose[4:7]
    return M


# ----------------------------------------------------------------------------------------------
# COLMAP text model
# ----------------------------------------------------------------------------------------------
def write_colmap_text(folder: str, width: int, height: int, fx: float, fy: float, poses: np.ndarray,
                      image_names: List[str], cx: float = None, cy: float = None) -> None:
    """One shared PINHOLE camera, one image per pose row [qw,qx,qy,qz,tx,ty,tz] (world-to-camera)."""
    os.makedirs(folder, exist_ok=True)
    cx = width / 2.0 if cx is None else cx
    cy = height / 2.0 if cy is None else cy
    with open(os.path.join(folder, "cameras.txt"), "w") as f:
        f.write("# Camera list with one line of data per camera:\n#   CAMERA_ID, MODEL, WIDTH, HEIGHT, PARAMS[]\n")
        f.write(f"# Number of cameras: {len(image_names)}\n")
        for i in range(len(image_names)):
            f.write(f"{i + 1} PINHOLE {width} {height} {fx:.10g} {fy:.10g} {cx:.10g} {cy:.10g}\n")
    with open(os.path.join(folder, "images.txt"), "w") as f:
        f.write("# Image list with two lines of data per image:\n#   IMAGE_ID, QW, QX, QY, QZ, TX, TY, TZ, CAMERA_ID, NAME\n"
                "#   POINTS2D[] as (X, Y, POINT3D_ID)\n")
        for i, (p, name) in enumerate(zip(poses, image_names)):
            q = np.asarray(p[:4], dtype=np.float64)
            q = q / np.linalg.norm(q)
            vals = " ".join(f"{v:.10g}" for v in list(q) + list(p[4:7]))
            f.write(f"{i + 1} {vals} {i + 1} {name}\n\n")


def read_colmap_text(folder: str, models: Tuple[str, ...] = ("PINHOLE",)) -> Tuple[Dict[int, dict], Dict[int, dict]]:
    """Returns (cameras, images) keyed by id; same fields the reference's readers expose.  models: the camera models
    accepted (the params are returned as listed: PINHOLE fx fy cx cy, SIMPLE_PINHOLE f cx cy)."""
    cameras, images = {}, {}
    with open(os.path.join(folder, "cameras.txt")) as f:
        for line in f:
            line = line.strip()
            if not line or line[0] == "#":
                continue
            e = line.split()
            if e[1] not in models:
                raise ValueError(f"only {' / '.join(models)} cameras are supported (as in the reference), got {e[1]}")
            cameras[int(e[0])] = dict(id=int(e[0]), model=e[1], width=int(e[2]), height=int(e[3]),
                                      params=np.array(list(map(float, e[4:]))))
    with open(os.path.join(folder, "images.txt")) as f:
        lines = f.readlines()
    i = 0
    while i < len(lines):
        line = lines[i].strip()
        i += 1
        if not line or line[0] == "#":
            continue
        e = line.split()
        images[int(e[0])] = dict(id=int(e[0]), qvec=np.array(list(map(float, e[1:5]))),
                                 tvec=np.array(list(map(float, e[5:8]))), camera_id=int(e[8]), name=e[9])
        i += 1                                     # the POINTS2D line
    return cameras, images


# ----------------------------------------------------------------------------------------------
# COLMAP binary images.bin (what read_colmap_gt_pose reads for the pose errors)
# ----------------------------------------------------------------------------------------------
def read_colmap_images_bin(path: str) -> Dict[int, dict]:
    """COLMAP's images.bin keyed by image id, the records of scene/colmap_loader.py's read_extrinsics_binary: id,
    qvec (w, x, y, z) and tvec as fp64 arrays, camera_id, name, xys [n, 2] fp64 and point3D_ids [n] int64.  Layout
    (little endian): u64 count, then per image i32 id, 7 f64, i32 camera id, a NUL-terminated name, u64 n and n
    (f64 x, f64 y, i64 point id)."""
    import struct
    images = {}
    with open(path, "rb") as f:
        data = f.read()
    off = 0

    def take(fmt: str):
        nonlocal off
        size = struct.calcsize("<" + fmt)
        if off + size > len(data):
            raise ValueError(f"{path}: truncated COLMAP images.bin")
        out = struct.unpack_from("<" + fmt, data, off)
        off += size
        return out

    (count,) = take("Q")
    for _ in range(count):
        rec = take("idddddddi")
        end = data.find(b"\x00", off)
        if end < 0:
            raise ValueError(f"{path}: truncated COLMAP images.bin (image name)")
        name = data[off:end].decode("utf-8")
        off = end + 1
        (n,) = take("Q")
        pts = np.frombuffer(data, dtype=np.dtype([("x", "<f8"), ("y", "<f8"), ("id", "<i8")]), count=n, offset=off) \
            if n else np.zeros(0, dtype=[("x", "<f8"), ("y", "<f8"), ("id", "<i8")])
        off += 24 * n
        if off > len(data):
            raise ValueError(f"{path}: truncated COLMAP images.bin (points)")
        images[rec[0]] = dict(id=rec[0], qvec=np.array(rec[1:5]), tvec=np.array(rec[5:8]), camera_id=rec[8], name=name,
                              xys=np.stack([pts["x"], pts["y"]], axis=1).astype(np.float64),
                              point3D_ids=pts["id"].astype(np.int64))
    return images


def write_colmap_images_bin(path: str, poses: np.ndarray, image_names: List[str], image_ids: List[int] = None,
                            camera_ids: List[int] = None, points2d: List[np.ndarray] = None) -> None:
    """The inverse of read_colmap_images_bin: one record per pose row [qw,qx,qy,qz,tx,ty,tz] (world-to-camera, written
    as given).  image_ids / camera_ids default to 1..n; points2d: per image an [n, 3] array of (x, y, point id)."""
    import struct
    n = len(image_names)
    ids = list(range(1, n + 1)) if image_ids is None else list(image_ids)
    cids = list(range(1, n + 1)) if camera_ids is None else list(camera_ids)
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", n))
        for k in range(n):
            p = np.asarray(poses[k], np.float64)
            f.write(struct.pack("<idddddddi", ids[k], *p[:7].tolist(), cids[k]))
            f.write(image_names[k].encode("utf-8") + b"\x00")
            pts = np.zeros((0, 3)) if points2d is None else np.asarray(points2d[k]).reshape(-1, 3)
            f.write(struct.pack("<Q", pts.shape[0]))
            for x, y, pid in pts:
                f.write(struct.pack("<ddq", float(x), float(y), int(pid)))


def read_colmap_gt_pose(source_path: str) -> np.ndarray:
    """utils/sfm_utils.py read_colmap_gt_pose: source/sparse/0/images.bin sorted by image name, each record as
    [qvec2rotmat(q)^T | t] in np.eye(4): [N, 4, 4] fp64 (the matrix metrics.py aligns; its rotation block is the
    transposed world-to-camera rotation, as in the reference)."""
    path = os.path.join(source_path, "sparse", "0", "images.bin")
    if not os.path.isfile(path):
        raise FileNotFoundError(f"{path} not found")
    recs = sorted(read_colmap_images_bin(path).values(), key=lambda r: r["name"])
    out = []
    for r in recs:
        pose = np.eye(4, 4)
        pose[:3, :3] = np.transpose(qvec2rotmat(r["qvec"]))
        pose[:3, 3] = np.array(r["tvec"])
        out.append(pose)
    return np.array(out)


def split_train_test(items, n_views: int):
    """utils/sfm_utils.py split_train_test (llffhold is unused there): 12 test items at np.linspace(1, N - 2, 12)
    (int), the rest thinned to n_views training items at np.linspace(0, n_rest - 1, n_views) (int).  Returns
    (train, test) lists."""
    test_idx = np.linspace(1, len(items) - 2, num=12, dtype=int)
    train_idx = [i for i in range(len(items)) if i not in test_idx]
    sparse_idx = np.linspace(0, len(train_idx) - 1, num=n_views, dtype=int)
    train_idx = [train_idx[i] for i in sparse_idx]
    return [items[i] for i in train_idx], [items[i] for i in test_idx]


# ----------------------------------------------------------------------------------------------
# the cameras render.py renders: readColmapSceneInfo + loadCam
# ----------------------------------------------------------------------------------------------
class Views:
    """The cameras of one sparse_<n>/<k> folder, sorted by image_name: names [N] (image_name, the file name without
    its extension), w2c [N, 4, 4] fp64 world-to-camera matrices [qvec2rotmat(q) | t], images [N, H, W, 3] uint8 (the
    decoded files), width / height (the images'), fovx / fovy (focal2fov of the intrinsics), camera_ids [N] (each
    view's COLMAP camera id, intr.id: what readColmapCameras stores as the CameraInfo uid and train.py's save_pose
    looks up as colmap_id; None when not known)."""

    def __init__(self, names, w2c, images, width, height, fovx, fovy, camera_ids=None):
        self.names, self.w2c, self.images = list(names), w2c, images
        self.width, self.height, self.fovx, self.fovy = width, height, fovx, fovy
        self.camera_ids = None if camera_ids is None else [int(c) for c in camera_ids]

    def __len__(self) -> int:
        return len(self.names)


def loaded_size(width: int, height: int, resolution: int) -> Tuple[int, int]:
    """The size loadCam (utils/camera_utils.py) resizes a width x height image to at `-r resolution` and resolution
    scale 1."""
    if resolution in (1, 2, 4, 8):
        return round(width / (1.0 * resolution)), round(height / (1.0 * resolution))
    if resolution == -1:
        global_down = width / 1600 if width > 1600 else 1
    else:
        global_down = width / resolution
    scale = float(global_down) * 1.0
    return int(width / scale), int(height / scale)


def load_views(source_path: str, n_views: int, split: int = 0, resolution: int = 1, images: str = "images") -> Views:
    """render.py's cameras: readColmapSceneInfo (scene/dataset_readers.py:315-369) reads source/sparse_<n_views>/<split>
    ({0: the training views, 1: the test views of --eval}), cameras.txt (PINHOLE or SIMPLE_PINHOLE) and images.txt,
    opens source/<images>/<basename of the name> (`images`: train.py's -i, the folder name) and sorts the views by
    image_name; loadCam resizes each image to loaded_size(resolution) and divides by 255.

    Refused, with the reason: a resolution at which loadCam would resample an image (only sizes PIL's resize copies
    are kept), an image that is not 8-bit RGB (RGBA included: Camera's alpha mask is not implemented), and views
    whose image size or field of view differ (one PoseTracker renders them all)."""
    import math
    from PIL import Image
    folder = os.path.join(source_path, f"sparse_{n_views}", str(split))
    for f in ("cameras.txt", "images.txt"):
        if not os.path.isfile(os.path.join(folder, f)):
            raise FileNotFoundError(f"{os.path.join(folder, f)} not found")
    cams, imgs = read_colmap_text(folder, ("PINHOLE", "SIMPLE_PINHOLE"))
    if not imgs:
        raise ValueError(f"{folder}/images.txt lists no image")
    focal2fov = lambda f, pixels: 2 * math.atan(pixels / (2 * f))
    recs = []
    for extr in imgs.values():
        intr = cams[extr["camera_id"]]
        path = os.path.join(source_path, images, os.path.basename(extr["name"]))
        name = os.path.basename(path).split(".")[0]
        with Image.open(path) as im:
            if im.mode != "RGB":
                raise ValueError(f"{path}: mode {im.mode}; only 8-bit RGB images are supported (an alpha channel "
                                 "would be Camera's gt_alpha_mask, which is not implemented)")
            W, H = im.size
            if loaded_size(W, H, resolution) != (W, H):
                raise ValueError(f"{path}: -r {resolution} resizes {W}x{H} to {loaded_size(W, H, resolution)}; "
                                 "resampled images are not supported (use -r 1, or -r -1 up to 1600 pixels wide)")
            pixels = np.array(im)
        fx = float(intr["params"][0])
        fy = fx if intr["model"] == "SIMPLE_PINHOLE" else float(intr["params"][1])
        w2c = np.eye(4)
        w2c[:3, :3] = qvec2rotmat(extr["qvec"])
        w2c[:3, 3] = extr["tvec"]
        recs.append((name, w2c, pixels, (W, H, focal2fov(fx, intr["width"]), focal2fov(fy, intr["height"])), intr["id"]))
    recs.sort(key=lambda r: r[0])
    keys = {r[3] for r in recs}
    if len(keys) != 1:
        raise ValueError(f"{folder}: the cameras' intrinsics differ ({len(keys)} distinct image sizes and fields of "
                         "view); the views are rendered with one camera")
    W, H, fovx, fovy = keys.pop()
    return Views([r[0] for r in recs], np.stack([r[1] for r in recs]), np.stack([r[2] for r in recs]), W, H, fovx, fovy,
                 [r[4] for r in recs])


# ----------------------------------------------------------------------------------------------
# PLY (binary little endian, single 'vertex' element)
# ----------------------------------------------------------------------------------------------
_PLY_TYPES = {"f4": "float", "u1": "uchar", "f8": "double", "i4": "int"}
_PLY_REV = {"float": "f4", "float32": "f4", "uchar": "u1", "uint8": "u1", "double": "f8", "float64": "f8",
            "int": "i4", "int32": "i4"}


def _write_ply(path: str, fields: List[Tuple[str, str]], columns: List[np.ndarray]) -> None:
    n = columns[0].shape[0]
    dt = np.dtype([(name, "<" + t) for name, t in fields])
    arr = np.empty(n, dtype=dt)
    for (name, _), col in zip(fields, columns):
        arr[name] = col
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "wb") as f:
        hdr = ["ply", "format binary_little_endian 1.0", f"element vertex {n}"]
        hdr += [f"property {_PLY_TYPES[t]} {name}" for name, t in fields]
        hdr.append("end_header")
        f.write(("\n".join(hdr) + "\n").encode("ascii"))
        f.write(arr.tobytes())


def _read_ply(path: str) -> np.ndarray:
    with open(path, "rb") as f:
        if f.readline().strip() != b"ply":
            raise ValueError("not a PLY file")
        fmt = f.readline().split()
        if fmt[1] != b"binary_little_endian":
            raise ValueError("only binary_little_endian PLY is supported")
        n, fields = None, []
        while True:
            line = f.readline().strip()
            if line == b"end_header":
                break
            tok = line.split()
            if tok[:2] == [b"element", b"vertex"]:
                n = int(tok[2])
            elif tok[0] == b"property":
                fields.append((tok[2].decode(), "<" + _PLY_REV[tok[1].decode()]))
        data = np.frombuffer(f.read(n * np.dtype(fields).itemsize), dtype=np.dtype(fields), count=n)
    return data


def write_points3d_ply(path: str, xyz: np.ndarray, rgb_u8: np.ndarray, normals: np.ndarray = None) -> None:
    normals = np.zeros_like(xyz) if normals is None else normals
    fields = [("x", "f4"), ("y", "f4"), ("z", "f4"), ("nx", "f4"), ("ny", "f4"), ("nz", "f4"),
              ("red", "u1"), ("green", "u1"), ("blue", "u1")]
    cols = [xyz[:, 0], xyz[:, 1], xyz[:, 2], normals[:, 0], normals[:, 1], normals[:, 2],
            rgb_u8[:, 0], rgb_u8[:, 1], rgb_u8[:, 2]]
    _write_ply(path, fields, cols)


def read_points3d_ply(path: str):
    d = _read_ply(path)
    xyz = np.stack([d["x"], d["y"], d["z"]], axis=1)
    rgb = np.stack([d["red"], d["green"], d["blue"]], axis=1)
    nrm = np.stack([d["nx"], d["ny"], d["nz"]], axis=1) if "nx" in d.dtype.names else np.zeros_like(xyz)
    return xyz, rgb, nrm


def gaussian_ply_fields(n_rest: int = 45) -> List[str]:
    """construct_list_of_attributes (scene/gaussian_model.py:247-259)."""
    return (["x", "y", "z", "nx", "ny", "nz"] + [f"f_dc_{i}" for i in range(3)] + [f"f_rest_{i}" for i in range(n_rest)]
            + ["opacity"] + [f"scale_{i}" for i in range(3)] + [f"rot_{i}" for i in range(4)])


def save_gaussians_ply(path: str, xyz, f_dc, f_rest, opacity, scaling, rotation, filter_3D=None) -> None:
    """Model tensors -> point_cloud.ply; f_dc [P,1,3], f_rest [P,M-1,3] are stored channel-major
    (transpose(1,2).flatten(1)), raw (un-activated) opacity / scaling / rotation, zero normals.  filter_3D [P] or
    [P,1] (Mip-Splatting's 3D smoothing filter), when given, is the last property, as Mip-Splatting stores it."""
    xyz = np.asarray(xyz, np.float32)
    P = xyz.shape[0]
    dc = np.asarray(f_dc, np.float32).reshape(P, -1, 3).transpose(0, 2, 1).reshape(P, -1)
    rest = np.asarray(f_rest, np.float32).reshape(P, -1, 3).transpose(0, 2, 1).reshape(P, -1)
    attrs = np.concatenate([xyz, np.zeros_like(xyz), dc, rest, np.asarray(opacity, np.float32).reshape(P, 1),
                            np.asarray(scaling, np.float32).reshape(P, 3), np.asarray(rotation, np.float32).reshape(P, 4)],
                           axis=1)
    names = gaussian_ply_fields(rest.shape[1])
    if filter_3D is not None:
        attrs = np.concatenate([attrs, np.asarray(filter_3D, np.float32).reshape(P, 1)], axis=1)
        names = names + ["filter_3D"]
    _write_ply(path, [(n, "f4") for n in names], [attrs[:, i] for i in range(attrs.shape[1])])


def load_gaussians_ply(path: str) -> Dict[str, np.ndarray]:
    """Inverse of save_gaussians_ply (what GaussianModel.load_ply does, gaussian_model.py:280+).  The dict has a
    `filter_3D` [P,1] entry only when the file carries that property."""
    d = _read_ply(path)
    P = d.shape[0]
    col = lambda prefix: np.stack([d[n] for n in sorted((n for n in d.dtype.names if n.startswith(prefix)),
                                                        key=lambda s: int(s.split("_")[-1]))], axis=1)
    # SH degree 0 stores no f_rest_* property: f_rest is then [P, 0, 3]
    has_rest = any(n.startswith("f_rest_") for n in d.dtype.names)
    rest = col("f_rest_") if has_rest else np.zeros((P, 0), np.float32)
    out = dict(xyz=np.stack([d["x"], d["y"], d["z"]], axis=1),
               f_dc=col("f_dc_").reshape(P, 3, 1).transpose(0, 2, 1).copy(),
               f_rest=rest.reshape(P, 3, rest.shape[1] // 3).transpose(0, 2, 1).copy(),
               opacity=d["opacity"].reshape(P, 1).copy(), scaling=col("scale_"), rotation=col("rot_"))
    if "filter_3D" in d.dtype.names:
        out["filter_3D"] = d["filter_3D"].reshape(P, 1).copy()
    return out


def save_pose_npy(path: str, poses7: np.ndarray, colmap_ids: List[int] = None) -> np.ndarray:
    """train.py:46-60: [n,7] quaternion poses -> [n,4,4] w2c matrices, row i = the camera with COLMAP id i+1."""
    n = poses7.shape[0]
    ids = list(range(1, n + 1)) if colmap_ids is None else list(colmap_ids)
    mats = np.stack([pose7_to_matrix(poses7[ids.index(i + 1)]) for i in range(n)]).astype(np.float32)
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    np.save(path, mats)
    return mats


# ----------------------------------------------------------------------------------------------
# a complete synthetic `source_path` for an unchanged train.py
# ----------------------------------------------------------------------------------------------
def write_synthetic_source(root: str, scene, images_u8: np.ndarray = None) -> str:
    """Writes <root>/sparse_<n>/0/{cameras.txt,images.txt,points3D.ply,confidence_dsp.npy} (+ <root>/images/*.png when
    `images_u8` [n,H,W,3] is given and PIL is importable) for a `instantsplat_b200.scenes.Scene`."""
    import math
    n = scene.n_views
    folder = os.path.join(root, f"sparse_{n}", "0")
    fx = scene.width / (2.0 * math.tan(scene.fovx / 2.0))
    fy = scene.height / (2.0 * math.tan(scene.fovy / 2.0))
    names = [f"{i:06d}.png" for i in range(n)]
    write_colmap_text(folder, scene.width, scene.height, fx, fy, scene.poses.numpy(), names)
    xyz = scene.params["xyz"].numpy()
    rgb = np.clip((scene.params["f_dc"].numpy().reshape(-1, 3) * 0.28209479177387814 + 0.5) * 255.0, 0, 255).astype(np.uint8)
    write_points3d_ply(os.path.join(folder, "points3D.ply"), xyz, rgb)
    conf = np.zeros((scene.P, 1), np.float32)
    if scene.per_point_lr is not None:       # invert train.py:63-85: lr = (1 - sigmoid(c)) * 99 + 1
        s = np.clip((scene.per_point_lr.numpy().reshape(-1, 1) - 1.0) / 99.0, 1e-6, 1 - 1e-6)
        conf = np.log((1 - s) / s).astype(np.float32)
    np.save(os.path.join(folder, "confidence_dsp.npy"), conf)
    if images_u8 is not None:
        try:
            from PIL import Image
            os.makedirs(os.path.join(root, "images"), exist_ok=True)
            for i, name in enumerate(names):
                Image.fromarray(images_u8[i]).save(os.path.join(root, "images", name))
        except ImportError:
            pass
    return folder
