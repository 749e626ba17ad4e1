"""Scene loaders for the fused trainer: Blender / NeRF-synthetic ('nerf', reference datasets/nerf.py) and COLMAP
('colmap', reference datasets/colmap.py), staged on the device.

    scene = load_scene('nerf', 'data/lego', split='train', downsample=0.5, device='cuda')
    tr.attach_bank(scene)                                            # device batch assembly draws from scene.rgb
    model.mark_invisible_cells(scene.K, scene.poses, scene.img_wh)
    metrics.evaluate(model, test.poses, test.directions, test.rgb, test.img_wh)

The host reads the metadata (json / COLMAP binary model), computes intrinsics, ray directions and poses exactly as the
reference does, and decodes the images with Pillow (the plugin imageio uses for PNG and JPEG, so the bytes are the
reference's). Each decoded image is uploaded as uint8 and `ngp_stage_image` (csrc/stage.cu) turns it into its fp32 row
of the bank: /255, alpha blend and cv2's bilinear resize, bitwise the reference's `read_image`. PyTorch only holds the
memory; there is no CPU path (device='cpu' raises).

Fields of the returned SceneData: K (3,3) f32, img_wh (w, h), directions (h*w,3) f32, poses (n,3,4) f32, rgb (n,h*w,3) f32
or None when the split has no images, and pts3d (m,3) float64 numpy (COLMAP; None for 'nerf'), all tensors on the device.
"""
import json
import os
import struct

import numpy as np
import torch

from . import _lib

SPLITS = ("train", "val", "test", "trainval")


class SceneData:
    def __init__(self, K, img_wh, directions, poses, rgb, pts3d=None):
        self.K, self.img_wh, self.directions, self.poses, self.rgb, self.pts3d = K, img_wh, directions, poses, rgb, pts3d


class SceneMeta:
    """The host half of a loader: everything but the pixels. K (3,3) float32, img_wh (w, h), directions (h*w,3) float32
    torch (CPU), poses (n,3,4) float32, image_paths (n; None entries when the split has no images), blend_a, pts3d."""

    def __init__(self, K, img_wh, directions, poses, image_paths, blend_a, pts3d=None):
        self.K, self.img_wh, self.directions, self.poses = K, img_wh, directions, poses
        self.image_paths, self.blend_a, self.pts3d = image_paths, blend_a, pts3d


def ray_directions(w, h, K):
    """(h*w, 3) camera-frame directions through the pixel centres, [right down front], in float32 as the reference's
    get_ray_directions (datasets/ray_utils.py:8-42) computes them from a float32 K"""
    K = torch.as_tensor(np.asarray(K, np.float32))
    v, u = torch.meshgrid(torch.arange(h, dtype=torch.float32), torch.arange(w, dtype=torch.float32), indexing="ij")
    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    d = torch.stack([(u - cx + 0.5) / fx, (v - cy + 0.5) / fy, torch.ones_like(u)], -1)
    return d.reshape(-1, 3)


# ---- Blender / NeRF-synthetic ------------------------------------------------------------------------------------------
def nerf_meta(root_dir, split="train", downsample=1.0):
    """reference datasets/nerf.py without the Jrender_Dataset path rules"""
    if split not in SPLITS:
        raise ValueError("ngp_pl_b200.datasets: unknown split %r (expected one of %s)" % (split, ", ".join(SPLITS)))
    with open(os.path.join(root_dir, "transforms_train.json")) as f:
        meta = json.load(f)
    w = h = int(800 * downsample)
    fx = 0.5 * 800 / np.tan(0.5 * meta["camera_angle_x"]) * downsample
    K = np.float32([[fx, 0, w / 2], [0, fx, h / 2], [0, 0, 1]])
    frames = []
    for s in (("train", "val") if split == "trainval" else (split,)):
        with open(os.path.join(root_dir, "transforms_%s.json" % s)) as f:
            frames += json.load(f)["frames"]
    poses, paths = [], []
    for fr in frames:
        c2w = np.array(fr["transform_matrix"], dtype=np.float64)[:3, :4]
        c2w[:, 1:3] *= -1                                      # [right up back] -> [right down front]
        c2w[:, 3] /= np.linalg.norm(c2w[:, 3]) / 1.5            # cameras on the radius-1.5 sphere
        poses.append(c2w)
        p = os.path.join(root_dir, "%s.png" % fr["file_path"])
        paths.append(p if os.path.isfile(p) else None)
    have = [p is not None for p in paths]
    if any(have) and not all(have):
        missing = [fr["file_path"] for fr, ok in zip(frames, have) if not ok]
        raise FileNotFoundError("ngp_pl_b200.datasets: %d of %d %s images are missing (e.g. %s.png); poses and images would "
                                "no longer line up" % (len(missing), len(frames), split, missing[0]))
    poses = np.asarray(poses).astype(np.float32).reshape(-1, 3, 4)
    return SceneMeta(K, (w, h), ray_directions(w, h, K), poses, paths, True)


# ---- COLMAP binary model (https://colmap.github.io/format.html#binary-file-format) --------------------------------------
# model id -> (name, number of parameters)
CAMERA_MODELS = {0: ("SIMPLE_PINHOLE", 3), 1: ("PINHOLE", 4), 2: ("SIMPLE_RADIAL", 4), 3: ("RADIAL", 5), 4: ("OPENCV", 8),
                 5: ("OPENCV_FISHEYE", 8), 6: ("FULL_OPENCV", 12), 7: ("FOV", 5), 8: ("SIMPLE_RADIAL_FISHEYE", 4),
                 9: ("RADIAL_FISHEYE", 5), 10: ("THIN_PRISM_FISHEYE", 12)}


class _Reader:
    def __init__(self, path):
        with open(path, "rb") as f:
            self.b = f.read()
        self.o = 0

    def get(self, fmt):
        v = struct.unpack_from("<" + fmt, self.b, self.o)
        self.o += struct.calcsize("<" + fmt)
        return v

    def cstring(self):
        e = self.b.index(b"\0", self.o)
        s = self.b[self.o:e].decode("utf-8")
        self.o = e + 1
        return s


def read_cameras_bin(path):
    """{camera_id: dict(model, width, height, params)}"""
    r, out = _Reader(path), {}
    for _ in range(r.get("Q")[0]):
        cam_id, model_id, width, height = r.get("iiQQ")
        if model_id not in CAMERA_MODELS:
            raise ValueError("ngp_pl_b200.datasets: unknown COLMAP camera model id %d in %s" % (model_id, path))
        name, n_par = CAMERA_MODELS[model_id]
        out[cam_id] = dict(model=name, width=width, height=height, params=np.array(r.get("%dd" % n_par)))
    return out


def read_images_bin(path):
    """[dict(id, qvec (w,x,y,z), tvec, camera_id, name)] in file order (the 2-D points are skipped)"""
    r, out = _Reader(path), []
    for _ in range(r.get("Q")[0]):
        img_id = r.get("i")[0]
        q = np.array(r.get("4d"))
        t = np.array(r.get("3d"))
        cam_id = r.get("i")[0]
        name = r.cstring()
        n2d = r.get("Q")[0]
        r.o += n2d * 24                                       # (x, y: double, point3D_id: int64) per point
        out.append(dict(id=img_id, qvec=q, tvec=t, camera_id=cam_id, name=name))
    return out


def read_points3d_bin(path):
    """(m, 3) float64 point positions in file order"""
    r, xyz = _Reader(path), []
    for _ in range(r.get("Q")[0]):
        r.get("Q")                                            # point3D_id
        xyz.append(r.get("3d"))
        r.get("3Bd")                                          # colour, reprojection error
        track = r.get("Q")[0]
        r.o += track * 8                                      # track: (image_id, point2D_idx) int32 pairs
    return np.array(xyz, np.float64).reshape(-1, 3)


def qvec_to_rotmat(q):
    w, x, y, z = q
    return np.array([[1 - 2 * y ** 2 - 2 * z ** 2, 2 * x * y - 2 * w * z, 2 * z * x + 2 * w * y],
                     [2 * x * y + 2 * w * z, 1 - 2 * x ** 2 - 2 * z ** 2, 2 * y * z - 2 * w * x],
                     [2 * z * x - 2 * w * y, 2 * y * z + 2 * w * x, 1 - 2 * x ** 2 - 2 * y ** 2]])


def _unit(v):
    return v / np.linalg.norm(v)


def recenter(poses, pts):
    """reference datasets/ray_utils.py:108-178 (center_poses with a point cloud): the frame whose origin is the cloud's mean,
    z the mean camera z, x = unit(mean camera y  x  z), y = z x x; poses and points expressed in it"""
    z = _unit(poses[..., 2].mean(0))
    x = _unit(np.cross(poses[..., 1].mean(0), z))
    avg = np.eye(4)
    avg[:3] = np.stack([x, np.cross(z, x), z, pts.mean(0)], 1)
    inv = np.linalg.inv(avg)
    homo = np.concatenate([poses, np.tile(np.array([0, 0, 0, 1]), (len(poses), 1, 1))], 1)
    return (inv @ homo)[:, :3], (pts @ inv[:, :3].T + inv[:, 3:].T)[:, :3]


def colmap_meta(root_dir, split="train", downsample=1.0):
    """reference datasets/colmap.py for plain captures and mip-NeRF 360 (no HDR-NeRF exposures, no test_traj)"""
    if split not in SPLITS:
        raise ValueError("ngp_pl_b200.datasets: unknown split %r (expected one of %s)" % (split, ", ".join(SPLITS)))
    cams = read_cameras_bin(os.path.join(root_dir, "sparse/0/cameras.bin"))
    if 1 not in cams:
        raise ValueError("ngp_pl_b200.datasets: %s has no camera 1" % root_dir)
    cam = cams[1]
    w, h = int(cam["width"] * downsample), int(cam["height"] * downsample)
    p = cam["params"]
    if cam["model"] == "SIMPLE_RADIAL":                       # distortion is ignored, as in the reference
        fx = fy = p[0] * downsample
        cx, cy = p[1] * downsample, p[2] * downsample
    elif cam["model"] in ("PINHOLE", "OPENCV"):
        fx, fy, cx, cy = (v * downsample for v in p[:4])
    else:
        raise ValueError("ngp_pl_b200.datasets: COLMAP camera model %s is not supported (SIMPLE_RADIAL, PINHOLE or OPENCV)"
                         % cam["model"])
    K = np.float32([[fx, 0, cx], [0, fy, cy], [0, 0, 1]])

    ims = read_images_bin(os.path.join(root_dir, "sparse/0/images.bin"))
    w2c = np.stack([np.concatenate([np.concatenate([qvec_to_rotmat(im["qvec"]), im["tvec"].reshape(3, 1)], 1),
                                    np.array([[0, 0, 0, 1.0]])], 0) for im in ims])
    order = np.argsort([im["name"] for im in ims])
    poses = np.linalg.inv(w2c)[order, :3]
    poses, pts = recenter(poses, read_points3d_bin(os.path.join(root_dir, "sparse/0/points3D.bin")))
    scale = np.linalg.norm(poses[..., 3], axis=-1).min()
    poses[..., 3] /= scale
    pts = pts / scale

    folder = "images_%d" % int(1 / downsample) if ("360_v2" in root_dir and downsample < 1) else "images"
    paths = [os.path.join(root_dir, folder, ims[i]["name"]) for i in order]
    keep = np.arange(len(paths))
    if split == "train":
        keep = keep[keep % 8 != 0]
    elif split == "test":
        keep = keep[keep % 8 == 0]
    paths = [paths[i] for i in keep]
    for q in paths:
        if not os.path.isfile(q):
            raise FileNotFoundError("ngp_pl_b200.datasets: image %s of the COLMAP model is missing" % q)
    return SceneMeta(K, (w, h), ray_directions(w, h, K), poses[keep].astype(np.float32), paths, False, pts)


def scene_meta(name, root_dir, split="train", downsample=1.0):
    if name == "nerf":
        return nerf_meta(root_dir, split, downsample)
    if name == "colmap":
        return colmap_meta(root_dir, split, downsample)
    raise ValueError("ngp_pl_b200.datasets: unknown dataset %r (expected 'nerf' or 'colmap')" % (name,))


# ---- decode + device staging --------------------------------------------------------------------------------------------
def decode_image(path):
    """uint8 (H, W, 3 or 4) as imageio.imread decodes it through Pillow; anything but RGB or RGBA raises"""
    try:
        from PIL import Image
    except ImportError as e:
        raise ImportError("ngp_pl_b200.datasets needs Pillow to decode images (pip install pillow)") from e
    with Image.open(path) as im:
        if im.mode not in ("RGB", "RGBA"):
            raise ValueError("ngp_pl_b200.datasets: %s is a %s image; only 8-bit RGB or RGBA images are supported"
                             % (path, im.mode))
        return np.array(im)


def stage_image(img_u8, w, h, blend_a, out):
    """one ngp_stage_image launch on the current stream: img_u8 a CUDA uint8 (H0, W0, 3|4) tensor, out a CUDA float32
    (h*w, 3) tensor (a row of the bank)"""
    if not (img_u8.is_cuda and out.is_cuda):
        raise RuntimeError("ngp_pl_b200.datasets.stage_image: tensors must be on a CUDA device (there is no CPU path)")
    if img_u8.dtype != torch.uint8 or img_u8.dim() != 3 or img_u8.shape[2] not in (3, 4) or not img_u8.is_contiguous():
        raise RuntimeError("ngp_pl_b200.datasets.stage_image: expected a contiguous uint8 (H, W, 3|4) image, got %s %s"
                           % (img_u8.dtype, tuple(img_u8.shape)))
    if out.dtype != torch.float32 or out.numel() != 3 * w * h or not out.is_contiguous():
        raise RuntimeError("ngp_pl_b200.datasets.stage_image: expected a contiguous float32 (%d, 3) output" % (w * h))
    H0, W0, C = img_u8.shape
    rc = _lib.lib().ngp_stage_image(img_u8.data_ptr(), H0, W0, C, int(bool(blend_a)), int(h), int(w), out.data_ptr(),
                                    torch.cuda.current_stream(out.device).cuda_stream)
    _lib.check(rc, "stage_image")


def load_scene(name, root_dir, split="train", downsample=1.0, device="cuda"):
    """Load split `split` of a 'nerf' or 'colmap' scene at `downsample` onto `device` (see the module docstring)."""
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError("ngp_pl_b200.datasets.load_scene needs a CUDA device (there is no CPU path)")
    m = scene_meta(name, root_dir, split, downsample)
    w, h = m.img_wh
    rgb = None
    if m.image_paths and m.image_paths[0] is not None:
        rgb = torch.empty(len(m.image_paths), w * h, 3, device=device, dtype=torch.float32)
        with torch.cuda.device(device):
            for i, p in enumerate(m.image_paths):
                src = torch.from_numpy(decode_image(p)).to(device)
                stage_image(src, w, h, m.blend_a, rgb[i])
    return SceneData(torch.as_tensor(m.K, device=device), (w, h), m.directions.to(device),
                     torch.as_tensor(m.poses, device=device), rgb, m.pts3d)
