"""Deterministic scene fixtures in the two on-disk formats ngp_pl_b200.datasets reads, rendered from the synthetic scenes.

write_nerf(root, scene, ...)    Blender / NeRF-synthetic: transforms_{train,val,test}.json + RGBA PNGs (alpha = hit mask),
                                Blender camera axes [right up back], cameras at a radius other than 1.5
write_colmap(root, scene, ...)  COLMAP binary model sparse/0/{cameras,images,points3D}.bin (images listed out of name order,
                                with 2-D points and tracks to skip) + RGB PNGs under images/ and, optionally, images_<f>/ at
                                ceil(size / f) like mip-NeRF 360's pre-downsampled folders

The committed fixtures under tests/golden/datasets/ were written by tests/golden/make_golden_datasets.py; the GPU tests
write larger ones of the same kind into a temporary directory.
"""
import json
import math
import os
import struct

import numpy as np
import torch

from ngp_pl_b200 import synth

MODEL_IDS = {"SIMPLE_PINHOLE": 0, "PINHOLE": 1, "SIMPLE_RADIAL": 2, "OPENCV": 4}


def render(scene, K, c2w, alpha=True):
    """uint8 (H, W, 4|3) image of `scene` seen from c2w (3,4) [right down front] with intrinsics dict K"""
    dirs = synth.ray_directions(K)
    o, d = synth.get_rays(dirs, torch.as_tensor(c2w, dtype=torch.float32))
    rgb = synth.trace(scene, o, d).numpy()
    img = np.round(rgb * 255).clip(0, 255).astype(np.uint8).reshape(K["H"], K["W"], 3)
    if not alpha:
        return img
    # alpha = hit mask: the background pixels (exactly the scene's bg colour) are transparent
    hit = ~np.all(rgb.reshape(K["H"], K["W"], 3) == np.float32(scene.bg), -1)
    return np.concatenate([img, (hit * 255).astype(np.uint8)[..., None]], -1)


def save_png(path, img):
    from PIL import Image
    os.makedirs(os.path.dirname(path), exist_ok=True)
    Image.fromarray(img).save(path)


def write_nerf(root, scene, size=80, splits=(("train", 4), ("val", 2), ("test", 2)), radius=4.0, seed=0, fx800=1111.11,
               images=True):
    """A NeRF-synthetic scene directory; returns {split: (n,3,4) float32 [right down front] poses at radius 1.5}"""
    os.makedirs(root, exist_ok=True)
    angle = 2 * math.atan(400.0 / fx800)
    K = synth.intrinsics(W=size, H=size, fx=fx800 * size / 800)
    out, k = {}, 0
    for split, n in splits:
        poses = synth.camera_poses(n, radius=1.5, seed=seed + 31 * k)
        k += 1
        frames = []
        for i, c2w in enumerate(poses):
            m = np.eye(4)
            m[:3, :4] = c2w
            m[:3, 1:3] *= -1                      # [right down front] -> Blender's [right up back]
            m[:3, 3] *= radius / 1.5
            name = "./%s/r_%d" % (split, i)
            frames.append({"file_path": name, "rotation": 0.0, "transform_matrix": m.tolist()})
            if images:
                save_png(os.path.join(root, split, "r_%d.png" % i), render(scene, K, c2w, alpha=True))
        with open(os.path.join(root, "transforms_%s.json" % split), "w") as f:
            json.dump({"camera_angle_x": angle, "frames": frames}, f, indent=1)
        out[split] = poses
    return out


def rotmat_to_qvec(R):
    """unit quaternion (w, x, y, z) of a rotation matrix (Shepperd's method)"""
    t = np.trace(R)
    if t > 0:
        s = 2 * math.sqrt(1 + t)
        q = [s / 4, (R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s]
    else:
        i = int(np.argmax(np.diag(R)))
        j, k = (i + 1) % 3, (i + 2) % 3
        s = 2 * math.sqrt(1 + R[i, i] - R[j, j] - R[k, k])
        q = [0.0] * 4
        q[0] = (R[k, j] - R[j, k]) / s
        q[1 + i] = s / 4
        q[1 + j] = (R[j, i] + R[i, j]) / s
        q[1 + k] = (R[k, i] + R[i, k]) / s
    q = np.array(q)
    return q / np.linalg.norm(q)


def write_colmap(root, scene, W=64, H=48, n=9, model="PINHOLE", radius=None, seed=3, folders=(), images=True):
    """A COLMAP scene directory; returns the (n,3,4) float32 c2w poses in image-name order and the (m,3) points"""
    fx = 0.9 * W
    K = synth.intrinsics(W=W, H=H, fx=fx)
    radius = synth.camera_radius(scene) if radius is None else radius
    poses = synth.camera_poses(n, radius=radius, seed=seed, upper_only=scene.scale <= 0.5)
    params = {"SIMPLE_PINHOLE": [fx, W / 2, H / 2], "PINHOLE": [fx, fx, W / 2, H / 2],
              "SIMPLE_RADIAL": [fx, W / 2, H / 2, 0.01],
              "OPENCV": [fx, fx, W / 2, H / 2, 0.01, -0.005, 0.001, 0.0]}[model]
    sp = os.path.join(root, "sparse", "0")
    os.makedirs(sp, exist_ok=True)
    with open(os.path.join(sp, "cameras.bin"), "wb") as f:
        f.write(struct.pack("<Q", 1))
        f.write(struct.pack("<iiQQ", 1, MODEL_IDS[model], W, H))
        f.write(struct.pack("<%dd" % len(params), *params))
    rng = np.random.RandomState(seed)
    names = ["img_%03d.png" % i for i in range(n)]
    with open(os.path.join(sp, "images.bin"), "wb") as f:
        f.write(struct.pack("<Q", n))
        for i in rng.permutation(n):                      # file order != name order
            R_cw = poses[i, :, :3].astype(np.float64)
            R = R_cw.T
            t = -R @ poses[i, :, 3].astype(np.float64)
            f.write(struct.pack("<i", 100 + int(i)))
            f.write(struct.pack("<4d", *rotmat_to_qvec(R)))
            f.write(struct.pack("<3d", *t))
            f.write(struct.pack("<i", 1))
            f.write(names[i].encode() + b"\0")
            n2d = int(i % 3)
            f.write(struct.pack("<Q", n2d))
            for p in range(n2d):
                f.write(struct.pack("<ddq", 1.5 * p, 2.5 * p, p if p % 2 else -1))
    corners = np.array([[x, y, z] for lo, hi in zip(scene.box_min, scene.box_max)
                        for x in (lo[0], hi[0]) for y in (lo[1], hi[1]) for z in (lo[2], hi[2])], np.float64)
    with open(os.path.join(sp, "points3D.bin"), "wb") as f:
        f.write(struct.pack("<Q", len(corners)))
        for j, xyz in enumerate(corners):
            f.write(struct.pack("<Q", 7 + j))
            f.write(struct.pack("<3d", *xyz))
            f.write(struct.pack("<3Bd", 10, 20, 30, 0.25))
            tl = j % 3
            f.write(struct.pack("<Q", tl))
            for t_ in range(tl):
                f.write(struct.pack("<ii", 100 + t_, j))
    if images:
        for i in range(n):
            img = render(scene, K, poses[i], alpha=False)
            save_png(os.path.join(root, "images", names[i]), img)
            for fct in folders:
                w_, h_ = -(-W // fct), -(-H // fct)
                save_png(os.path.join(root, "images_%d" % fct, names[i]),
                         render(scene, synth.intrinsics(W=w_, H=h_, fx=fx * w_ / W, fy=fx * h_ / H), poses[i], alpha=False))
    return poses, corners
