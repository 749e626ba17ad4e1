"""Golden depth images: the reference's OWN depth2img (train.py:45-50), run on seeded depth maps.

    python tests/golden/make_golden_images.py    rewrite tests/golden/images.npz (needs the reference tree and OpenCV)

depth2img is taken out of the reference's train.py with `ast` (importing train.py needs Lightning and apex) and executed
with only numpy and cv2 in scope. The inputs, all float32:
  smooth    a seeded sum of sinusoids, 37 x 53
  ramp      a linear ramp with values far from 0, 64 x 48
  zero_bg   a smooth map with a zero background, as a render's depth where opacity is 0, 40 x 40
  constant  every pixel 2.5 (0/0: index 0), 9 x 7
  nan       a smooth map with one NaN (NaN everywhere after the min/max), 16 x 12
  lego      the first-hit distance of synth.lego_scene(0) seen from camera_poses(1, seed=3), 0 where no box is hit, 80 x 80
Regenerating gives byte-identical files (fixed seeds, np.savez without compression and fixed key order).
"""
import ast
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("NGP_REFERENCE_DIR", "/root/reference")
OUT = os.path.join(HERE, "images.npz")


def load_depth2img():
    src = open(os.path.join(REF, "train.py")).read()
    fn = [n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name == "depth2img"][0]
    import cv2
    scope = {"np": np, "cv2": cv2}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), "train.py", "exec"), scope)
    return scope["depth2img"]


def lego_depth(n=80):
    sys.path.insert(0, ROOT)
    import torch
    from ngp_pl_b200 import synth
    scene = synth.lego_scene(0)
    K = synth.intrinsics(W=n, H=n, fx=1111.11 * n / 800)
    o, d = synth.get_rays(synth.ray_directions(K), torch.as_tensor(synth.camera_poses(1, seed=3))[0])
    o, d = o.double().numpy()[:, None], d.double().numpy()[:, None]
    with np.errstate(divide="ignore", invalid="ignore"):
        ta, tb = (scene.box_min - o) / d, (scene.box_max - o) / d
    t1 = np.minimum(ta, tb).max(-1)
    t2 = np.maximum(ta, tb).min(-1)
    t1 = np.where((t1 <= t2) & (t1 > 0), t1, np.inf).min(-1)
    return np.where(np.isfinite(t1), t1, 0).astype(np.float32).reshape(n, n)


def inputs():
    rng = np.random.RandomState(2024)
    yy, xx = np.mgrid[0:37, 0:53].astype(np.float32)
    smooth = (2 + np.sin(xx * 0.21 + rng.rand()) * np.cos(yy * 0.17) + 0.3 * rng.rand(37, 53)).astype(np.float32)
    ramp = np.linspace(3.0, 3.7, 64 * 48, dtype=np.float32).reshape(64, 48)
    yy, xx = np.mgrid[0:40, 0:40].astype(np.float32)
    zero_bg = np.where((xx - 20) ** 2 + (yy - 18) ** 2 < 150, 1.5 + 0.01 * xx + 0.003 * yy * yy, 0).astype(np.float32)
    nan = rng.rand(16, 12).astype(np.float32) * 4
    nan[5, 7] = np.nan
    return {"smooth": smooth, "ramp": ramp, "zero_bg": zero_bg, "constant": np.full((9, 7), 2.5, np.float32),
            "nan": nan, "lego": lego_depth()}


def main():
    depth2img = load_depth2img()
    arrays = {}
    with np.errstate(invalid="ignore", divide="ignore"):
        for k, v in inputs().items():
            arrays["depth_" + k] = v
            arrays["img_" + k] = depth2img(v)
    np.savez(OUT, **arrays)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
