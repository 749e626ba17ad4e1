"""Writes the dataset fixtures under tests/golden/datasets/ and, from the reference's own loaders run on them
(oracle/ref_datasets.py: datasets/{base,nerf,colmap,colmap_utils,ray_utils,color_utils}.py staged byte-identical, with
shims for imageio -> Pillow, kornia.create_meshgrid and tqdm), the goldens tests/golden/datasets_<case>.npz:

    K (3,3) f32, img_wh (2,), directions (hw,3) f32, poses (n,3,4) f32, rays (n,hw,3) f32 (the reference's `rays`, i.e. its
    read_image output: /255, alpha blend, cv2.resize), pts3d (m,3) f64 (COLMAP; the reference keeps a 4th, homogeneous column)

Run from the repository root where the reference tree and cv2 exist: python tests/golden/make_golden_datasets.py
"""
import os
import shutil
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

FIX = os.path.join(HERE, "datasets")

# case -> (dataset name, scene directory under tests/golden/datasets, split, downsample)
CASES = {
    "nerf_train_copy": ("nerf", "lego", "train", 0.1),          # 80 -> 80: copy
    "nerf_train_half": ("nerf", "lego", "train", 0.05),         # 80 -> 40: exact halving
    "nerf_test_04": ("nerf", "lego", "test", 0.04),             # 80 -> 32
    "nerf_trainval_odd": ("nerf", "lego", "trainval", 0.0613),  # 80 -> 49
    "colmap_train_copy": ("colmap", "pinhole", "train", 1.0),   # 64x48 copy
    "colmap_test_half": ("colmap", "pinhole", "test", 0.5),
    "colmap_trainval_odd": ("colmap", "pinhole", "trainval", 0.37),
    "colmap_radial_04": ("colmap", "radial", "train", 0.4),
    "colmap_360_images4": ("colmap", "360_v2/garden", "test", 0.25),   # images_4 at 17x12 -> 16x11
    "colmap_360_full": ("colmap", "360_v2/garden", "train", 1.0),
}


def write_fixtures():
    from ngp_pl_b200 import synth
    import dataset_fixtures as F
    shutil.rmtree(FIX, ignore_errors=True)
    lego, mip = synth.lego_scene(0), synth.mip360_scene(0)
    F.write_nerf(os.path.join(FIX, "lego"), lego, size=80)
    F.write_colmap(os.path.join(FIX, "pinhole"), lego, W=64, H=48, n=9, model="PINHOLE")
    F.write_colmap(os.path.join(FIX, "radial"), lego, W=64, H=48, n=9, model="SIMPLE_RADIAL", seed=5)
    F.write_colmap(os.path.join(FIX, "360_v2", "garden"), mip, W=67, H=45, n=9, model="OPENCV", seed=8, folders=(4,))


def make_goldens():
    from oracle import ref_datasets
    ref_datasets.stage()
    for case, (name, sub, split, ds) in CASES.items():
        cls = ref_datasets.load(name)
        d = cls(os.path.join(FIX, sub), split=split, downsample=ds)
        out = dict(K=d.K.numpy(), img_wh=np.array(d.img_wh), directions=d.directions.numpy(), poses=d.poses.numpy(),
                   rays=np.asarray(d.rays, np.float32))
        if name == "colmap":
            out["pts3d"] = np.asarray(d.pts3d, np.float64)[:, :3]
        np.savez_compressed(os.path.join(HERE, "datasets_%s.npz" % case), **out)
        print(case, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    if "--goldens-only" not in sys.argv:
        write_fixtures()
    make_goldens()
