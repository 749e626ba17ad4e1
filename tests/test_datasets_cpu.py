"""Host half of the scene loaders (ngp_pl_b200/datasets.py) against the reference's loaders run on the committed fixtures
(tests/golden/datasets_*.npz, tests/golden/make_golden_datasets.py), the COLMAP reader, and the numpy restatement of the
staging kernel (oracle/stage_ref.py) against cv2 and the goldens. No GPU."""
import glob
import os
import shutil

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")
FIX = os.path.join(GOLDEN, "datasets")

import sys
sys.path.insert(0, GOLDEN)
from make_golden_datasets import CASES  # noqa: E402


def _golden(case):
    return dict(np.load(os.path.join(GOLDEN, "datasets_%s.npz" % case)))


def _meta(case):
    from ngp_pl_b200 import datasets
    name, sub, split, ds = CASES[case]
    return datasets.scene_meta(name, os.path.join(FIX, sub), split, ds)


@pytest.mark.parametrize("case", sorted(CASES))
def test_host_metadata_matches_reference_loader(case):
    """K, img_wh, directions and poses bitwise; COLMAP points bitwise in float64"""
    g, m = _golden(case), _meta(case)
    assert m.K.dtype == np.float32 and np.array_equal(m.K, g["K"])
    assert tuple(m.img_wh) == tuple(g["img_wh"])
    d = m.directions.numpy()
    assert d.dtype == np.float32 and np.array_equal(d.view(np.int32), g["directions"].view(np.int32))
    assert m.poses.dtype == np.float32 and np.array_equal(m.poses.view(np.int32), g["poses"].view(np.int32))
    assert len(m.image_paths) == g["poses"].shape[0] == g["rays"].shape[0]
    if "pts3d" in g:
        assert np.array_equal(m.pts3d, g["pts3d"])
    else:
        assert m.pts3d is None


@pytest.mark.parametrize("case", sorted(CASES))
def test_staging_restatement_matches_reference_rays(case):
    """oracle/stage_ref.py on the Pillow-decoded fixture images == the reference's read_image output, bitwise"""
    from ngp_pl_b200 import datasets
    from oracle import stage_ref
    g, m = _golden(case), _meta(case)
    w, h = m.img_wh
    for i, p in enumerate(m.image_paths):
        out = stage_ref.stage_image(datasets.decode_image(p), w, h, m.blend_a)
        assert np.array_equal(out.view(np.int32), g["rays"][i].view(np.int32)), (case, i)


def test_staging_restatement_matches_cv2_resize():
    """the evaluation order stated in oracle/stage_ref.py reproduces cv2.resize(INTER_LINEAR) on fp32 bitwise"""
    cv2 = pytest.importorskip("cv2")
    from oracle import stage_ref
    rng = np.random.RandomState(0)
    sizes = [((80, 80), (49, 49)), ((80, 80), (40, 40)), ((12, 17), (11, 16)), ((800, 800), (400, 400)), ((45, 67), (97, 131))]
    sizes += [(tuple(rng.randint(2, 160, 2)), tuple(rng.randint(1, 160, 2))) for _ in range(60)]
    for (H0, W0), (h, w) in sizes:
        for C in (3, 4):
            u8 = rng.randint(0, 256, (H0, W0, C)).astype(np.uint8)
            for blend in (True, False):
                img = u8.astype(np.float32) / 255.0
                if C == 4:
                    img = img[..., :3] * img[..., -1:] + (1 - img[..., -1:]) if blend else img[..., :3] * img[..., -1:]
                ref = cv2.resize(img, (int(w), int(h))).reshape(-1, 3)
                out = stage_ref.stage_image(u8, int(w), int(h), blend)
                assert np.array_equal(out.view(np.int32), ref.view(np.int32)), ((H0, W0), (h, w), C, blend)


def test_fma32_rounds_once():
    from oracle import stage_ref
    from fractions import Fraction
    rng = np.random.RandomState(1)
    a, b, c = (rng.randn(2000).astype(np.float32) for _ in range(3))
    c[::3] = -(a[::3].astype(np.float64) * b[::3]).astype(np.float32)  # heavy cancellation
    got = stage_ref.fma32(a, b, c)
    for x, y, z, r in zip(a[:300], b[:300], c[:300], got[:300]):
        exact = Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))
        cand = [np.float32(r), np.nextafter(np.float32(r), np.float32(np.inf)), np.nextafter(np.float32(r), np.float32(-np.inf))]
        assert abs(Fraction(float(cand[0])) - exact) <= min(abs(Fraction(float(v)) - exact) for v in cand)


def test_colmap_reader_round_trips_the_writer(tmp_path):
    from ngp_pl_b200 import datasets, synth
    import dataset_fixtures as F
    scene = synth.lego_scene(0)
    poses, corners = F.write_colmap(str(tmp_path), scene, W=64, H=48, n=9, model="OPENCV", images=False)
    cams = datasets.read_cameras_bin(str(tmp_path / "sparse/0/cameras.bin"))
    assert list(cams) == [1] and cams[1]["model"] == "OPENCV" and (cams[1]["width"], cams[1]["height"]) == (64, 48)
    assert np.array_equal(cams[1]["params"], [0.9 * 64, 0.9 * 64, 32, 24, 0.01, -0.005, 0.001, 0.0])
    ims = datasets.read_images_bin(str(tmp_path / "sparse/0/images.bin"))
    names = [im["name"] for im in ims]
    assert names != sorted(names) and sorted(names) == ["img_%03d.png" % i for i in range(9)]
    for im in ims:
        i = int(im["name"][4:7])
        assert im["id"] == 100 + i and im["camera_id"] == 1
        R = datasets.qvec_to_rotmat(im["qvec"])
        c2w = np.concatenate([R.T, (-R.T @ im["tvec"])[:, None]], 1)
        assert np.abs(c2w - poses[i]).max() < 1e-6
    assert np.array_equal(datasets.read_points3d_bin(str(tmp_path / "sparse/0/points3D.bin")), corners)


def test_partly_missing_nerf_images_raise(tmp_path):
    from ngp_pl_b200 import datasets
    root = tmp_path / "lego"
    shutil.copytree(os.path.join(FIX, "lego"), root)
    os.remove(root / "train" / "r_2.png")
    with pytest.raises(FileNotFoundError, match="1 of 4 train images are missing"):
        datasets.scene_meta("nerf", str(root), "train", 0.1)
    # a split without any image is fine (poses only, as the reference's test_traj-style splits)
    for p in glob.glob(str(root / "train" / "*.png")):
        os.remove(p)
    m = datasets.scene_meta("nerf", str(root), "train", 0.1)
    assert m.poses.shape == (4, 3, 4) and all(p is None for p in m.image_paths)


def test_unsupported_camera_model_raises(tmp_path):
    from ngp_pl_b200 import datasets, synth
    import dataset_fixtures as F
    F.write_colmap(str(tmp_path), synth.lego_scene(0), model="SIMPLE_PINHOLE", images=False)
    with pytest.raises(ValueError, match="SIMPLE_PINHOLE is not supported"):
        datasets.scene_meta("colmap", str(tmp_path), "train", 1.0)


def test_non_rgb_images_raise(tmp_path):
    from PIL import Image
    from ngp_pl_b200 import datasets
    for mode, arr in (("L", np.zeros((8, 8), np.uint8)), ("LA", np.zeros((8, 8, 2), np.uint8))):
        p = str(tmp_path / ("%s.png" % mode))
        Image.fromarray(arr, mode=mode).save(p)
        with pytest.raises(ValueError, match="only 8-bit RGB or RGBA"):
            datasets.decode_image(p)
    p = str(tmp_path / "rgb.png")
    Image.fromarray(np.zeros((8, 8, 3), np.uint8)).save(p)
    assert datasets.decode_image(p).shape == (8, 8, 3)


def test_unknown_names_and_cpu_device_raise():
    from ngp_pl_b200 import datasets
    with pytest.raises(ValueError):
        datasets.scene_meta("nsvf", FIX, "train", 1.0)
    with pytest.raises(ValueError):
        datasets.scene_meta("nerf", os.path.join(FIX, "lego"), "test_traj", 1.0)
    with pytest.raises(RuntimeError, match="no CPU path"):
        datasets.load_scene("nerf", os.path.join(FIX, "lego"), "train", 0.1, device="cpu")
