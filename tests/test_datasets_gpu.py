"""GPU tests of the scene front end: ngp_stage_image against the reference loaders' goldens, ngp_sample_rays_ex (fp32
banks, 'same_image') against ngp_sample_rays and a numpy Philox restatement, Trainer.attach_bank's checks, and training
on scenes loaded through datasets.load_scene."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")
FIX = os.path.join(GOLDEN, "datasets")
sys.path.insert(0, GOLDEN)
from make_golden_datasets import CASES  # noqa: E402


# ---- staging ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", sorted(CASES))
def test_load_scene_stages_the_reference_rays_bitwise(case):
    """cases with and without a resize (copy, exact halving, 80->49, 17x12->16x11, ...): bitwise the reference's rays"""
    from ngp_pl_b200 import datasets
    g = dict(np.load(os.path.join(GOLDEN, "datasets_%s.npz" % case)))
    name, sub, split, ds = CASES[case]
    s = datasets.load_scene(name, os.path.join(FIX, sub), split, ds, device="cuda")
    assert s.rgb.is_cuda and s.rgb.dtype == torch.float32 and s.rgb.shape == g["rays"].shape
    assert np.array_equal(s.rgb.cpu().numpy().view(np.int32), g["rays"].view(np.int32))
    assert np.array_equal(s.poses.cpu().numpy(), g["poses"]) and np.array_equal(s.directions.cpu().numpy(), g["directions"])
    assert np.array_equal(s.K.cpu().numpy(), g["K"]) and tuple(s.img_wh) == tuple(g["img_wh"])


def test_stage_image_matches_restatement_on_random_images_and_rejects_bad_arguments():
    from ngp_pl_b200 import _lib, datasets
    from oracle import stage_ref
    rng = np.random.RandomState(0)
    for (H0, W0), (h, w), C_, blend in [((800, 800), (400, 400), 4, True), ((801, 799), (123, 457), 4, False),
                                        ((45, 67), (97, 131), 3, True), ((2, 2), (5, 3), 4, True), ((33, 31), (33, 31), 4, False)]:
        u8 = rng.randint(0, 256, (H0, W0, C_)).astype(np.uint8)
        out = torch.empty(h * w, 3, device="cuda")
        datasets.stage_image(torch.as_tensor(u8).cuda(), w, h, blend, out)
        ref = stage_ref.stage_image(u8, w, h, blend)
        assert np.array_equal(out.cpu().numpy().view(np.int32), ref.view(np.int32)), ((H0, W0), (h, w))
    L, st = _lib.lib(), torch.cuda.current_stream().cuda_stream
    src = torch.zeros(4, 4, 4, dtype=torch.uint8, device="cuda")
    dst = torch.empty(16, 3, device="cuda")
    assert L.ngp_stage_image(src.data_ptr(), 4, 4, 2, 1, 4, 4, dst.data_ptr(), st) == -22      # 2 channels
    assert L.ngp_stage_image(src.data_ptr(), 1, 16, 4, 1, 2, 8, dst.data_ptr(), st) == -22     # resize of a single row
    assert L.ngp_stage_image(None, 4, 4, 4, 1, 4, 4, dst.data_ptr(), st) == -22
    with pytest.raises(RuntimeError):
        datasets.stage_image(src.cpu(), 4, 4, True, dst)


# ---- batch assembly -----------------------------------------------------------------------------------------------------
def philox4x32_10(ctr, key):
    """numpy restatement of the kernel's Philox-4x32-10 (ctr: 4 uint32 arrays, key: 2 uint32)"""
    M = np.uint64(0xFFFFFFFF)
    x = [np.asarray(c, np.uint64) & M for c in ctr]
    k0, k1 = np.uint64(key[0]), np.uint64(key[1])
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * x[0]
        p1 = np.uint64(0xCD9E8D57) * x[2]
        hi0, lo0 = p0 >> np.uint64(32), p0 & M
        hi1, lo1 = p1 >> np.uint64(32), p1 & M
        x = [hi1 ^ x[1] ^ k0, lo1, hi0 ^ x[3] ^ k1, lo0]
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & M, (k1 + np.uint64(0xBB67AE85)) & M
    return x


def umulhi(a, n):
    return ((np.asarray(a, np.uint64) * np.uint64(n)) >> np.uint64(32)).astype(np.int64)


def _bank(store_dtype=torch.uint8, n_images=7):
    from ngp_pl_b200 import synth
    return synth.RayBank(synth.lego_scene(0), n_images=n_images, K=synth.intrinsics(W=40, H=30, fx=300.0), device="cuda",
                         store_dtype=store_dtype)


def _draw_ex(bank, n, seed, stream, ctr, dtype, strategy, rgb=None):
    from ngp_pl_b200 import _lib
    rgb = bank.rgb if rgb is None else rgb
    o, d, c = (torch.empty(n, 3, device="cuda") for _ in range(3))
    z = torch.empty(n, device="cuda")
    _lib.check(_lib.lib().ngp_sample_rays_ex(bank.poses.data_ptr(), bank.directions.data_ptr(), rgb.data_ptr(), dtype,
                                             strategy, bank.poses.shape[0], bank.directions.shape[0], n, seed, stream,
                                             ctr.data_ptr(), o.data_ptr(), d.data_ptr(), c.data_ptr(), z.data_ptr(),
                                             torch.cuda.current_stream().cuda_stream), "sample_rays_ex")
    return o, d, c, z


def _recover(bank, o, d):
    """(image, pixel) of every ray, through ngp_gen_rays' convention (as test_fused_gpu does)"""
    origins = bank.poses[:, :, 3]
    im = (o[:, None, :] - origins[None]).abs().sum(-1).argmin(1)
    assert torch.equal(o, origins[im])
    all_d = torch.einsum("pc,ikc->ipk", bank.directions, bank.poses[:, :, :3])
    px = (all_d[im] - d[:, None, :]).abs().sum(-1).argmin(1)
    return im, px


def test_sample_rays_ex_u8_all_images_is_sample_rays_bitwise():
    from ngp_pl_b200 import _lib
    bank = _bank()
    n = 20000
    L = _lib.lib()
    c1 = torch.zeros(2, dtype=torch.int32, device="cuda")
    c2 = torch.zeros(2, dtype=torch.int32, device="cuda")
    for step in range(3):
        o, d, c, z = (torch.empty(n, 3, device="cuda"), torch.empty(n, 3, device="cuda"), torch.empty(n, 3, device="cuda"),
                      torch.empty(n, device="cuda"))
        _lib.check(L.ngp_sample_rays(bank.poses.data_ptr(), bank.directions.data_ptr(), bank.rgb.data_ptr(), 7,
                                     bank.directions.shape[0], n, 11, 1, c1.data_ptr(), o.data_ptr(), d.data_ptr(), c.data_ptr(),
                                     z.data_ptr(), torch.cuda.current_stream().cuda_stream), "sample_rays")
        o2, d2, c2_, z2 = _draw_ex(bank, n, 11, 1, c2, 0, 0)
        for a, b in ((o, o2), (d, d2), (c, c2_), (z, z2)):
            assert torch.equal(a, b)
        assert torch.equal(c1, c2) and c1.tolist() == [step + 1, 0]
    assert L.ngp_sample_rays_ex(bank.poses.data_ptr(), bank.directions.data_ptr(), bank.rgb.data_ptr(), 2, 0, 7, 1200, 8,
                                0, 0, c2.data_ptr(), o.data_ptr(), d.data_ptr(), c.data_ptr(), z.data_ptr(), None) == -22
    assert L.ngp_sample_rays_ex(bank.poses.data_ptr(), bank.directions.data_ptr(), bank.rgb.data_ptr(), 0, 2, 7, 1200, 8,
                                0, 0, c2.data_ptr(), o.data_ptr(), d.data_ptr(), c.data_ptr(), z.data_ptr(), None) == -22


def test_f32_bank_rgb_gt_is_the_bank_entry_and_indices_match_philox():
    bank = _bank(torch.float32)
    n, seed, stream = 20000, 5, 0
    ctr = torch.zeros(2, dtype=torch.int32, device="cuda")
    o, d, c, z = _draw_ex(bank, n, seed, stream, ctr, 1, 0)
    im, px = _recover(bank, o, d)
    assert torch.equal(c, bank.rgb[im, px])
    r = philox4x32_10([np.arange(n), np.zeros(n), np.zeros(n), np.zeros(n)], (seed, stream))
    assert np.array_equal(im.cpu().numpy(), umulhi(r[0], 7)) and np.array_equal(px.cpu().numpy(), umulhi(r[1], 1200))
    assert np.array_equal(z.cpu().numpy(), (r[2] >> np.uint64(8)).astype(np.float32) * np.float32(1 / 16777216))
    # the same draw on the uint8 bank of the same scene: same rays, colours v/255
    ub = _bank(torch.uint8)
    o2, d2, c2, z2 = _draw_ex(ub, n, seed, stream, torch.zeros(2, dtype=torch.int32, device="cuda"), 0, 0)
    assert torch.equal(o2, o) and torch.equal(d2, d) and torch.equal(z2, z)
    assert torch.equal(c2, ub.rgb[im, px].float() * (torch.ones((), device="cuda") / 255))


@pytest.mark.parametrize("dtype", [0, 1])
def test_same_image_draws_one_image_per_batch_from_philox(dtype):
    bank = _bank(torch.uint8 if dtype == 0 else torch.float32)
    n, seed, stream = 5000, 9, 1
    ctr = torch.zeros(2, dtype=torch.int32, device="cuda")
    ctr_all = torch.zeros(2, dtype=torch.int32, device="cuda")
    for draw in range(4):
        o, d, c, z = _draw_ex(bank, n, seed, stream, ctr, dtype, 1)
        oa, da, ca, za = _draw_ex(bank, n, seed, stream, ctr_all, dtype, 0)
        im, px = _recover(bank, o, d)
        assert im.unique().numel() == 1
        q = philox4x32_10([np.zeros(1), np.full(1, draw), np.ones(1), np.zeros(1)], (seed, stream))
        assert int(im[0]) == int(umulhi(q[0], 7)[0])
        r = philox4x32_10([np.arange(n), np.full(n, draw), np.zeros(n), np.zeros(n)], (seed, stream))
        assert np.array_equal(px.cpu().numpy(), umulhi(r[1], 1200))
        # pixels and jitter are those of 'all_images'; only the image differs
        _, pxa = _recover(bank, oa, da)
        assert torch.equal(px, pxa) and torch.equal(z, za)
        ref = bank.rgb[im, px]
        assert torch.equal(c, ref if dtype == 1 else ref.float() * (torch.ones((), device="cuda") / 255))
    assert ctr.tolist() == [4, 0]


def test_same_image_histogram_over_graph_replays():
    """every replay of a captured graph draws a new image; over 2100 replays the image histogram passes a chi-square test"""
    from scipy import stats
    from ngp_pl_b200 import _lib
    bank = _bank(torch.float32)
    n, n_img = 64, bank.poses.shape[0]
    ctr = torch.zeros(2, dtype=torch.int32, device="cuda")
    o, d, c = (torch.empty(n, 3, device="cuda") for _ in range(3))
    z = torch.empty(n, device="cuda")
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            _lib.check(_lib.lib().ngp_sample_rays_ex(bank.poses.data_ptr(), bank.directions.data_ptr(), bank.rgb.data_ptr(), 1,
                                                     1, n_img, bank.directions.shape[0], n, 21, 0, ctr.data_ptr(),
                                                     o.data_ptr(), d.data_ptr(), c.data_ptr(), z.data_ptr(), s.cuda_stream),
                       "sample_rays_ex")
    origins = bank.poses[:, :, 3]
    R = 2100
    lo = torch.zeros(R, dtype=torch.int64, device="cuda")
    hi = torch.zeros(R, dtype=torch.int64, device="cuda")
    for k in range(R):
        g.replay()
        im = (o[:, None, :] - origins[None]).abs().sum(-1).argmin(1)
        lo[k], hi[k] = im.min(), im.max()
    torch.cuda.synchronize()
    assert ctr.tolist() == [R, 0] and torch.equal(lo, hi)
    h = lo.cpu().numpy()
    q = philox4x32_10([np.zeros(R), np.arange(R), np.ones(R), np.zeros(R)], (21, 0))
    assert np.array_equal(h, umulhi(q[0], n_img))
    cnt = np.bincount(h, minlength=n_img)
    assert stats.chisquare(cnt).pvalue > 1e-3, cnt


# ---- Trainer ------------------------------------------------------------------------------------------------------------
class _B:
    def __init__(self, poses, directions, rgb):
        self.poses, self.directions, self.rgb = poses, directions, rgb


def test_attach_bank_rejects_bad_banks_and_a_float32_raybank_trains():
    from ngp_pl_b200 import synth
    from ngp_pl_b200.models.networks import NGP
    from ngp_pl_b200.trainer import Trainer
    scene = synth.lego_scene(0)
    model = NGP(scene.scale).cuda()
    tr = Trainer(model, n_rays=4096)
    with pytest.raises(ValueError):
        Trainer(NGP(scene.scale).cuda(), n_rays=256, ray_sampling_strategy="same_pixel")
    P = torch.zeros(3, 3, 4, device="cuda")
    D = torch.zeros(20, 3, device="cuda")
    RGB = torch.zeros(3, 20, 3, device="cuda")
    bad = [_B(P.cpu(), D, RGB), _B(P, D.cpu(), RGB), _B(P, D, RGB.cpu()),                   # CPU tensors
           _B(P, D, RGB.double()), _B(P, D, RGB.half()), _B(P.double(), D, RGB), _B(P, D.half(), RGB),  # dtypes
           _B(P, D, RGB[:, :10]), _B(P, D, RGB[:2]), _B(P[:, :, :3].contiguous(), D, RGB),  # shapes
           _B(P, D, RGB.transpose(0, 1).contiguous().transpose(0, 1)),                     # non-contiguous
           _B(P, D, None), object()]
    for b in bad:
        with pytest.raises(RuntimeError):
            tr.attach_bank(b)
    tr.attach_bank(_B(P, D, RGB.to(torch.uint8)))
    tr.attach_bank(_B(P, D, RGB))

    bank = synth.RayBank(scene, n_images=50, K=synth.intrinsics(W=100, H=100, fx=1111.11 / 8), device="cuda",
                         store_dtype=torch.float32)
    tr.attach_bank(bank)
    tr.capture()
    for _ in range(600):
        tr.train_step()
    torch.cuda.synchronize()
    st = tr.stats()
    assert np.isfinite(st["loss"]) and st["psnr"] > 22, st
    # the batch's ground truth is the bank's fp32 values, not their bytes
    o, d = tr.rays_o.clone(), tr.rays_d.clone()
    im, px = _recover(bank, o, d)
    assert torch.equal(tr.rgb_gt, bank.rgb[im, px])


def _train_and_score(bank, test, strategy, steps=1000, seed=0):
    from ngp_pl_b200 import metrics, synth
    from ngp_pl_b200.models.networks import NGP
    from ngp_pl_b200.trainer import Trainer
    torch.manual_seed(seed)
    model = NGP(0.5).cuda()
    tr = Trainer(model, n_rays=8192, seed=seed, ray_sampling_strategy=strategy)
    tr.attach_bank(bank)
    tr.capture()
    for _ in range(steps):
        tr.train_step()
    torch.cuda.synchronize()
    del tr
    return metrics.evaluate(model, test.poses, test.directions, test.rgb, test.img_wh)["psnr"]


def test_nerf_fixture_trains_like_the_in_memory_bank(tmp_path):
    """SynthLego written as a NeRF-synthetic scene (RGBA PNGs, Blender axes, radius 4) and loaded back trains to the test
    PSNR of the same run on synth.RayBank -- same resolution, steps, seed and sampling strategy, hence the same (image,
    pixel) draws -- within 0.5 dB (means over six seeds), under both strategies. (At 1000 steps 'same_image' itself scores
    ~0.9 dB below 'all_images' on this scene: one image per batch gives correlated gradients.)"""
    import dataset_fixtures as F
    from ngp_pl_b200 import datasets, synth
    scene = synth.lego_scene(0)
    F.write_nerf(str(tmp_path), scene, size=100, splits=(("train", 50), ("val", 1), ("test", 8)), radius=4.0)
    train = datasets.load_scene("nerf", str(tmp_path), "train", 0.125)
    test = datasets.load_scene("nerf", str(tmp_path), "test", 0.125)
    assert train.rgb.shape == (50, 100 * 100, 3) and train.img_wh == (100, 100)
    bank = synth.RayBank(scene, n_images=50, K=synth.intrinsics(W=100, H=100, fx=1111.11 / 8), device="cuda")
    # same cameras up to the radius rescale; same pixels up to v/255 vs v*(1/255), except box edges the CPU trace of the
    # fixture and the GPU trace of the bank round differently
    assert (bank.poses - train.poses).abs().max() < 1e-6
    assert ((bank.rgb.float() / 255 - train.rgb).abs().max(-1)[0] > 1e-6).float().mean() < 0.01
    # Training is not bitwise repeatable (the table gradients are fp32 atomics), and 'same_image' amplifies that: two runs
    # of the same seed on the same bank differed by up to 1.3 dB (seed 0; seeds 1-7 by <= 0.35 dB; 'all_images' by
    # <= 0.12 dB; H100 80GB HBM3, 700 W). A mean over two seeds then moves by 0.6 dB from run to run; over six, one such
    # seed moves it by <= 0.22 dB
    seeds = range(6)
    for s in ("all_images", "same_image"):
        base = np.mean([_train_and_score(bank, test, s, seed=k) for k in seeds])
        got = np.mean([_train_and_score(train, test, s, seed=k) for k in seeds])
        print("%s test PSNR: RayBank %.3f, load_scene %.3f" % (s, base, got))
        assert base > 24 and abs(got - base) < 0.5, (s, got, base)


def test_colmap_fixture_trains_with_erode():
    from ngp_pl_b200 import datasets, metrics
    from ngp_pl_b200.models.networks import NGP
    from ngp_pl_b200.trainer import Trainer
    root = os.path.join(FIX, "pinhole")
    train = datasets.load_scene("colmap", root, "train", 1.0)
    test = datasets.load_scene("colmap", root, "test", 1.0)
    assert isinstance(train.pts3d, np.ndarray) and train.pts3d.shape[1] == 3
    model = NGP(0.5).cuda()
    # the buffers the reference's train.py:72-76 registers before mark_invisible_cells (train.py:155-157)
    G = model.grid_size
    model.register_buffer("density_grid", torch.zeros(model.cascades, G ** 3, device="cuda"))
    model.register_buffer("grid_coords", torch.stack(torch.meshgrid(
        *[torch.arange(G, dtype=torch.int32, device="cuda")] * 3, indexing="ij"), -1).reshape(-1, 3))
    model.mark_invisible_cells(train.K, train.poses, train.img_wh)
    tr = Trainer(model, n_rays=4096, erode=True, bg=(1.0, 1.0, 1.0))
    assert (model.density_grid < 0).any() and (model.density_grid == 0).any()
    tr.attach_bank(train)
    before = metrics.evaluate(model, test.poses, test.directions, test.rgb, test.img_wh)["psnr"]
    tr.capture()
    losses = []
    for k in range(400):
        tr.train_step()
        if k % 100 == 99:
            torch.cuda.synchronize()
            losses.append(tr.stats()["loss"])
    after = metrics.evaluate(model, test.poses, test.directions, test.rgb, test.img_wh)["psnr"]
    print("colmap fixture: test PSNR %.2f -> %.2f, losses %s" % (before, after, losses))
    assert all(np.isfinite(losses)) and after > before + 3
