"""ngp_png_encode_mode (csrc/images.cu) on the device: NGP_PNG_DYNAMIC bytes against the host restatement
oracle/png_dynamic_ref.py, NGP_PNG_FIXED against ngp_png_encode, argument refusal, and
metrics.evaluate(save_dir=, png_mode="dynamic") against the default mode on a briefly trained model."""
import ctypes as C
import glob
import os
import socket

import numpy as np
import pytest
import torch

from oracle import images_ref as R
from oracle import png_dynamic_ref as D
from oracle import png_ref as P
from test_images_cpu import GOLDEN, ROOT
from test_png_dynamic_cpu import SIZES, make

pytestmark = pytest.mark.gpu


def _pillow(data):
    import io
    from PIL import Image
    with Image.open(io.BytesIO(data)) as im:
        return np.array(im)


def _renders(W, H, n=1, seed=4321):
    from ngp_pl_b200 import synth
    from ngp_pl_b200.models.rendering import render
    from test_render_gpu import make_model
    model = make_model(synth.lego_scene(0))
    dirs = synth.ray_directions(synth.intrinsics(W=W, H=H, fx=1111.11 * W / 800), "cuda")
    poses = torch.as_tensor(synth.camera_poses(n, seed=seed)).cuda()
    return [render(model, *synth.get_rays(dirs, poses[i]), test_time=True) for i in range(n)]


def _trained(W, H, n_views, steps=60):
    """a Lego model after a few captured training steps, its ray directions, view poses and ground truth"""
    from ngp_pl_b200 import synth
    from ngp_pl_b200.models.networks import NGP
    from ngp_pl_b200.trainer import Trainer
    torch.manual_seed(0)
    scene = synth.lego_scene(0)
    bank = synth.RayBank(scene, n_images=8, device="cuda", seed=0)
    model = NGP(scene.scale).cuda()
    tr = Trainer(model, n_rays=2048, lr=1e-2)
    tr.attach_bank(bank)
    tr.capture(sample=True)
    for _ in range(steps):
        tr.train_step()
    torch.cuda.synchronize()
    del tr, bank
    dirs = synth.ray_directions(synth.intrinsics(W=W, H=H, fx=1111.11 * W / 800), "cuda")
    poses = torch.as_tensor(synth.camera_poses(n_views, seed=4321)).cuda()
    gts = torch.stack([(synth.trace(scene, *synth.get_rays(dirs, poses[i])) * 255).round().to(torch.uint8)
                       for i in range(n_views)])
    return model, dirs, poses, gts


@pytest.mark.parametrize("H,W", SIZES)
@pytest.mark.parametrize("kind", ["noise", "flat", "gradient", "smooth"])
def test_dynamic_bytes_equal_restatement(H, W, kind):
    from ngp_pl_b200 import images
    img = make(H, W, kind)
    assert images.encode_png(torch.as_tensor(img).cuda(), mode="dynamic") == D.encode(img)


def test_dynamic_bytes_of_goldens_fixtures_and_a_render_equal_restatement():
    from PIL import Image
    from ngp_pl_b200 import images
    z = np.load(GOLDEN)
    imgs = [z[k] for k in z.files if k.startswith("img_")]
    for p in sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "datasets", "*", "*", "*.png")))[:8]:
        with Image.open(p) as im:
            imgs.append(np.ascontiguousarray(np.array(im.convert("RGB"))))
    W, H = 64, 48
    out = _renders(W, H)[0]
    a, b = images.view_images(out["rgb"].float(), out["depth"].float(), H, W)
    imgs += [a.cpu().numpy(), b.cpu().numpy()]
    for i, img in enumerate(imgs):
        assert images.encode_png(torch.as_tensor(img).cuda(), mode="dynamic") == D.encode(img), i


def _encode_raw(img, out, n, ws, mode):
    from ngp_pl_b200 import images
    images.encode_png_into(img, out, n, ws, mode)
    torch.cuda.synchronize()
    return int(n[0])


def test_800_is_repeatable_mapped_equals_device_and_fixed_equals_ngp_png_encode():
    from ngp_pl_b200 import _lib, images
    H = W = 800
    out = _renders(W, H)[0]
    rgb_img, depth_img = images.view_images(out["rgb"].float(), out["depth"].float(), H, W)
    cap = images.png_capacity(H, W)
    ws = images.png_workspace(H, W, "cuda", "dynamic")
    ws_fixed = images.png_workspace(H, W, "cuda")
    lib = _lib.lib()
    st = torch.cuda.current_stream().cuda_stream
    for name, img in (("noise", torch.as_tensor(make(H, W, "noise")).cuda()),
                      ("flat", torch.as_tensor(make(H, W, "flat")).cuda()),
                      ("rgb", rgb_img), ("depth", depth_img)):
        host = img.cpu().numpy()
        out_d = torch.full((cap,), 0xAB, dtype=torch.uint8, device="cuda")
        n_d = torch.zeros(1, dtype=torch.int64, device="cuda")
        n1 = _encode_raw(img, out_d, n_d, ws, "dynamic")
        first = out_d[:n1].cpu().numpy().tobytes()
        assert _encode_raw(img, out_d, n_d, ws, "dynamic") == n1
        assert out_d[:n1].cpu().numpy().tobytes() == first, name
        assert bool((out_d[n1:] == 0xAB).all()), name
        out_h = torch.zeros(cap, dtype=torch.uint8, pin_memory=True)
        n_h = torch.zeros(1, dtype=torch.int64, pin_memory=True)
        assert _encode_raw(img, out_h, n_h, ws, "dynamic") == n1
        assert out_h[:n1].numpy().tobytes() == first, name
        assert first == D.encode(host), name
        assert np.array_equal(P.decode(first), host) and np.array_equal(_pillow(first), host), name
        # NGP_PNG_FIXED through the new entry point is ngp_png_encode's file
        want = torch.zeros(cap, dtype=torch.uint8, device="cuda")
        assert lib.ngp_png_encode(img.data_ptr(), H, W, want.data_ptr(), cap, n_d.data_ptr(), ws_fixed.data_ptr(),
                                  ws_fixed.numel(), st) == 0
        torch.cuda.synchronize()
        n_f = int(n_d[0])
        fixed = _encode_raw(img, out_h, n_h, ws_fixed, "fixed")
        assert fixed == n_f and out_h[:n_f].numpy().tobytes() == want[:n_f].cpu().numpy().tobytes(), name
        assert n1 <= n_f, name
        print("%s 800x800: dynamic %d bytes, fixed %d (capacity %d)" % (name, n1, n_f, cap))


def test_bad_arguments_return_einval():
    from ngp_pl_b200 import _lib
    lib = _lib.lib()
    st = torch.cuda.current_stream().cuda_stream
    H, W = 40, 6
    a = torch.randint(0, 256, (H, W, 3), dtype=torch.uint8, device="cuda")
    cap = lib.ngp_png_capacity(H, W)
    wsz = lib.ngp_png_workspace_mode(H, W, 1)
    assert wsz > lib.ngp_png_workspace(H, W) == lib.ngp_png_workspace_mode(H, W, 0)
    for m in (-1, 2, 7):
        assert lib.ngp_png_workspace_mode(H, W, m) == 0
    for args in ((0, 5), (5, 0), (1 << 20, 1 << 12)):
        assert lib.ngp_png_workspace_mode(*args, 1) == 0
    ws = torch.empty(wsz + 256, dtype=torch.uint8, device="cuda")
    out = torch.empty(cap, dtype=torch.uint8, device="cuda")
    n = torch.zeros(2, dtype=torch.int64, device="cuda")
    E = lambda *args: lib.ngp_png_encode_mode(*args, st)  # noqa: E731
    ok = [a.data_ptr(), H, W, 1, out.data_ptr(), cap, n.data_ptr(), ws.data_ptr(), wsz]
    assert E(*ok) == 0
    torch.cuda.synchronize()
    host = np.zeros(H * W * 3, np.uint8)
    hbuf = (C.c_uint8 * cap)()
    changes = [(0, None), (0, host.ctypes.data), (1, 0), (2, 0), (1, -3), (2, 1 << 20), (3, -1), (3, 2), (4, None),
               (4, C.addressof(hbuf)), (5, cap - 1), (6, None), (6, n.data_ptr() + 4), (7, None), (7, ws.data_ptr() + 16),
               (8, wsz - 1)]
    for k, v in changes:
        args = list(ok)
        args[k] = v
        assert E(*args) == -22, (k, v)
    big = [a.data_ptr(), 1 << 20, 1 << 12, 1, out.data_ptr(), cap, n.data_ptr(), ws.data_ptr(), wsz]
    assert E(*big) == -22


def test_unknown_mode_strings_raise_value_error(tmp_path):
    from ngp_pl_b200 import images, metrics
    img = torch.zeros(2, 2, 3, dtype=torch.uint8, device="cuda")
    for fn in (lambda: images.encode_png(img, mode="zlib"), lambda: images.png_workspace(2, 2, "cuda", "Dynamic"),
               lambda: images.write_png(str(tmp_path / "a.png"), img, mode=1),
               lambda: images.ViewWriter(str(tmp_path / "v"), 2, 2, "cuda", png_mode="best"),
               lambda: metrics.evaluate(None, torch.zeros(1, 3, 4, device="cuda"), torch.zeros(4, 3, device="cuda"),
                                        torch.zeros(1, 4, 3, dtype=torch.uint8, device="cuda"), (2, 2), png_mode="x")):
        with pytest.raises(ValueError):
            fn()
    assert not os.path.exists(tmp_path / "a.png")


def _compare_dirs(d_fixed, d_dyn, idx):
    names = sorted(["%03d.png" % i for i in idx] + ["%03d_d.png" % i for i in idx])
    assert sorted(os.listdir(d_fixed)) == names and sorted(os.listdir(d_dyn)) == names
    for name in names:
        a = open(os.path.join(d_fixed, name), "rb").read()
        b = open(os.path.join(d_dyn, name), "rb").read()
        assert np.array_equal(P.decode(b), P.decode(a)) and np.array_equal(_pillow(b), P.decode(a)), name
        assert len(b) < len(a), (name, len(b), len(a))


def test_evaluate_dynamic_files_decode_to_the_default_arrays(tmp_path):
    from ngp_pl_b200 import metrics
    from ngp_pl_b200.models.rendering import render
    W, H, n = 96, 72, 5
    model, dirs, poses, gts = _trained(W, H, n)
    outs = []

    def render_fn(o, d):
        outs.append(render(model, o, d, test_time=True))
        return outs[-1]
    d0, d1 = str(tmp_path / "fixed"), str(tmp_path / "dynamic")
    r1 = metrics.evaluate(render_fn, poses, dirs, gts, (W, H), save_dir=d1, png_mode="dynamic")
    replay = iter(outs)
    r0 = metrics.evaluate(lambda o, d: next(replay), poses, dirs, gts, (W, H), save_dir=d0)
    replay = iter(outs)
    assert r1 == r0 == metrics.evaluate(lambda o, d: next(replay), poses, dirs, gts, (W, H))
    _compare_dirs(d0, d1, range(n))
    for i, out in enumerate(outs):
        rgb = open(os.path.join(d1, "%03d.png" % i), "rb").read()
        dep = open(os.path.join(d1, "%03d_d.png" % i), "rb").read()
        assert np.array_equal(P.decode(rgb), R.rgb_image(out["rgb"].float().cpu().numpy(), H, W))
        assert np.array_equal(P.decode(dep), R.depth_image(out["depth"].float().cpu().numpy(), H, W))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


N_VIEWS = 5  # shards of 3 and 2


def _rank_worker(rank, world, port, root):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.cuda.set_device(0)
    from ngp_pl_b200 import metrics
    W, H = 48, 36
    model, dirs, poses, gts = _trained(W, H, N_VIEWS, steps=30)
    res = {}
    for mode in ("fixed", "dynamic"):
        res[mode] = metrics.evaluate(model, poses, dirs, gts, (W, H), world_size=world, rank=rank,
                                     save_dir=os.path.join(root, mode, "rank%d" % rank), png_mode=mode)
    torch.save(res, os.path.join(root, "r%d.pt" % rank))
    dist.destroy_process_group()


def test_two_ranks_write_their_dynamic_shards(tmp_path):
    import torch.multiprocessing as mp
    from ngp_pl_b200.trainer import shard_range
    root = str(tmp_path)
    mp.spawn(_rank_worker, args=(2, _free_port(), root), nprocs=2, join=True)
    for r in range(2):
        lo, hi = shard_range(N_VIEWS, 2, r)
        got = torch.load(os.path.join(root, "r%d.pt" % r))
        assert got["fixed"] == got["dynamic"] and len(got["dynamic"]["psnr_per_view"]) == N_VIEWS
        _compare_dirs(os.path.join(root, "fixed", "rank%d" % r), os.path.join(root, "dynamic", "rank%d" % r),
                      range(lo, hi))
