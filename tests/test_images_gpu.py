"""ngp_view_images and ngp_png_encode (csrc/images.cu), images.py and metrics.evaluate(save_dir=) on the device:
the images bitwise against the reference's depth2img goldens and oracle/images_ref.py, the PNG bytes against the host
restatement oracle/png_ref.py, every file decoded by oracle/png_ref.decode and by Pillow."""
import ctypes as C
import io
import os
import socket

import numpy as np
import pytest
import torch

from oracle import images_ref as R
from oracle import png_ref as P
from test_images_cpu import GOLDEN, KINDS, SIZES, make_image

pytestmark = pytest.mark.gpu


def _pillow(data):
    from PIL import Image
    with Image.open(io.BytesIO(data)) as im:
        assert im.mode == "RGB"
        return np.array(im)


def _lego_view(W, H, seed=4321, n=1):
    """a Lego model (tests/test_render_gpu.make_model) and its test-time renders of n seeded views at W x H"""
    from ngp_pl_b200 import synth
    from ngp_pl_b200.models.rendering import render
    from test_render_gpu import make_model
    scene = synth.lego_scene(0)
    model = make_model(scene)
    K = synth.intrinsics(W=W, H=H, fx=1111.11 * W / 800)
    dirs = synth.ray_directions(K, "cuda")
    poses = torch.as_tensor(synth.camera_poses(n, seed=seed)).cuda()
    outs = [render(model, *synth.get_rays(dirs, poses[i]), test_time=True) for i in range(n)]
    return model, dirs, poses, outs, scene


def test_depth_images_equal_reference_goldens():
    from ngp_pl_b200 import images
    z = np.load(GOLDEN)
    for k in z.files:
        if not k.startswith("depth_"):
            continue
        d = z[k]
        got = images.depth_image(torch.as_tensor(d).cuda().reshape(-1), *d.shape)
        assert got.is_cuda and got.dtype == torch.uint8 and tuple(got.shape) == z["img_" + k[6:]].shape
        assert np.array_equal(got.cpu().numpy(), z["img_" + k[6:]]), k


def test_rgb_image_is_numpy_cast():
    from ngp_pl_b200 import images
    H, W = 37, 29
    rng = np.random.RandomState(3)
    rgb = (rng.rand(H * W, 3) * (256 / 255)).astype(np.float32)
    rgb[:256, 0] = np.arange(256, dtype=np.float32) / np.float32(255)  # every exact level
    rgb[:256, 1] = np.nextafter(rgb[:256, 0], np.float32(0))
    rgb[5, 2] = np.nan
    rgb[6, 2] = np.nextafter(np.float32(256 / 255), np.float32(0))
    got = images.rgb_image(torch.as_tensor(rgb).cuda(), H, W).cpu().numpy()
    assert np.array_equal(got, R.rgb_image(rgb, H, W))


def test_view_images_of_a_render_equal_images_ref():
    from ngp_pl_b200 import images
    W, H = 120, 90
    _, _, _, outs, _ = _lego_view(W, H, n=2)
    for out in outs:
        rgb, depth = out["rgb"].float(), out["depth"].float()
        assert float(depth.max()) > float(depth.min())
        a, b = images.view_images(rgb, depth, H, W)
        assert np.array_equal(a.cpu().numpy(), R.rgb_image(rgb.cpu().numpy(), H, W))
        assert np.array_equal(b.cpu().numpy(), R.depth_image(depth.cpu().numpy(), H, W))
        assert np.array_equal(images.depth_image(depth, H, W).cpu().numpy(), b.cpu().numpy())


@pytest.mark.parametrize("H,W", SIZES + [(3, 6000), (2, 22000)])  # 2L > 32768; L > 32768 and > 65535 (split stored)
@pytest.mark.parametrize("kind", KINDS)
def test_png_bytes_equal_restatement(H, W, kind):
    from ngp_pl_b200 import images
    img = make_image(H, W, kind)
    got = images.encode_png(torch.as_tensor(img).cuda())
    want = P.encode(img)
    assert len(got) == len(want) and got == want


def test_png_bytes_of_a_small_render_equal_restatement():
    from ngp_pl_b200 import images
    W, H = 64, 48
    _, _, _, outs, _ = _lego_view(W, H)
    a, b = images.view_images(outs[0]["rgb"].float(), outs[0]["depth"].float(), H, W)
    for img in (a, b):
        assert images.encode_png(img) == P.encode(img.cpu().numpy())


def _encode_raw(img, out, n, ws):
    from ngp_pl_b200 import images
    images.encode_png_into(img, out, n, ws)
    torch.cuda.synchronize()
    return int(n[0])


def test_png_800_decodes_is_repeatable_and_mapped_equals_device():
    from ngp_pl_b200 import images
    H = W = 800
    _, _, _, outs, _ = _lego_view(W, H)
    rgb_img, depth_img = images.view_images(outs[0]["rgb"].float(), outs[0]["depth"].float(), H, W)
    cap = images.png_capacity(H, W)
    ws = images.png_workspace(H, W, "cuda")
    for name, img in (("noise", torch.as_tensor(make_image(H, W, "noise")).cuda()),
                      ("flat", torch.as_tensor(make_image(H, W, "flat")).cuda()),
                      ("rgb", rgb_img), ("depth", depth_img)):
        host = img.cpu().numpy()
        out_d = torch.full((cap,), 0xAB, dtype=torch.uint8, device="cuda")
        n_d = torch.zeros(1, dtype=torch.int64, device="cuda")
        n1 = _encode_raw(img, out_d, n_d, ws)
        first = out_d[:n1].cpu().numpy().tobytes()
        n2 = _encode_raw(img, out_d, n_d, ws)
        assert n2 == n1 and out_d[:n2].cpu().numpy().tobytes() == first, name  # two calls, same bytes
        assert bool((out_d[n1:] == 0xAB).all()), name  # nothing written past the file's length
        out_h = torch.zeros(cap, dtype=torch.uint8, pin_memory=True)
        n_h = torch.zeros(1, dtype=torch.int64, pin_memory=True)
        assert _encode_raw(img, out_h, n_h, ws) == n1
        assert out_h[:n1].numpy().tobytes() == first, name  # mapped pinned memory == device memory
        assert first.endswith(b"\x00\x00\x00\x00IEND\xaeB`\x82") and n1 <= cap
        assert np.array_equal(P.decode(first), host), name  # P.decode also requires the file to end at n1
        assert np.array_equal(_pillow(first), host), name
        print("%s 800x800: %d bytes (capacity %d)" % (name, n1, cap))


def test_bad_arguments_return_einval():
    from ngp_pl_b200 import _lib
    lib = _lib.lib()
    st = torch.cuda.current_stream().cuda_stream
    H, W = 8, 6
    rgb = torch.rand(H * W, 3, device="cuda")
    depth = torch.rand(H * W, device="cuda")
    a = torch.empty(H, W, 3, dtype=torch.uint8, device="cuda")
    b = torch.empty_like(a)
    vws = torch.empty(4096, dtype=torch.uint8, device="cuda")
    host = np.zeros(H * W * 3, np.float32)
    hp = host.ctypes.data
    V = lambda *args: lib.ngp_view_images(*args, st)  # noqa: E731
    assert V(rgb.data_ptr(), depth.data_ptr(), H, W, a.data_ptr(), b.data_ptr(), vws.data_ptr(), 4096) == 0
    torch.cuda.synchronize()
    bad = [
        (rgb.data_ptr(), depth.data_ptr(), 0, W, a.data_ptr(), b.data_ptr(), vws.data_ptr(), 4096),
        (rgb.data_ptr(), depth.data_ptr(), H, 0, a.data_ptr(), b.data_ptr(), vws.data_ptr(), 4096),
        (rgb.data_ptr(), depth.data_ptr(), H, W, None, None, vws.data_ptr(), 4096),
        (None, depth.data_ptr(), H, W, a.data_ptr(), b.data_ptr(), vws.data_ptr(), 4096),
        (rgb.data_ptr(), None, H, W, a.data_ptr(), b.data_ptr(), vws.data_ptr(), 4096),
        (hp, depth.data_ptr(), H, W, a.data_ptr(), b.data_ptr(), vws.data_ptr(), 4096),
        (rgb.data_ptr(), hp, H, W, a.data_ptr(), b.data_ptr(), vws.data_ptr(), 4096),
        (rgb.data_ptr(), depth.data_ptr(), H, W, hp, b.data_ptr(), vws.data_ptr(), 4096),
        (rgb.data_ptr(), depth.data_ptr(), H, W, a.data_ptr(), b.data_ptr(), None, 4096),
        (rgb.data_ptr(), depth.data_ptr(), H, W, a.data_ptr(), b.data_ptr(), vws.data_ptr(), 4095),
        (rgb.data_ptr(), depth.data_ptr(), H, W, a.data_ptr(), b.data_ptr(), vws.data_ptr() + 4, 4092),
    ]
    for i, args in enumerate(bad):
        assert V(*args) == -22, i
    # the rgb image alone needs no workspace
    assert V(rgb.data_ptr(), None, H, W, a.data_ptr(), None, None, 0) == 0

    cap = lib.ngp_png_capacity(H, W)
    wsz = lib.ngp_png_workspace(H, W)
    ws = torch.empty(wsz + 256, dtype=torch.uint8, device="cuda")
    out = torch.empty(cap, dtype=torch.uint8, device="cuda")
    n = torch.zeros(2, dtype=torch.int64, device="cuda")
    E = lambda *args: lib.ngp_png_encode(*args, st)  # noqa: E731
    ok = [a.data_ptr(), H, W, out.data_ptr(), cap, n.data_ptr(), ws.data_ptr(), wsz]
    assert E(*ok) == 0
    torch.cuda.synchronize()
    hbuf = (C.c_uint8 * cap)()  # pageable host memory: not reachable from the device
    changes = [(0, None), (0, hp), (1, 0), (2, 0), (1, -3), (2, 1 << 20), (3, None), (3, C.addressof(hbuf)), (4, cap - 1),
               (5, None), (5, n.data_ptr() + 4), (6, None), (6, ws.data_ptr() + 16), (7, wsz - 1)]
    for k, v in changes:
        args = list(ok)
        args[k] = v
        assert E(*args) == -22, (k, v)
    assert lib.ngp_png_capacity(1 << 20, 1 << 12) == 0  # an IDAT over 2^31 - 1 bytes
    big = [a.data_ptr(), 1 << 20, 1 << 12, out.data_ptr(), cap, n.data_ptr(), ws.data_ptr(), wsz]
    assert E(*big) == -22


def _files(d):
    return sorted(os.listdir(d))


def _check_saved(d, idx, outs, H, W):
    assert _files(d) == sorted(["%03d.png" % i for i in idx] + ["%03d_d.png" % i for i in idx])
    for i, out in zip(idx, outs):
        rgb = open(os.path.join(d, "%03d.png" % i), "rb").read()
        dep = open(os.path.join(d, "%03d_d.png" % i), "rb").read()
        want_rgb = R.rgb_image(out["rgb"].float().cpu().numpy(), H, W)
        want_dep = R.depth_image(out["depth"].float().cpu().numpy(), H, W)
        assert np.array_equal(P.decode(rgb), want_rgb) and np.array_equal(_pillow(rgb), want_rgb)
        assert np.array_equal(P.decode(dep), want_dep) and np.array_equal(_pillow(dep), want_dep)


@pytest.mark.parametrize("with_lpips", [False, True])
def test_evaluate_save_dir(tmp_path, with_lpips):
    from ngp_pl_b200 import metrics, synth
    from ngp_pl_b200.models.rendering import render
    W, H = 64, 48
    n = 5  # more views than the writer has slots
    model, dirs, poses, _, scene = _lego_view(W, H, n=n)
    images = torch.stack([(synth.trace(scene, *synth.get_rays(dirs, poses[i])) * 255).round().to(torch.uint8)
                          for i in range(n)])
    net = None
    if with_lpips:
        from oracle import lpips_ref
        vgg, lin = lpips_ref.random_weights(7)
        net = metrics.LpipsNet.from_state_dicts(lpips_ref.fp16_convs(vgg), lin, "cuda")
    outs = []

    def render_fn(o, d):
        outs.append(render(model, o, d, test_time=True))
        return outs[-1]
    d = str(tmp_path / "results" / "lego")  # created by evaluate
    res = metrics.evaluate(render_fn, poses, dirs, images, (W, H), lpips_net=net, save_dir=d)
    replay = iter(outs)
    plain = metrics.evaluate(lambda o, dd: next(replay), poses, dirs, images, (W, H), lpips_net=net)
    assert res == plain
    assert ("lpips" in res) == with_lpips
    _check_saved(d, range(n), outs, H, W)


def test_evaluate_save_dir_needs_depth(tmp_path):
    from ngp_pl_b200 import metrics
    W, H = 32, 24
    model, dirs, poses, outs, _ = _lego_view(W, H)
    images = torch.zeros(1, H * W, 3, dtype=torch.uint8, device="cuda")
    with pytest.raises(RuntimeError, match="depth"):
        metrics.evaluate(lambda o, d: {"rgb": outs[0]["rgb"], "total_samples": outs[0]["total_samples"]}, poses, dirs,
                         images, (W, H), save_dir=str(tmp_path / "x"))


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
    from ngp_pl_b200.models.rendering import render
    W, H = 40, 30
    model, dirs, poses, _, _ = _lego_view(W, H, n=N_VIEWS)
    images = torch.zeros(N_VIEWS, H * W, 3, dtype=torch.uint8, device="cuda")
    outs = []

    def render_fn(o, d):
        outs.append(render(model, o, d, test_time=True))
        return outs[-1]
    res = metrics.evaluate(render_fn, poses, dirs, images, (W, H), world_size=world, rank=rank,
                           save_dir=os.path.join(root, "rank%d" % rank))
    torch.save({"res": res, "outs": [{k: v.cpu() for k, v in o.items()} for o in outs]},
               os.path.join(root, "r%d.pt" % rank))
    dist.destroy_process_group()


def test_two_ranks_write_their_shards(tmp_path):
    import torch.multiprocessing as mp
    from ngp_pl_b200.trainer import shard_range
    root = str(tmp_path)
    mp.spawn(_rank_worker, args=(2, _free_port(), root), nprocs=2, join=True)
    W, H = 40, 30
    results = []
    for r in range(2):
        lo, hi = shard_range(N_VIEWS, 2, r)
        got = torch.load(os.path.join(root, "r%d.pt" % r))
        assert len(got["outs"]) == hi - lo
        _check_saved(os.path.join(root, "rank%d" % r), range(lo, hi), got["outs"], H, W)
        results.append(got["res"])
    assert results[0] == results[1] and len(results[0]["psnr_per_view"]) == N_VIEWS
