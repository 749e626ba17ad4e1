"""ngp_jpeg_encode (csrc/jpeg.cu) and the videos of images.py / metrics.evaluate(video_fps=) on the device: the JPEG bytes
against the host restatement oracle/jpeg_ref.py (which tests/test_jpeg_cpu.py pins to libjpeg), the AVI files frame by
frame against encode_jpeg of the same images."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import jpeg_ref as J
from test_images_gpu import _free_port, _lego_view
from test_jpeg_cpu import KINDS, QUALITIES, SIZES, make_image, parse_avi, pillow_decode

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("quality", QUALITIES)
@pytest.mark.parametrize("kind", KINDS)
def test_jpeg_bytes_equal_restatement(kind, quality):
    from ngp_pl_b200 import images
    for H, W in SIZES:
        img = make_image(H, W, kind)
        got = images.encode_jpeg(torch.as_tensor(img).cuda(), quality)
        want = J.encode(img, quality)
        assert len(got) == len(want) and got == want, (H, W)


def _encode_raw(img, out, n, ws, quality):
    from ngp_pl_b200 import images
    images.encode_jpeg_into(img, out, n, ws, quality)
    torch.cuda.synchronize()
    return int(n[0])


def test_jpeg_800_equals_restatement_is_repeatable_and_mapped_equals_device():
    from ngp_pl_b200 import images
    H = W = 800
    _, _, _, outs, _ = _lego_view(W, H)
    rgb_img, depth_img = images.view_images(outs[0]["rgb"].float(), outs[0]["depth"].float(), H, W)
    cap = images.jpeg_capacity(H, W)
    ws = images.jpeg_workspace(H, W, "cuda")
    for name, img, quality in (("noise", torch.as_tensor(make_image(H, W, "noise")).cuda(), 100),
                               ("checker", torch.as_tensor(make_image(H, W, "checker")).cuda(), 1),
                               ("rgb", rgb_img, 90), ("depth", depth_img, 90)):
        host = img.cpu().numpy()
        out_d = torch.full((cap,), 0xAB, dtype=torch.uint8, device="cuda")
        n_d = torch.zeros(1, dtype=torch.int64, device="cuda")
        n1 = _encode_raw(img, out_d, n_d, ws, quality)
        first = out_d[:n1].cpu().numpy().tobytes()
        assert first == J.encode(host, quality), name
        n2 = _encode_raw(img, out_d, n_d, ws, quality)
        assert n2 == n1 and out_d[:n2].cpu().numpy().tobytes() == first, name  # two calls, same bytes
        assert bool((out_d[n1:] == 0xAB).all()), name  # nothing written past the file's length
        out_h = torch.zeros(cap, dtype=torch.uint8, pin_memory=True)
        n_h = torch.zeros(1, dtype=torch.int64, pin_memory=True)
        assert _encode_raw(img, out_h, n_h, ws, quality) == n1
        assert out_h[:n1].numpy().tobytes() == first, name  # mapped pinned memory == device memory
        assert n1 <= cap
        dec = pillow_decode(first, H, W)
        if quality == 90:
            assert np.abs(dec.astype(np.int32) - host).mean() < 2, name
        print("%s 800x800 at quality %d: %d bytes (capacity %d)" % (name, quality, n1, cap))


def test_bad_arguments_return_einval():
    from ngp_pl_b200 import _lib, images
    lib = _lib.lib()
    st = torch.cuda.current_stream().cuda_stream
    H, W = 9, 6
    a = torch.zeros(H, W, 3, dtype=torch.uint8, device="cuda")
    cap = lib.ngp_jpeg_capacity(H, W)
    wsz = lib.ngp_jpeg_workspace(H, W)
    assert cap == 623 + 416 * 3 * 2 + 2
    ws = torch.empty(wsz + 256, dtype=torch.uint8, device="cuda")
    out = torch.empty(cap, dtype=torch.uint8, device="cuda")
    n = torch.zeros(2, dtype=torch.int64, device="cuda")
    host = np.zeros(H * W * 3, np.uint8)
    hbuf = (C.c_uint8 * cap)()  # pageable host memory: not reachable from the device
    E = lambda *args: lib.ngp_jpeg_encode(*args, st)  # noqa: E731
    ok = [a.data_ptr(), H, W, 90, out.data_ptr(), cap, n.data_ptr(), ws.data_ptr(), wsz]
    assert E(*ok) == 0
    torch.cuda.synchronize()
    changes = [(0, None), (0, host.ctypes.data), (1, 0), (2, 0), (1, -3), (1, 65536), (2, 1 << 20), (3, 0), (3, 101),
               (3, -5), (4, None), (4, C.addressof(hbuf)), (5, cap - 1), (6, None), (6, n.data_ptr() + 4), (7, None),
               (7, ws.data_ptr() + 16), (8, wsz - 1)]
    for k, v in changes:
        args = list(ok)
        args[k] = v
        assert E(*args) == -22, (k, v)
    assert lib.ngp_jpeg_capacity(6000, 6000) == 0 and lib.ngp_jpeg_workspace(6000, 6000) == 0  # over 2^31 - 1 coded bits
    assert lib.ngp_jpeg_capacity(5000, 5000) > 0
    assert E(a.data_ptr(), 6000, 6000, 90, out.data_ptr(), cap, n.data_ptr(), ws.data_ptr(), wsz) == -22
    with pytest.raises(RuntimeError):
        images.jpeg_capacity(0, 5)
    with pytest.raises(RuntimeError, match="invalid argument"):
        images.encode_jpeg(a, quality=0)


def _frames(path):
    data = open(path, "rb").read()
    a = parse_avi(data)
    return a, [data[p:p + n] for p, n in a["frames"]]


def _check_videos(d, tag, outs, H, W, fps, quality):
    from ngp_pl_b200 import images
    for name, key in (("rgb", 0), ("depth", 1)):
        a, frames = _frames(os.path.join(d, "%s%s.avi" % (name, tag)))
        assert a["strh"][6:8] == (1, fps) and a["avih"][8:10] == (W, H) and len(frames) == len(outs)
        for f, out in zip(frames, outs):
            img = images.view_images(out["rgb"].float().cuda(), out["depth"].float().cuda(), H, W)[key]
            assert f == images.encode_jpeg(img, quality)
            assert f == J.encode(img.cpu().numpy(), quality)


def test_evaluate_video(tmp_path):
    from ngp_pl_b200 import metrics, synth
    from ngp_pl_b200.models.rendering import render
    W, H = 64, 48
    n = 6  # more views than the writer has slots
    model, dirs, poses, _, scene = _lego_view(W, H, n=n)
    gt = torch.stack([(synth.trace(scene, *synth.get_rays(dirs, poses[i])) * 255).round().to(torch.uint8) for i in range(n)])
    outs = []

    def render_fn(o, d):
        outs.append(render(model, o, d, test_time=True))
        return outs[-1]
    d_video, d_plain = str(tmp_path / "video"), str(tmp_path / "plain")
    res = metrics.evaluate(render_fn, poses, dirs, gt, (W, H), save_dir=d_video, video_fps=30, video_quality=85)
    replay = iter(outs)
    plain = metrics.evaluate(lambda o, dd: next(replay), poses, dirs, gt, (W, H), save_dir=d_plain)
    assert res == plain
    pngs = sorted(os.listdir(d_plain))
    assert len(pngs) == 2 * n and sorted(os.listdir(d_video)) == sorted(pngs + ["rgb.avi", "depth.avi"])
    for name in pngs:
        assert open(os.path.join(d_video, name), "rb").read() == open(os.path.join(d_plain, name), "rb").read(), name
    _check_videos(d_video, "", outs, H, W, 30, 85)
    with pytest.raises(RuntimeError, match="save_dir"):
        metrics.evaluate(render_fn, poses, dirs, gt, (W, H), video_fps=30)


def test_render_video(tmp_path):
    from ngp_pl_b200 import images, synth
    from ngp_pl_b200.models.rendering import render
    W, H = 56, 40
    model, dirs, _, _, _ = _lego_view(W, H)
    poses = torch.as_tensor(synth.camera_poses(5, seed=11)).cuda()
    d = str(tmp_path / "path")
    images.render_video(model, poses, dirs, (W, H), d, fps=24)
    assert sorted(os.listdir(d)) == ["depth.avi", "rgb.avi"]
    outs = [render(model, *synth.get_rays(dirs, poses[i]), test_time=True) for i in range(5)]
    _check_videos(d, "", outs, H, W, 24, 90)


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
    gt = torch.zeros(N_VIEWS, H * W, 3, dtype=torch.uint8, device="cuda")
    outs = []

    def render_fn(o, d):
        outs.append(render(model, o, d, test_time=True))
        return outs[-1]
    metrics.evaluate(render_fn, poses, dirs, gt, (W, H), world_size=world, rank=rank, save_dir=os.path.join(root, "out"),
                     video_fps=30)
    torch.save([{k: v.cpu() for k, v in o.items()} for o in outs], os.path.join(root, "r%d.pt" % rank))
    dist.destroy_process_group()


def test_two_ranks_write_their_video_shards(tmp_path):
    import torch.multiprocessing as mp
    from ngp_pl_b200.trainer import shard_range
    root = str(tmp_path)
    mp.spawn(_rank_worker, args=(2, _free_port(), root), nprocs=2, join=True)
    W, H = 40, 30
    d = os.path.join(root, "out")
    assert sorted(f for f in os.listdir(d) if f.endswith(".avi")) == ["depth.rank0.avi", "depth.rank1.avi", "rgb.rank0.avi",
                                                                      "rgb.rank1.avi"]
    assert len([f for f in os.listdir(d) if f.endswith(".png")]) == 2 * N_VIEWS
    total = 0
    for r in range(2):
        lo, hi = shard_range(N_VIEWS, 2, r)
        outs = torch.load(os.path.join(root, "r%d.pt" % r))
        assert len(outs) == hi - lo
        _check_videos(d, ".rank%d" % r, outs, H, W, 30, 90)
        total += len(outs)
    assert total == N_VIEWS
