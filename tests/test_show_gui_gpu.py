"""ngp_render_view_frame (csrc/infer.cu) and show_gui's ViewRenderer / server on the device: the frame's rays bitwise
ngp_gen_rays', its outputs bitwise ngp_render_infer_frame's on those rays, its JPEG bitwise encode_jpeg of
view_images and oracle/jpeg_ref.py, no graph rebuild while the camera moves or the mode toggles, the refused arguments,
and `python -m ngp_pl_b200.show_gui`'s server end to end on a model the command-line trainer wrote."""
import ctypes as C
import http.client
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import jpeg_ref as J

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIX = os.path.join(ROOT, "tests", "golden", "datasets")
SIZES = [(800, 800), (41, 29)]  # (W, H)


def _intrinsics(W, H):
    f = 1111.11 * W / 800
    return np.float32([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]])


def _renderer(W, H, quality=90):
    """a ViewRenderer of the Lego model of tests/test_render_gpu.make_model at W x H"""
    from ngp_pl_b200 import synth
    from ngp_pl_b200.show_gui import ViewRenderer
    from test_render_gpu import make_model
    model = make_model(synth.lego_scene(0))
    K = _intrinsics(W, H)
    return ViewRenderer(model, K, (W, H), 0.0, quality), K


def _poses(K, W, H, n, seed):
    """n orbit-camera poses around the Lego model"""
    from ngp_pl_b200.show_gui import OrbitCamera
    rng = np.random.RandomState(seed)
    cam = OrbitCamera(K, (W, H), 1.6)
    cam.orbit(0, -600)  # look down on the model a little
    out = []
    for _ in range(n):
        cam.orbit(*rng.uniform(-300, 300, 2))
        cam.pan(*rng.uniform(-800, 800, 2))
        cam.scale(rng.uniform(-1, 1))
        out.append(cam.pose)
    return out


def _gen_rays(vr, pose):
    """ngp_gen_rays with img_idx = 0, pix_idx = arange(H*W) on the frame's float32 pose"""
    from ngp_pl_b200 import _lib
    n = vr.n
    c2w = torch.as_tensor(np.asarray(pose, np.float64)[:3, :4].astype(np.float32)).cuda().contiguous()
    img = torch.zeros(n, dtype=torch.int64, device="cuda")
    pix = torch.arange(n, dtype=torch.int64, device="cuda")
    o, d = torch.empty(n, 3, device="cuda"), torch.empty(n, 3, device="cuda")
    rc = _lib.lib().ngp_gen_rays(img.data_ptr(), pix.data_ptr(), c2w.data_ptr(), vr.directions.data_ptr(), None, n, n,
                                 o.data_ptr(), d.data_ptr(), None, torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "ngp_gen_rays")
    return o, d


def _composed(vr, rays_o, rays_d, mode):
    """render(test_time=True) with the viewer's settings on the given rays, the display image and its JPEG"""
    from ngp_pl_b200 import images
    from ngp_pl_b200.models.rendering import render
    res = render(vr.model, rays_o, rays_d, test_time=True, T_threshold=1e-2, max_samples=100, exp_step_factor=0.0)
    rgb_img, depth_img = images.view_images(res["rgb"] if mode == "rgb" else None,
                                            res["depth"] if mode == "depth" else None, vr.H, vr.W)
    img = rgb_img if mode == "rgb" else depth_img
    return res, img, images.encode_jpeg(img, vr.views[mode].quality)


def test_rays_are_ngp_gen_rays_bitwise_and_close_to_float64():
    W, H = 41, 29
    vr, K = _renderer(W, H)
    for pose in _poses(K, W, H, 3, seed=1):
        vr.frame(pose, "rgb")
        o, d = _gen_rays(vr, pose)
        torch.cuda.synchronize()
        assert torch.equal(vr.rays_o, o) and torch.equal(vr.rays_d, d)
        P = np.asarray(pose, np.float64)[:3, :4].astype(np.float32).astype(np.float64)
        dirs = vr.directions.cpu().numpy().astype(np.float64)
        want = dirs @ P[:, :3].T
        got = vr.rays_d.cpu().numpy().astype(np.float64)
        # two fp32 roundings of products and sums: |err| <= 4 eps (sum_c |dir_c R_kc|)
        bound = 4 * np.finfo(np.float32).eps * (np.abs(dirs) @ np.abs(P[:, :3]).T)
        assert np.all(np.abs(got - want) <= bound)
        assert np.array_equal(vr.rays_o.cpu().numpy(), np.broadcast_to(P[:, 3].astype(np.float32), (vr.n, 3)))


@pytest.mark.parametrize("mode", ["rgb", "depth"])
@pytest.mark.parametrize("W,H", SIZES)
def test_outputs_and_jpeg_equal_the_composed_path(W, H, mode):
    from ngp_pl_b200 import _lib
    vr, K = _renderer(W, H)
    L = _lib.lib()
    for pose in _poses(K, W, H, 2, seed=2):
        jpeg, info = vr.frame(pose, mode)
        o, d = vr.rays_o.clone(), vr.rays_d.clone()
        # ngp_render_infer_frame on the frame's rays with the same cfg
        from ngp_pl_b200.models.networks import _net_struct
        net, keep = _net_struct(vr.model)
        n = vr.n
        ws = torch.empty(L.ngp_render_infer_workspace(n, vr.cfg.max_round_samples), dtype=torch.uint8, device="cuda")
        op, dp, rgb = torch.empty(n, device="cuda"), torch.empty(n, device="cuda"), torch.empty(n, 3, device="cuda")
        total = torch.zeros(1, dtype=torch.int64, device="cuda")
        rc = L.ngp_render_infer_frame(C.byref(net), C.byref(vr.cfg), o.data_ptr(), d.data_ptr(),
                                      vr.model.density_bitfield.data_ptr(), op.data_ptr(), dp.data_ptr(), rgb.data_ptr(),
                                      total.data_ptr(), ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream)
        _lib.check(rc, "ngp_render_infer_frame")
        torch.cuda.synchronize()
        assert torch.equal(vr.opacity, op) and torch.equal(vr.depth, dp) and torch.equal(vr.rgb, rgb)
        assert info["total_samples"] == int(total[0]) > 0 and info["samples_per_ray"] == int(total[0]) / n
        # the display image and the JPEG
        res, img, want = _composed(vr, o, d, mode)
        assert torch.equal(res["rgb"], rgb) and torch.equal(res["depth"], dp) and int(res["total_samples"]) == int(total[0])
        assert jpeg == want
        assert jpeg == J.encode(img.cpu().numpy(), vr.views[mode].quality)


def test_no_rebuilds_while_the_camera_moves_and_the_mode_toggles():
    from ngp_pl_b200 import _lib
    W, H = 120, 90
    vr, K = _renderer(W, H)
    poses = _poses(K, W, H, 21, seed=3)
    vr.frame(poses[0], "rgb")
    vr.frame(poses[0], "depth")
    n0 = int(_lib.lib().ngp_launch_count())
    frames = []
    for i, pose in enumerate(poses[1:]):
        mode = ("rgb", "depth")[(i // 3) % 2]
        jpeg, info = vr.frame(pose, mode)
        frames.append((pose, mode, jpeg, info))
    assert int(_lib.lib().ngp_launch_count()) == n0
    assert len({f[2] for f in frames}) == len(frames)  # every pose gives its own picture
    for pose, mode, jpeg, info in frames:
        o, d = _gen_rays(vr, pose)
        res, _, want = _composed(vr, o, d, mode)
        assert jpeg == want and info["total_samples"] == int(res["total_samples"])


def test_two_frames_of_one_pose_are_byte_identical():
    W, H = 41, 29
    vr, K = _renderer(W, H, quality=75)
    pose = _poses(K, W, H, 1, seed=4)[0]
    for mode in ("rgb", "depth"):
        a, ia = vr.frame(pose, mode)
        b, ib = vr.frame(pose, mode)
        assert a == b and ia["total_samples"] == ib["total_samples"]
        assert a[:2] == b"\xff\xd8" and a[-2:] == b"\xff\xd9"


def test_frames_from_a_new_thread_on_the_models_device():
    """frame() renders on the model's device whatever the calling thread's current device is: a new thread (the
    server's render thread) starts on device 0. On a second GPU, when there is one, the frames equal device 0's"""
    import threading
    W, H = 41, 29
    want = {}
    for dev in range(min(torch.cuda.device_count(), 2)):
        with torch.cuda.device(dev):
            vr, K = _renderer(W, H)
        assert vr.device == torch.device("cuda", dev) and torch.cuda.current_device() == 0
        poses = _poses(K, W, H, 2, seed=6)
        got = {}

        def run():
            got["frames"] = [vr.frame(p, m)[0] for p in poses for m in ("rgb", "depth")]
        t = threading.Thread(target=run)
        t.start()
        t.join()
        main = [vr.frame(p, m)[0] for p in poses for m in ("rgb", "depth")]
        assert got["frames"] == main
        want.setdefault("frames", main)
        assert main == want["frames"], dev


def test_invalid_arguments_return_einval():
    from ngp_pl_b200 import _lib
    from ngp_pl_b200.models.networks import _net_struct
    L = _lib.lib()
    W, H = 41, 29
    vr, K = _renderer(W, H)
    vr.frame(_poses(K, W, H, 1, seed=5)[0], "rgb")
    net, keep = _net_struct(vr.model)
    st = torch.cuda.current_stream().cuda_stream
    pageable = (C.c_float * 12)()

    def call(**over):
        a = dict(net=C.byref(net), cfg=C.byref(vr.cfg), view=C.byref(vr.views["rgb"]), directions=vr.directions.data_ptr(),
                 pose=vr.pose.data_ptr(), bits=vr.model.density_bitfield.data_ptr(), o=vr.rays_o.data_ptr(),
                 d=vr.rays_d.data_ptr(), op=vr.opacity.data_ptr(), dp=vr.depth.data_ptr(), rgb=vr.rgb.data_ptr(),
                 jpeg=vr.jpeg.data_ptr(), cap=vr.jpeg.numel(), stats=vr.stats.data_ptr(), ws=vr.ws.data_ptr(),
                 ws_bytes=vr.ws.numel())
        a.update(over)
        return L.ngp_render_view_frame(a["net"], a["cfg"], a["view"], a["directions"], a["pose"], a["bits"], a["o"], a["d"],
                                       a["op"], a["dp"], a["rgb"], a["jpeg"], a["cap"], a["stats"], a["ws"], a["ws_bytes"], st)

    def view(**kw):
        v = _lib.NgpViewCfg(vr.views["rgb"].mode, vr.views["rgb"].quality, H, W)
        for k, x in kw.items():
            setattr(v, k, x)
        return v

    def cfg(**kw):
        c = _lib.NgpInferCfg.from_buffer_copy(vr.cfg)
        for k, x in kw.items():
            setattr(c, k, x)
        return c

    n0 = int(L.ngp_launch_count())
    assert call() == 0
    torch.cuda.synchronize()
    assert L.ngp_render_view_workspace(C.byref(vr.cfg), C.byref(view(H=H + 1))) == 0
    bad = [dict(view=C.byref(view(**kw))) for kw in (dict(H=H + 1), dict(W=W - 1), dict(mode=2), dict(mode=-1),
                                                      dict(quality=0), dict(quality=101))]
    bad += [dict(cfg=C.byref(cfg(**kw))) for kw in (dict(n_rays=0), dict(cascades=0), dict(grid_size=0),
                                                    dict(grid_size=2048), dict(max_samples=0),
                                                    dict(max_round_samples=vr.n - 1), dict(max_round_samples=1 << 31),
                                                    dict(sample_budget=0))]
    bad += [dict(cap=vr.jpeg.numel() - 1), dict(cap=L.ngp_jpeg_capacity(H, W) - 1), dict(ws_bytes=vr.ws.numel() - 1),
            dict(ws=vr.ws.data_ptr() + 16), dict(stats=vr.stats.data_ptr() + 4), dict(pose=C.addressof(pageable))]
    for name in ("net", "cfg", "view", "directions", "pose", "bits", "o", "d", "op", "dp", "rgb", "jpeg", "stats", "ws"):
        bad.append({name: None})
    for over in bad:
        assert call(**over) == -22, over
    assert int(L.ngp_launch_count()) == n0  # the good call replayed the cached graph, and no refused call captured any


def test_show_gui_serves_a_trained_checkpoint(tmp_path):
    """train the lego fixture with the command line, serve its _slim.ckpt in-process, fetch a frame, orbit, fetch the
    next: both are ViewRenderer.frame of the OrbitCamera poses"""
    from ngp_pl_b200 import show_gui, train
    from ngp_pl_b200.models.networks import NGP
    out = str(tmp_path)
    env = {k: v for k, v in os.environ.items() if k not in ("WORLD_SIZE", "RANK", "LOCAL_RANK")}
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    lego = os.path.join(FIX, "lego")
    r = subprocess.run([sys.executable, "-m", "ngp_pl_b200.train", "--root_dir", lego, "--dataset_name", "nerf",
                        "--downsample", "0.1", "--num_epochs", "1", "--epoch_steps", "30", "--batch_size", "1024",
                        "--exp_name", "view", "--out_dir", out, "--no_save_test"], cwd=out, env=env,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:]
    slim = os.path.join(out, "ckpts", "nerf", "view", "epoch=0_slim.ckpt")
    args = show_gui.parse_args(["--root_dir", lego, "--dataset_name", "nerf", "--downsample", "0.1", "--ckpt_path", slim,
                                "--port", "0"])
    srv = show_gui.open_viewer(args)
    try:
        assert srv.address[0] == "127.0.0.1"

        def get(path, body=None):
            c = http.client.HTTPConnection(*srv.address, timeout=60)
            try:
                c.request("POST" if body else "GET", path, body=body)
                resp = c.getresponse()
                return resp.status, dict(resp.getheaders()), resp.read()
            finally:
                c.close()

        code, hdr, first = get("/frame?after=0")
        assert code == 200 and hdr["X-Frame"] == "1" and float(hdr["X-Samples-Per-Ray"]) > 0
        assert get("/input", b'{"orbit": [40, -25]}')[0] == 204
        code, hdr, second = get("/frame?after=1")
        assert code == 200 and hdr["X-Frame"] == "2"
    finally:
        srv.close()
    # the same frames from a fresh model and renderer
    from ngp_pl_b200 import datasets
    meta = datasets.scene_meta("nerf", lego, "test", 0.1)
    assert tuple(meta.img_wh) == (srv.renderer.W, srv.renderer.H)
    assert torch.equal(meta.directions.cuda(), srv.renderer.directions)
    model = NGP(scale=args.scale).cuda()
    train.load_weights(model, slim)
    vr = show_gui.ViewRenderer(model, meta.K, meta.img_wh, 0.0, args.quality)
    cam = show_gui.OrbitCamera(meta.K, meta.img_wh, r=args.radius)
    assert vr.frame(cam.pose, "rgb")[0] == first
    cam.orbit(40.0, -25.0)
    assert vr.frame(cam.pose, "rgb")[0] == second != first
