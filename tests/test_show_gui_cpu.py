"""CPU tests of `python -m ngp_pl_b200.show_gui`: the orbit camera against the reference's own OrbitCamera
(tests/golden/viewer_orbit.npz, tests/golden/make_golden_viewer.py), the command line's flags against the reference's
opt.py and its refusals, and the HTTP server's protocol with a fake renderer (no CUDA anywhere)."""
import http.client
import json
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

from test_train_cli_cpu import _flags, _ref_module

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "viewer_orbit.npz")
K = np.float32([[1111.11, 0, 400], [0, 1111.11, 400], [0, 0, 1]])


def _apply(cam, calls):
    for kind, a0, a1, a2, has_dz in calls:
        if kind == 0:
            cam.orbit(a0, a1)
        elif kind == 1:
            cam.scale(a0)
        elif has_dz:
            cam.pan(a0, a1, a2)
        else:
            cam.pan(a0, a1)
    return cam.pose


def test_orbit_camera_equals_the_reference():
    from ngp_pl_b200.show_gui import OrbitCamera
    z = np.load(GOLDEN)
    n = len([k for k in z.files if k.startswith("pose_")])
    assert n >= 40
    for s in range(n):
        cam = OrbitCamera(K, (800, 800), float(z["radius_%02d" % s]))
        got = _apply(cam, z["calls_%02d" % s])
        want = z["pose_%02d" % s]
        assert got.dtype == np.float64 and got.shape == (4, 4)
        assert np.abs(got - want).max() <= 1e-12, (s, np.abs(got - want).max())


def test_from_rotvec_is_a_rotation_and_exact_at_zero():
    from ngp_pl_b200.show_gui import from_rotvec
    rng = np.random.RandomState(0)
    assert np.array_equal(from_rotvec(np.zeros(3)), np.eye(3))
    for scale in (1e-12, 1e-6, 1.0, 10.0):
        v = rng.normal(size=3) * scale
        R = from_rotvec(v)
        assert np.abs(R @ R.T - np.eye(3)).max() < 1e-14
        assert np.abs(R @ v - v).max() <= 1e-14 * max(1.0, np.abs(v).max())  # the axis is fixed


# ---- command line ---------------------------------------------------------------------------------------------------------
VIEWER_FLAGS = {"host", "port", "radius", "quality"}
TRAIN_ADDITIONS = {"seed", "out_dir", "epoch_steps", "lpips_vgg", "lpips_lin", "video_fps"}


def test_flags_match_the_reference_opt_py(monkeypatch):
    """the reference's viewer takes opt.get_opts(): every flag of opt.py, as `train` has them, plus the viewer's own"""
    import argparse
    opt = _ref_module("opt")
    captured = {}

    def grab(self, *a, **k):
        captured["parser"] = self
        return argparse.Namespace()

    monkeypatch.setattr(argparse.ArgumentParser, "parse_args", grab)
    opt.get_opts()
    ref = _flags(captured["parser"])
    monkeypatch.undo()
    from ngp_pl_b200 import show_gui, train
    ours = _flags(show_gui.get_parser())
    assert len(ref) >= 20
    for dest, spec in ref.items():
        assert dest in ours, "flag --%s of the reference is missing" % dest
        got = dict(ours[dest])
        if dest == "dataset_name":
            assert spec["default"] == "nsvf" and got["default"] == "nerf"
            got["default"] = spec["default"]
        assert got == spec, (dest, got, spec)
    assert set(ours) - set(ref) == TRAIN_ADDITIONS | VIEWER_FLAGS
    assert set(_flags(train.get_parser())) - set(ref) == TRAIN_ADDITIONS  # train's parser is untouched


def _run(argv, code=None):
    env = {k: v for k, v in os.environ.items() if k not in ("WORLD_SIZE", "RANK", "LOCAL_RANK")}
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    env["CUDA_VISIBLE_DEVICES"] = ""
    cmd = [sys.executable, "-c", code] if code else [sys.executable, "-m", "ngp_pl_b200.show_gui"] + argv
    return subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=120)


def _refused(tmp):
    ok = os.path.join(tmp, "model_slim.ckpt")
    unreadable = os.path.join(tmp, "dir.ckpt")  # a directory cannot be opened as a file
    return [
        (["--dataset_name", "nsvf", "--ckpt_path", ok], "--dataset_name"),
        (["--dataset_name", "nerfpp", "--ckpt_path", ok], "--dataset_name"),
        (["--dataset_name", "rtmv", "--ckpt_path", ok], "--dataset_name"),
        (["--use_exposure", "--ckpt_path", ok], "--use_exposure"),
        ([], "--ckpt_path"),
        (["--ckpt_path", os.path.join(tmp, "missing.ckpt")], "--ckpt_path"),
        (["--ckpt_path", unreadable], "--ckpt_path"),
        (["--ckpt_path", ok, "--quality", "0"], "--quality"),
        (["--ckpt_path", ok, "--port", "70000"], "--port"),
    ]


def test_refusals_exit_2_naming_the_flag(tmp_path):
    tmp = str(tmp_path)
    open(os.path.join(tmp, "model_slim.ckpt"), "wb").close()
    os.mkdir(os.path.join(tmp, "dir.ckpt"))
    for argv, flag in _refused(tmp):
        r = _run(["--root_dir", "does/not/exist"] + argv)
        assert r.returncode == 2, (argv, r.returncode, r.stderr)
        assert flag in r.stderr, (argv, r.stderr)


def test_refusals_happen_before_torch_or_cuda(tmp_path):
    code = ("import sys; from ngp_pl_b200 import show_gui\n"
            "try:\n    show_gui.main(['--root_dir', 'x', '--use_exposure', '--ckpt_path', %r])\n"
            "except SystemExit as e:\n    code = e.code\n"
            "print(code, 'torch' in sys.modules)\n" % __file__)
    r = _run(None, code)
    assert r.stdout.split() == ["2", "False"], (r.stdout, r.stderr)


def test_accepted_flags_parse_without_torch():
    code = ("import sys; from ngp_pl_b200 import show_gui\n"
            "a = show_gui.parse_args(['--root_dir', 'x', '--dataset_name', 'colmap', '--ckpt_path', %r, '--port', '0',"
            " '--radius', '3', '--quality', '75', '--downsample', '0.25'])\n"
            "print(a.host, a.port, a.radius, a.quality, a.downsample, 'torch' in sys.modules)\n" % __file__)
    r = _run(None, code)
    assert r.stdout.split() == ["127.0.0.1", "0", "3.0", "75", "0.25", "False"], (r.stdout, r.stderr)


# ---- server protocol with a fake renderer ---------------------------------------------------------------------------------
class FakeRenderer:
    """fixed bytes per frame; records each call's pose, mode and thread"""

    def __init__(self):
        self.calls = []
        self.lock = threading.Lock()

    def frame(self, pose, mode):
        with self.lock:
            self.calls.append((np.array(pose), mode, threading.current_thread().name))
            k = len(self.calls)
        return b"\xff\xd8fake-%s-%d\xff\xd9" % (mode.encode(), k), {"render_ms": 1.5, "samples_per_ray": 2.25,
                                                                     "total_samples": 9}


@pytest.fixture
def viewer():
    from ngp_pl_b200.show_gui import OrbitCamera, ViewServer
    before = set(threading.enumerate())
    fake = FakeRenderer()
    srv = ViewServer(fake, OrbitCamera(K, (800, 800), 2.5), "127.0.0.1", 0, poll_timeout=0.3)
    yield srv, fake
    srv.close()
    assert set(threading.enumerate()) <= before


def _request(srv, method, path, body=None, headers=None):
    c = http.client.HTTPConnection(*srv.address, timeout=10)
    try:
        c.request(method, path, body=body, headers=headers or {})
        r = c.getresponse()
        return r.status, dict(r.getheaders()), r.read()
    finally:
        c.close()


def _post(srv, obj):
    body = obj if isinstance(obj, bytes) else json.dumps(obj).encode()
    return _request(srv, "POST", "/input", body, {"Content-Type": "application/json"})


def test_server_listens_on_loopback_only(viewer):
    srv, _ = viewer
    assert srv.address[0] == "127.0.0.1" and srv.address[1] > 0


def test_page_and_first_frame(viewer):
    srv, fake = viewer
    code, hdr, body = _request(srv, "GET", "/")
    assert code == 200 and hdr["Content-Type"].startswith("text/html") and b"/frame?after=" in body
    code, hdr, body = _request(srv, "GET", "/frame?after=0")
    assert code == 200 and hdr["Content-Type"] == "image/jpeg"
    assert body == b"\xff\xd8fake-rgb-1\xff\xd9"
    assert hdr["X-Frame"] == "1" and hdr["X-Render-Ms"] == "1.50" and hdr["X-Samples-Per-Ray"] == "2.25"
    pose, mode, thread = fake.calls[0]
    assert mode == "rgb" and thread == "ngp-view-render" and np.array_equal(pose, srv.camera.pose)


def test_inputs_move_the_camera_as_orbit_camera_does(viewer):
    from ngp_pl_b200.show_gui import OrbitCamera
    srv, fake = viewer
    ref = OrbitCamera(K, (800, 800), 2.5)
    _request(srv, "GET", "/frame?after=0")
    steps = [({"orbit": [12, -7]}, lambda c: c.orbit(12.0, -7.0)),
             ({"pan": [300, 45.5]}, lambda c: c.pan(300.0, 45.5)),
             ({"scale": 1}, lambda c: c.scale(1.0)),
             ({"scale": -2.5}, lambda c: c.scale(-2.5)),
             ({"orbit": [-0.5, 1e4]}, lambda c: c.orbit(-0.5, 1e4))]
    seq = 1
    for body, move in steps:
        code, _, _ = _post(srv, body)
        assert code == 204, body
        move(ref)
        assert np.array_equal(srv.camera.pose, ref.pose), body
        code, hdr, data = _request(srv, "GET", "/frame?after=%d" % seq)
        assert code == 200
        seq = int(hdr["X-Frame"])
    # the newest frame renders the camera as it stands after the last input
    assert np.array_equal(fake.calls[-1][0], ref.pose)
    assert all(t == "ngp-view-render" for _, _, t in fake.calls)


def test_mode_toggles_the_rendered_output(viewer):
    srv, fake = viewer
    _request(srv, "GET", "/frame?after=0")
    assert _post(srv, {"mode": "depth"})[0] == 204
    code, hdr, body = _request(srv, "GET", "/frame?after=1")
    assert code == 200 and body.startswith(b"\xff\xd8fake-depth-")
    assert _post(srv, {"mode": "rgb"})[0] == 204
    code, hdr, body = _request(srv, "GET", "/frame?after=%s" % hdr["X-Frame"])
    assert code == 200 and body.startswith(b"\xff\xd8fake-rgb-")


BAD = [b"not json", b"[1, 2]", b"{}", b'{"orbit": [1]}', b'{"orbit": [1, 2, 3]}', b'{"orbit": "12"}',
       b'{"orbit": [1, NaN]}', b'{"pan": [Infinity, 0]}', b'{"scale": -Infinity}', b'{"scale": 1e400}',
       b'{"scale": 10001}', b'{"orbit": [0, -1e5]}', b'{"pan": [true, 1]}', b'{"scale": null}', b'{"mode": "normals"}',
       b'{"mode": ["rgb"]}', b'{"mode": {}}', b'{"mode": 1}',
       b'{"zoom": 1}', b'{"orbit": [1, 2], "scale": 1}', b'{"scale": 1' + b"0" * 400 + b"}", b"\xff\xfe"]


def test_malformed_input_is_refused_and_leaves_the_camera(viewer):
    srv, fake = viewer
    _request(srv, "GET", "/frame?after=0")
    pose0, n0 = srv.camera.pose.copy(), len(fake.calls)
    for body in BAD:
        code, _, _ = _post(srv, body)
        assert code == 400, body
    code, _, _ = _post(srv, b'{"scale": 1, "pad": "' + b"x" * 5000 + b'"}')
    assert code == 413
    for method, path in (("GET", "/input"), ("GET", "/etc/passwd"), ("GET", "/../show_gui.py"), ("POST", "/frame"),
                         ("GET", "/frame/../x")):
        code, _, _ = _request(srv, method, path, b"{}" if method == "POST" else None)
        assert code == 404, (method, path)
    assert _request(srv, "GET", "/frame?after=x")[0] == 400
    assert np.array_equal(srv.camera.pose, pose0) and srv.mode == "rgb"
    assert srv.wait_frame(1, 0.2) is None and len(fake.calls) == n0  # nothing asked for a new frame


def test_poll_at_the_latest_frame_times_out_with_204(viewer):
    srv, _ = viewer
    code, hdr, _ = _request(srv, "GET", "/frame?after=0")
    assert code == 200
    code, _, body = _request(srv, "GET", "/frame?after=%s" % hdr["X-Frame"])
    assert code == 204 and body == b""


def _raw(srv, data, half_close):
    """send raw bytes on one connection and return everything the server answers before it closes"""
    import socket
    with socket.create_connection(srv.address, timeout=20) as s:
        s.sendall(data)
        if half_close:
            s.shutdown(socket.SHUT_WR)
        out = b""
        while True:
            chunk = s.recv(4096)
            if not chunk:
                return out
            out += chunk


def test_a_body_shorter_than_its_length_is_refused_quietly(viewer, capfd):
    """a client that sends less than its Content-Length and stops gets a 400; one that stalls is disconnected when
    the request timeout passes; neither leaves a traceback, and the server goes on serving"""
    srv, _ = viewer
    head = b"POST /input HTTP/1.0\r\nContent-Length: 100\r\n\r\n"
    short = _raw(srv, head + b'{"scale": 1}', half_close=True)
    assert short.startswith(b"HTTP/1.0 400"), short
    assert _raw(srv, head + b'{"scale": 1}', half_close=False) == b""
    assert _request(srv, "GET", "/frame?after=0")[0] == 200
    assert srv.camera.radius == 2.5
    assert "Traceback" not in capfd.readouterr().err


def test_close_ends_a_pending_poll_and_every_thread():
    from ngp_pl_b200.show_gui import OrbitCamera, ViewServer
    before = set(threading.enumerate())
    srv = ViewServer(FakeRenderer(), OrbitCamera(K, (800, 800), 2.5), "127.0.0.1", 0, poll_timeout=30)
    assert _request(srv, "GET", "/frame?after=0")[0] == 200
    got = {}
    t = threading.Thread(target=lambda: got.setdefault("r", _request(srv, "GET", "/frame?after=1")))
    t.start()
    import time
    time.sleep(0.3)
    t0 = time.monotonic()
    srv.close()
    t.join(10)
    assert time.monotonic() - t0 < 5
    assert got["r"][0] == 204
    assert set(threading.enumerate()) <= before


def test_a_renderer_error_is_kept_and_polls_end():
    from ngp_pl_b200.show_gui import OrbitCamera, ViewServer

    class Broken:
        def frame(self, pose, mode):
            raise RuntimeError("no device")

    srv = ViewServer(Broken(), OrbitCamera(K, (800, 800), 2.5), "127.0.0.1", 0, poll_timeout=30)
    try:
        code, _, _ = _request(srv, "GET", "/frame?after=0")
        assert code == 204 and isinstance(srv.error, RuntimeError)
    finally:
        srv.close()


def test_view_renderer_refuses_a_model_off_the_gpu():
    import torch
    from ngp_pl_b200.show_gui import ViewRenderer
    m = torch.nn.Module()
    m.register_buffer("density_bitfield", torch.zeros(8, dtype=torch.uint8))
    with pytest.raises(RuntimeError):
        ViewRenderer(m, K, (8, 8), 0.0)


def test_view_cfg_layout_matches_the_header():
    """sizeof and field offsets of NgpViewCfg as the C compiler sees them == the ctypes mirror"""
    import ctypes
    import tempfile
    from ngp_pl_b200 import _lib
    fields = [f for f, _ in _lib.NgpViewCfg._fields_]
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        body = 'printf("%zu\\n", sizeof(NgpViewCfg));' + "".join(
            'printf("%%zu\\n", offsetof(NgpViewCfg, %s));' % f for f in fields)
        open(c, "w").write('#include <stddef.h>\n#include <stdio.h>\n#include "ngp_b200.h"\nint main(void){%s return 0;}\n'
                           % body)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).decode().split()]
    assert got == [ctypes.sizeof(_lib.NgpViewCfg)] + [getattr(_lib.NgpViewCfg, f).offset for f in fields]
