"""Inspect a trained model interactively, in a browser: the reference's `show_gui.py` orbit viewer, served over HTTP.

    python -m ngp_pl_b200.show_gui --root_dir data/lego --dataset_name nerf \\
        --ckpt_path ckpts/nerf/lego/epoch=29_slim.ckpt
    # on the workstation:  ssh -L 8000:localhost:8000 <gpu host>   then open http://localhost:8000

The reference opens a dearpygui window; a GPU server has no display, so the frames go to a browser instead. Left-drag
orbits, middle-drag or shift-drag pans, the wheel zooms, the button or the `d` key toggles the depth view, and the page
shows the render time and the samples per ray as the reference's control window does.

    OrbitCamera(K, img_wh, r)      the reference's camera (show_gui.py:19-51), in float64 numpy, no scipy at run time
    ViewRenderer(model, K, img_wh, exp_step_factor, quality=90)
                                   frame(pose, mode) -> (JPEG bytes, stats): one ngp_render_view_frame call, a CUDA graph
                                   from the pose to the JPEG (csrc/infer.cu), with the reference GUI's render settings
    ViewServer(renderer, camera, host, port)
                                   the HTTP server: one render thread owns every CUDA call, handler threads never touch CUDA
    serve(model, K, img_wh, exp_step_factor, host, port, radius, quality)
                                   the three of them for a model; returns the running ViewServer

HTTP interface (loopback by default; nothing serves files):
    GET  /                 the viewer page
    GET  /frame?after=k    the first frame with sequence number > k (long poll): image/jpeg with X-Frame, X-Render-Ms
                           and X-Samples-Per-Ray headers, or 204 when none arrives in time
    POST /input            one of {"orbit": [dx, dy]}, {"pan": [dx, dy]}, {"scale": d}, {"mode": "rgb" | "depth"};
                           413 over 4 KiB, 400 for anything else (the camera is then left as it was)
"""
import ctypes as C
import http.server
import json
import math
import sys
import threading
import time
import urllib.parse

import numpy as np

VIEWER_DATASETS = ("nerf", "colmap")
MODES = {"rgb": 0, "depth": 1}
MAX_BODY = 4096
MAX_MAGNITUDE = 1e4
# the reference GUI's render() settings (show_gui.py:82-88)
T_THRESHOLD = 1e-2
SAMPLE_BUDGET = 100


# ---- camera ---------------------------------------------------------------------------------------------------------------
def from_rotvec(v):
    """rotation matrix of the rotation vector v (axis * angle in radians), Rodrigues' formula"""
    v = np.asarray(v, np.float64)
    theta = math.sqrt(float(v @ v))
    Kx = np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])
    if theta < 1e-8:  # series of sin(t)/t and (1 - cos(t))/t^2; exact to double precision here
        a, b = 1.0 - theta * theta / 6.0, 0.5 - theta * theta / 24.0
    else:
        a, b = math.sin(theta) / theta, (1.0 - math.cos(theta)) / (theta * theta)
    return np.eye(3) + a * Kx + b * (Kx @ Kx)


class OrbitCamera:
    """The reference's orbit camera: pose is the 4x4 camera-to-world matrix of a camera at distance `radius` from
    `center`, looking at it, turned by `rot`."""

    def __init__(self, K, img_wh, r):
        self.K = K
        self.W, self.H = img_wh
        self.radius = r
        self.center = np.zeros(3)
        self.rot = np.eye(3)

    @property
    def pose(self):
        res = np.eye(4)
        res[2, 3] -= self.radius  # move the camera to the radius
        rot = np.eye(4)
        rot[:3, :3] = self.rot
        res = rot @ res           # rotate
        res[:3, 3] -= self.center  # translate
        return res

    def orbit(self, dx, dy):
        rotvec_x = self.rot[:, 1] * np.radians(0.05 * dx)
        rotvec_y = self.rot[:, 0] * np.radians(-0.05 * dy)
        self.rot = from_rotvec(rotvec_y) @ from_rotvec(rotvec_x) @ self.rot

    def scale(self, delta):
        self.radius *= 1.1 ** (-delta)

    def pan(self, dx, dy, dz=0):
        self.center += 1e-4 * self.rot @ np.array([dx, dy, dz])


# ---- rendering ------------------------------------------------------------------------------------------------------------
class ViewRenderer:
    """Frames of a model at img_wh = (W, H) with intrinsics K, as the reference GUI renders them: render(test_time=True,
    T_threshold=1e-2, max_samples=100) with the marcher's 1024-step bound and the background rule of render() (white
    when exp_step_factor == 0, else black), then the RGB image or depth2img of the depth. Every buffer is allocated once,
    so every frame replays the same cached graph. Not thread-safe: one thread makes every call."""

    def __init__(self, model, K, img_wh, exp_step_factor, quality=90):
        import torch
        from . import _lib, datasets
        from .models.rendering import infer_cfg
        bits = getattr(model, "density_bitfield", None)
        if bits is None or not bits.is_cuda:
            raise RuntimeError("ngp_pl_b200.show_gui: the model must live on a CUDA device (there is no CPU path)")
        if not 1 <= int(quality) <= 100:
            raise ValueError("ngp_pl_b200.show_gui: quality must be in 1..100, got %r" % (quality,))
        self.model, self.device = model, bits.device
        self.W, self.H = int(img_wh[0]), int(img_wh[1])
        n = self.W * self.H
        self.n = n
        L = self._L = _lib.lib()
        self.cfg = cfg = infer_cfg(model, n, exp_step_factor, 1.0 if exp_step_factor == 0 else 0.0, T_THRESHOLD,
                                   SAMPLE_BUDGET)
        self.views = {m: _lib.NgpViewCfg(k, int(quality), self.H, self.W) for m, k in MODES.items()}
        ws = L.ngp_render_view_workspace(C.byref(cfg), C.byref(self.views["rgb"]))
        cap = L.ngp_jpeg_capacity(self.H, self.W)
        if ws == 0 or cap == 0:
            raise RuntimeError("ngp_pl_b200.show_gui: no view of %d x %d" % (self.W, self.H))
        dev = self.device
        with torch.cuda.device(dev):
            self.directions = datasets.ray_directions(self.W, self.H, K).to(dev)
            self.pose = torch.zeros(12, dtype=torch.float32).pin_memory()
            self.jpeg = torch.empty(cap, dtype=torch.uint8).pin_memory()
            self.stats = torch.zeros(2, dtype=torch.int64).pin_memory()
            self.rays_o, self.rays_d = torch.empty(n, 3, device=dev), torch.empty(n, 3, device=dev)
            self.opacity, self.depth = torch.empty(n, device=dev), torch.empty(n, device=dev)
            self.rgb = torch.empty(n, 3, device=dev)
            self.ws = torch.empty(ws, dtype=torch.uint8, device=dev)
            self.event = torch.cuda.Event()

    def frame(self, pose, mode="rgb"):
        """the JPEG of the view from pose (4x4 or 3x4 camera-to-world; its top 3x4 rows, in float32) in mode "rgb" or
        "depth", and {"render_ms": wall time of the call, "samples_per_ray", "total_samples"}"""
        import torch
        from . import _lib
        from .models.networks import _net_struct
        if mode not in MODES:
            raise ValueError("ngp_pl_b200.show_gui: mode must be 'rgb' or 'depth', got %r" % (mode,))
        t0 = time.perf_counter()
        self.pose.numpy()[:] = np.asarray(pose, np.float64)[:3, :4].reshape(-1)
        # the library builds and launches the graph on the calling thread's current device, which is device 0 in a new
        # thread (the server's render thread): make it the model's
        with torch.cuda.device(self.device):
            net, _keep = _net_struct(self.model)  # _keep: the fp16 weights the call reads
            st = torch.cuda.current_stream(self.device)
            rc = self._L.ngp_render_view_frame(
                C.byref(net), C.byref(self.cfg), C.byref(self.views[mode]), self.directions.data_ptr(),
                self.pose.data_ptr(), self.model.density_bitfield.data_ptr(), self.rays_o.data_ptr(),
                self.rays_d.data_ptr(), self.opacity.data_ptr(), self.depth.data_ptr(), self.rgb.data_ptr(),
                self.jpeg.data_ptr(), self.jpeg.numel(), self.stats.data_ptr(), self.ws.data_ptr(), self.ws.numel(),
                st.cuda_stream)
            _lib.check(rc, "ngp_render_view_frame")
            self.event.record(st)
        self.event.synchronize()
        ms = 1e3 * (time.perf_counter() - t0)
        n_bytes, total = int(self.stats[0]), int(self.stats[1])
        return self.jpeg[:n_bytes].numpy().tobytes(), {"render_ms": ms, "samples_per_ray": total / self.n,
                                                       "total_samples": total}


# ---- server ---------------------------------------------------------------------------------------------------------------
class BadInput(ValueError):
    pass


def _number(v):
    if isinstance(v, bool) or not isinstance(v, (int, float)):
        raise BadInput("expected a number, got %r" % (v,))
    try:
        v = float(v)
    except OverflowError:
        raise BadInput("number out of range")
    if not math.isfinite(v) or abs(v) > MAX_MAGNITUDE:
        raise BadInput("expected a finite number of magnitude at most %g, got %r" % (MAX_MAGNITUDE, v))
    return v


def _pair(v):
    if not isinstance(v, list) or len(v) != 2:
        raise BadInput("expected [dx, dy], got %r" % (v,))
    return _number(v[0]), _number(v[1])


def parse_input(body):
    """(kind, value) of one POST /input body (bytes); BadInput for anything else"""
    try:
        msg = json.loads(body.decode("utf-8"), parse_constant=lambda c: _number(float(c)))
    except BadInput:
        raise
    except (UnicodeDecodeError, ValueError) as e:
        raise BadInput("not JSON: %s" % e)
    if not isinstance(msg, dict) or len(msg) != 1:
        raise BadInput("expected one of {orbit, pan, scale, mode}")
    (kind, v), = msg.items()
    if kind in ("orbit", "pan"):
        return kind, _pair(v)
    if kind == "scale":
        return kind, _number(v)
    if kind == "mode":
        if not isinstance(v, str) or v not in MODES:
            raise BadInput("mode must be 'rgb' or 'depth', got %r" % (v,))
        return kind, v
    raise BadInput("unknown input %r" % (kind,))


class ViewServer:
    """Serves the frames of `renderer` (anything with frame(pose, mode) -> (jpeg bytes, stats dict)) for `camera` (an
    OrbitCamera) on host:port (port 0: any free port; see `address`). The render thread renders whenever the camera or
    the mode changed since its last frame; handler threads only read frames and move the camera under the lock.
    poll_timeout: seconds a GET /frame waits before answering 204. close() stops the server and joins every thread; an
    error of the renderer stops the render thread and is kept in `error`."""

    def __init__(self, renderer, camera, host="127.0.0.1", port=8000, poll_timeout=10.0):
        self.renderer, self.camera, self.poll_timeout = renderer, camera, float(poll_timeout)
        self.cond = threading.Condition()
        self.mode = "rgb"
        self.dirty = True
        self.stopping = False
        self.error = None
        self.latest = (0, None, None)  # (sequence number, jpeg, stats) of the newest frame
        self.httpd = http.server.ThreadingHTTPServer((host, int(port)), _handler(self))
        self.httpd.block_on_close = True  # server_close() joins the handler threads
        self.address = self.httpd.server_address[:2]
        self._render_thread = threading.Thread(target=self._render_loop, name="ngp-view-render")
        self._serve_thread = threading.Thread(target=self.httpd.serve_forever, kwargs={"poll_interval": 0.05},
                                              name="ngp-view-http")
        self._render_thread.start()
        self._serve_thread.start()

    @property
    def url(self):
        return "http://%s:%d/" % self.address

    def _render_loop(self):
        while True:
            with self.cond:
                while not self.dirty and not self.stopping:
                    self.cond.wait()
                if self.stopping:
                    return
                pose, mode = self.camera.pose.copy(), self.mode
                self.dirty = False
            try:
                jpeg, stats = self.renderer.frame(pose, mode)
            except BaseException as e:  # kept for the caller; the viewer stops rendering
                with self.cond:
                    self.error = e
                    self.cond.notify_all()
                return
            with self.cond:
                self.latest = (self.latest[0] + 1, jpeg, stats)
                self.cond.notify_all()

    def apply(self, kind, value):
        """apply one parsed input to the camera or the mode and wake the render thread"""
        with self.cond:
            if kind == "orbit":
                self.camera.orbit(*value)
            elif kind == "pan":
                self.camera.pan(*value)
            elif kind == "scale":
                self.camera.scale(value)
            else:
                self.mode = value
            self.dirty = True
            self.cond.notify_all()

    def wait_frame(self, after, timeout):
        """the newest (seq, jpeg, stats) with seq > after, or None after `timeout` seconds, an error or close()"""
        deadline = time.monotonic() + timeout
        with self.cond:
            while self.latest[0] <= after and not self.stopping and self.error is None:
                left = deadline - time.monotonic()
                if left <= 0:
                    return None
                self.cond.wait(left)
            return self.latest if self.latest[0] > after else None

    def close(self):
        with self.cond:
            self.stopping = True
            self.cond.notify_all()
        self.httpd.shutdown()
        self._serve_thread.join()
        self.httpd.server_close()
        self._render_thread.join()


def _handler(server):
    class Handler(http.server.BaseHTTPRequestHandler):
        timeout = 5  # seconds a connection may take to send its request (bounds how long close() can wait)

        def log_message(self, fmt, *args):
            pass

        def _send(self, code, body=b"", ctype="text/plain; charset=utf-8", headers=()):
            self.send_response(code)
            if code != 204:
                self.send_header("Content-Type", ctype)
                self.send_header("Content-Length", str(len(body)))
            self.send_header("Cache-Control", "no-store")
            for k, v in headers:
                self.send_header(k, v)
            self.end_headers()
            if code != 204:
                self.wfile.write(body)

        def do_GET(self):
            url = urllib.parse.urlsplit(self.path)
            if url.path == "/":
                return self._send(200, PAGE.encode("utf-8"), "text/html; charset=utf-8")
            if url.path != "/frame":
                return self._send(404, b"not found\n")
            q = urllib.parse.parse_qs(url.query)
            try:
                after = int(q.get("after", ["0"])[0])
            except ValueError:
                return self._send(400, b"after must be an integer\n")
            got = server.wait_frame(after, server.poll_timeout)
            if got is None:
                return self._send(204)
            seq, jpeg, stats = got
            self._send(200, jpeg, "image/jpeg", (("X-Frame", str(seq)), ("X-Render-Ms", "%.2f" % stats["render_ms"]),
                                                  ("X-Samples-Per-Ray", "%.2f" % stats["samples_per_ray"])))

        def do_POST(self):
            if urllib.parse.urlsplit(self.path).path != "/input":
                self.close_connection = True
                return self._send(404, b"not found\n")
            try:
                n = int(self.headers.get("Content-Length", ""))
            except ValueError:
                self.close_connection = True
                return self._send(400, b"Content-Length required\n")
            if n < 0:
                self.close_connection = True
                return self._send(400, b"bad Content-Length\n")
            # a modest body is read even when it is refused, so that the client sees the answer, not a reset
            try:
                body = self.rfile.read(n) if n <= 16 * MAX_BODY else None
            except OSError:  # the client sent less than its Content-Length within the timeout, or went away
                self.close_connection = True
                return
            if n > MAX_BODY:
                self.close_connection = True
                return self._send(413, b"input over 4 KiB\n")
            if len(body) != n:  # the client closed its side early
                self.close_connection = True
                return self._send(400, b"body shorter than its Content-Length\n")
            try:
                kind, value = parse_input(body)
            except BadInput as e:
                return self._send(400, (str(e) + "\n").encode("utf-8"))
            server.apply(kind, value)
            self._send(204)

    return Handler


def serve(model, K, img_wh, exp_step_factor, host="127.0.0.1", port=8000, radius=2.5, quality=90):
    """a running ViewServer of model's frames (see the module docstring); the caller close()s it"""
    renderer = ViewRenderer(model, K, img_wh, exp_step_factor, quality)
    return ViewServer(renderer, OrbitCamera(K, img_wh, r=radius), host, port)


# ---- command line ---------------------------------------------------------------------------------------------------------
def get_parser():
    """every flag of `python -m ngp_pl_b200.train` (the reference's viewer takes opt.get_opts()) and the viewer's own"""
    from . import train
    p = train.get_parser()
    p.prog = "python -m ngp_pl_b200.show_gui"
    p.description = "Inspect a trained Instant-NGP model in a browser (the reference's show_gui.py)."
    p.add_argument("--host", type=str, default="127.0.0.1", help="address to listen on (loopback: reach it over ssh -L)")
    p.add_argument("--port", type=int, default=8000, help="port to listen on (0: any free port)")
    p.add_argument("--radius", type=float, default=2.5, help="initial distance of the orbit camera")
    p.add_argument("--quality", type=int, default=90, help="JPEG quality of the frames, 1..100")
    return p


def check_args(args, parser):
    """the refusals, before torch or CUDA: parser.error() (exit status 2) names the flag"""
    if args.dataset_name not in VIEWER_DATASETS:
        parser.error("--dataset_name %s: only %s scenes are viewed here" % (args.dataset_name, " and ".join(VIEWER_DATASETS)))
    if args.use_exposure:
        parser.error("--use_exposure: HDR exposure is not supported")
    if not args.ckpt_path:
        parser.error("--ckpt_path: the viewer needs a trained model's checkpoint")
    try:
        with open(args.ckpt_path, "rb"):
            pass
    except OSError as e:
        parser.error("--ckpt_path %s: cannot be read (%s)" % (args.ckpt_path, e.strerror or e))
    if not 0 <= args.port <= 65535:
        parser.error("--port must be in 0..65535")
    if not 1 <= args.quality <= 100:
        parser.error("--quality must be in 1..100")
    if not (args.radius > 0 and math.isfinite(args.radius)):
        parser.error("--radius must be positive")
    return args


def parse_args(argv=None):
    parser = get_parser()
    return check_args(parser.parse_args(argv), parser)


def open_viewer(args):
    """load the model of parsed args and return its running ViewServer"""
    import torch
    from . import datasets, train
    from .models.networks import NGP
    if not torch.cuda.is_available():
        raise SystemExit("ngp_pl_b200.show_gui: no CUDA device (there is no CPU path)")
    dev = torch.device("cuda", torch.cuda.current_device())
    meta = datasets.scene_meta(args.dataset_name, args.root_dir, "test", args.downsample)
    model = NGP(scale=args.scale).to(dev)
    train.load_weights(model, args.ckpt_path)
    exp_step_factor = 1 / 256 if args.dataset_name == "colmap" else 0.0  # show_gui.py:78-80
    return serve(model, meta.K, meta.img_wh, exp_step_factor, args.host, args.port, args.radius, args.quality)


def main(argv=None):
    args = parse_args(argv)
    server = open_viewer(args)
    print("ngp_pl_b200.show_gui: serving %s (Ctrl-C stops)" % server.url, flush=True)
    try:
        while server.error is None:
            time.sleep(0.2)
    except KeyboardInterrupt:
        pass
    finally:
        server.close()
    if server.error is not None:
        print("ngp_pl_b200.show_gui: rendering failed: %r" % (server.error,), file=sys.stderr)
        return 1
    return 0


PAGE = """<!doctype html>
<html><head><meta charset="utf-8"><title>ngp_pl</title>
<style>
body { margin: 0; background: #222; color: #ddd; font: 14px sans-serif; }
#view { display: block; cursor: grab; user-select: none; }
#panel { position: fixed; top: 8px; left: 8px; background: rgba(0,0,0,.6); padding: 8px; border-radius: 4px; }
</style></head>
<body>
<img id="view" draggable="false" alt="">
<div id="panel">
  <button id="depth">show depth</button>
  <div id="time">no data</div><div id="spr">no data</div>
</div>
<script>
"use strict";
const view = document.getElementById("view");
let mode = "rgb", last = 0;
// inputs of one kind are summed while a POST is in flight, so a fast drag never queues requests
const pending = {orbit: [0, 0], pan: [0, 0], scale: 0};
let busy = false;
function flush() {
  if (busy) return;
  let body = null;
  for (const k of ["orbit", "pan"]) {
    const v = pending[k];
    if (v[0] || v[1]) { body = {[k]: v.slice()}; pending[k] = [0, 0]; break; }
  }
  if (!body && pending.scale) { body = {scale: pending.scale}; pending.scale = 0; }
  if (!body) return;
  busy = true;
  post(body).finally(() => { busy = false; flush(); });
}
function post(body) {
  return fetch("/input", {method: "POST", headers: {"Content-Type": "application/json"}, body: JSON.stringify(body)})
    .catch(() => {});
}
function toggle() {
  mode = mode === "rgb" ? "depth" : "rgb";
  document.getElementById("depth").textContent = mode === "rgb" ? "show depth" : "show rgb";
  post({mode: mode});
}
document.getElementById("depth").onclick = toggle;
document.addEventListener("keydown", e => { if (e.key === "d") toggle(); });
view.addEventListener("contextmenu", e => e.preventDefault());
view.addEventListener("mousedown", e => e.preventDefault());
view.addEventListener("pointerdown", e => view.setPointerCapture(e.pointerId));
view.addEventListener("pointermove", e => {
  if (!e.buttons) return;
  const pan = (e.buttons & 4) || ((e.buttons & 1) && e.shiftKey);
  const v = pending[pan ? "pan" : "orbit"];
  if (!pan && !(e.buttons & 1)) return;
  v[0] += e.movementX; v[1] += e.movementY;
  flush();
});
view.addEventListener("wheel", e => {
  e.preventDefault();
  if (e.deltaY) { pending.scale += e.deltaY < 0 ? 1 : -1; flush(); }
}, {passive: false});
async function poll() {
  for (;;) {
    try {
      const r = await fetch("/frame?after=" + last, {cache: "no-store"});
      if (r.status === 200) {
        last = parseInt(r.headers.get("X-Frame"));
        const url = URL.createObjectURL(await r.blob());
        const old = view.src;
        view.src = url;
        if (old) URL.revokeObjectURL(old);
        document.getElementById("time").textContent = "Render time: " + r.headers.get("X-Render-Ms") + " ms";
        document.getElementById("spr").textContent = "Samples/ray: " + r.headers.get("X-Samples-Per-Ray");
      } else if (r.status !== 204) {
        await new Promise(ok => setTimeout(ok, 1000));
      }
    } catch (err) {
      await new Promise(ok => setTimeout(ok, 1000));
    }
  }
}
poll();
</script>
</body></html>
"""


if __name__ == "__main__":
    sys.exit(main())
