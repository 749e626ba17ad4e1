"""Test-view images of the validation pass on the device (reference train.py:215-221): the quantised RGB image and the
turbo depth image of a render, and PNG files of both.

    rgb_image(rgb, H, W)     (rgb_pred * 255).astype(np.uint8): an (H, W, 3) uint8 device tensor
    depth_image(depth, H, W) depth2img(depth) (train.py:45-50): per-view min/max, * 255, uint8, cv2's turbo colour map;
                             an (H, W, 3) uint8 device tensor whose channels are cv2's B, G, R -- the array the reference
                             writes to its `_d.png` files, blue in the red position included
    encode_png(img, mode="fixed")
                             the PNG file of an (H, W, 3) uint8 device image, as bytes; mode "dynamic" writes a smaller
                             file of the same image (dynamic Huffman blocks over a wider match search)
    write_png(path, img, mode="fixed")
                             the same, written to `path`
    encode_jpeg(img, quality=90), write_jpeg(path, img, quality=90)
                             the same for a baseline JPEG (4:4:4, libjpeg's bytes for that quality)
    AviWriter(path, W, H, fps)
                             a Motion-JPEG AVI file of such JPEGs (host only)
    render_video(model, poses, directions, img_wh, save_dir)
                             `rgb.avi` and `depth.avi` of a camera path

The arithmetic is ngp_view_images and ngp_png_encode (csrc/images.cu) and ngp_jpeg_encode (csrc/jpeg.cu); the byte
streams of the PNG and the JPEG are specified in include/ngp_b200.h. Tensors must live on a CUDA device, otherwise
RuntimeError; there is no CPU path. metrics.evaluate(save_dir=...) writes every view of the validation pass through
`ViewWriter`, and with video_fps= the two videos as well. The reference assembles `rgb.mp4` / `depth.mp4` (H.264) from
its PNGs; the videos here hold the same frames as Motion-JPEG in an AVI 1.0 container, which ffmpeg, VLC, mpv and OpenCV
play.
"""
import os
import queue
import struct
import threading
from fractions import Fraction

import torch

from . import _lib


def _stream(t):
    return torch.cuda.current_stream(t.device).cuda_stream


def _check_input(t, dtype, numel, what):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError("ngp_pl_b200.images: %s must be a CUDA tensor" % what)
    if t.dtype != dtype:
        raise RuntimeError("ngp_pl_b200.images: %s must be %s, got %s" % (what, dtype, t.dtype))
    if t.numel() != numel:
        raise RuntimeError("ngp_pl_b200.images: %s has %d values, expected %d" % (what, t.numel(), numel))
    return t.contiguous()


def _check_image(img):
    if not isinstance(img, torch.Tensor) or not img.is_cuda:
        raise RuntimeError("ngp_pl_b200.images: the image must be a CUDA tensor")
    if img.dtype != torch.uint8 or img.dim() != 3 or img.shape[2] != 3 or img.shape[0] < 1 or img.shape[1] < 1:
        raise RuntimeError("ngp_pl_b200.images: expected an (H, W, 3) uint8 image, got %s %s" % (img.dtype, tuple(img.shape)))
    return img.contiguous()


def view_images(rgb, depth, H, W, rgb_img=None, depth_img=None, ws=None):
    """One ngp_view_images call on the current stream, no synchronisation. rgb: fp32 (H*W, 3) or None; depth: fp32
    (H*W,) or None. Returns (rgb_img, depth_img), (H, W, 3) uint8 device tensors (None where the input is None); the
    outputs and ws (NGP_VIEW_IMAGES_WORKSPACE bytes) may be passed in to be reused."""
    H, W = int(H), int(W)
    if H < 1 or W < 1:
        raise RuntimeError("ngp_pl_b200.images: H and W must be at least 1, got %d x %d" % (H, W))
    if rgb is None and depth is None:
        raise RuntimeError("ngp_pl_b200.images: nothing to do")
    ref = rgb if rgb is not None else depth
    if rgb is not None:
        rgb = _check_input(rgb, torch.float32, 3 * H * W, "rgb")
        rgb_img = torch.empty(H, W, 3, dtype=torch.uint8, device=rgb.device) if rgb_img is None else rgb_img
    if depth is not None:
        depth = _check_input(depth, torch.float32, H * W, "depth")
        depth_img = torch.empty(H, W, 3, dtype=torch.uint8, device=depth.device) if depth_img is None else depth_img
        if ws is None:
            ws = torch.empty(_lib.NGP_VIEW_IMAGES_WORKSPACE, dtype=torch.uint8, device=depth.device)
    ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    rc = _lib.lib().ngp_view_images(ptr(rgb), ptr(depth), H, W, ptr(rgb_img) if rgb is not None else None,
                                    ptr(depth_img) if depth is not None else None, ptr(ws),
                                    0 if ws is None else ws.numel(), _stream(ref))
    _lib.check(rc, "ngp_view_images")
    return (rgb_img if rgb is not None else None), (depth_img if depth is not None else None)


@torch.no_grad()
def rgb_image(rgb, H, W):
    """(rgb * 255).astype(uint8) of an fp32 (H*W, 3) (or (H, W, 3)) render: (H, W, 3) uint8 on the device"""
    return view_images(rgb, None, H, W)[0]


@torch.no_grad()
def depth_image(depth, H, W):
    """depth2img of an fp32 (H*W,) (or (H, W)) depth map: (H, W, 3) uint8 on the device, cv2's B, G, R order"""
    return view_images(None, depth, H, W)[1]


def png_capacity(H, W):
    n = _lib.lib().ngp_png_capacity(int(H), int(W))
    if n == 0:
        raise RuntimeError("ngp_pl_b200.images: no PNG of %d x %d (an IDAT over 2^31 - 1 bytes, or an empty image)" % (H, W))
    return n


PNG_MODES = {"fixed": _lib.NGP_PNG_FIXED, "dynamic": _lib.NGP_PNG_DYNAMIC}


def _png_mode(mode):
    if mode not in PNG_MODES:
        raise ValueError("ngp_pl_b200.images: the PNG mode must be one of %s, got %r" % (sorted(PNG_MODES), mode))
    return PNG_MODES[mode]


def png_workspace(H, W, device, mode="fixed"):
    m = _png_mode(mode)
    png_capacity(H, W)
    return torch.empty(_lib.lib().ngp_png_workspace_mode(int(H), int(W), m), dtype=torch.uint8, device=device)


def encode_png_into(img, out, out_len, ws, mode="fixed"):
    """One ngp_png_encode_mode call on the current stream, no synchronisation: the file of img ((H, W, 3) uint8,
    device) into out (uint8, device or pinned host memory, at least png_capacity(H, W) bytes) and its length into
    out_len[0] (int64, device or pinned host memory). ws: png_workspace(H, W, device, mode). mode "fixed" is
    ngp_png_encode's stream, "dynamic" the smaller one of include/ngp_b200.h."""
    m = _png_mode(mode)
    img = _check_image(img)
    _check_buffers(out, out_len, ws)
    H, W = img.shape[0], img.shape[1]
    rc = _lib.lib().ngp_png_encode_mode(img.data_ptr(), H, W, m, out.data_ptr(), out.numel(), out_len.data_ptr(),
                                        ws.data_ptr(), ws.numel(), _stream(img))
    _lib.check(rc, "ngp_png_encode_mode")


@torch.no_grad()
def encode_png(img, mode="fixed"):
    """the PNG file of an (H, W, 3) uint8 device image, as bytes (written into pinned host memory by the device, so only
    the file's bytes cross PCIe; synchronises the current stream). mode: "fixed" or "dynamic" (smaller)"""
    _png_mode(mode)
    img = _check_image(img)
    H, W = img.shape[0], img.shape[1]
    out = torch.empty(png_capacity(H, W), dtype=torch.uint8, pin_memory=True)
    n = torch.zeros(1, dtype=torch.int64, pin_memory=True)
    encode_png_into(img, out, n, png_workspace(H, W, img.device, mode), mode)
    torch.cuda.current_stream(img.device).synchronize()
    return out[:int(n[0])].numpy().tobytes()


def write_png(path, img, mode="fixed"):
    """write the PNG file of an (H, W, 3) uint8 device image to path"""
    data = encode_png(img, mode)
    with open(path, "wb") as f:
        f.write(data)


def _check_buffers(out, out_len, ws):
    for t, dt in ((out, torch.uint8), (out_len, torch.int64), (ws, torch.uint8)):
        if not isinstance(t, torch.Tensor) or t.dtype != dt or not t.is_contiguous():
            raise RuntimeError("ngp_pl_b200.images: out, out_len and ws must be contiguous uint8 / int64 / uint8 tensors")
        if not (t.is_cuda or t.is_pinned()):
            raise RuntimeError("ngp_pl_b200.images: out and out_len must be CUDA or pinned host tensors")
    if not ws.is_cuda:
        raise RuntimeError("ngp_pl_b200.images: the workspace must be a CUDA tensor")


def jpeg_capacity(H, W):
    n = _lib.lib().ngp_jpeg_capacity(int(H), int(W))
    if n == 0:
        raise RuntimeError("ngp_pl_b200.images: no JPEG of %d x %d (a side outside 1..65535, or over 2^31 - 1 coded bits)"
                           % (H, W))
    return n


def jpeg_workspace(H, W, device):
    jpeg_capacity(H, W)
    return torch.empty(_lib.lib().ngp_jpeg_workspace(int(H), int(W)), dtype=torch.uint8, device=device)


def encode_jpeg_into(img, out, out_len, ws, quality=90):
    """One ngp_jpeg_encode call on the current stream, no synchronisation: the file of img ((H, W, 3) uint8, device)
    into out (uint8, device or pinned host memory, at least jpeg_capacity(H, W) bytes) and its length into out_len[0]
    (int64, device or pinned host memory). ws: jpeg_workspace(H, W, device); quality 1..100."""
    img = _check_image(img)
    _check_buffers(out, out_len, ws)
    H, W = img.shape[0], img.shape[1]
    rc = _lib.lib().ngp_jpeg_encode(img.data_ptr(), H, W, int(quality), out.data_ptr(), out.numel(), out_len.data_ptr(),
                                    ws.data_ptr(), ws.numel(), _stream(img))
    _lib.check(rc, "ngp_jpeg_encode")


@torch.no_grad()
def encode_jpeg(img, quality=90):
    """the baseline JPEG file of an (H, W, 3) uint8 device image, as bytes (written into pinned host memory by the
    device; synchronises the current stream)"""
    img = _check_image(img)
    H, W = img.shape[0], img.shape[1]
    out = torch.empty(jpeg_capacity(H, W), dtype=torch.uint8, pin_memory=True)
    n = torch.zeros(1, dtype=torch.int64, pin_memory=True)
    encode_jpeg_into(img, out, n, jpeg_workspace(H, W, img.device), quality)
    torch.cuda.current_stream(img.device).synchronize()
    return out[:int(n[0])].numpy().tobytes()


def write_jpeg(path, img, quality=90):
    """write the baseline JPEG file of an (H, W, 3) uint8 device image to path"""
    data = encode_jpeg(img, quality)
    with open(path, "wb") as f:
        f.write(data)


class AviWriter:
    """A Motion-JPEG video file: AVI 1.0 (RIFF) with one `vids` / `MJPG` stream, every frame a complete JPEG in a `00dc`
    chunk (padded to an even length) appended by add(); close() appends the `idx1` index and patches the sizes, the
    frame count and dwSuggestedBufferSize (the largest frame) into the headers. fps is stored as dwRate / dwScale.
    An AVI 1.0 file holds at most 2^31 - 1 bytes; add() raises RuntimeError before a frame would pass that."""

    LIMIT = (1 << 31) - 1
    MOVI = 220  # file offset of the 'movi' tag, which the index offsets count from

    def __init__(self, path, W, H, fps):
        r = Fraction(fps).limit_denominator(100000)
        if r <= 0 or int(W) < 1 or int(H) < 1:
            raise RuntimeError("ngp_pl_b200.images.AviWriter: fps, W and H must be positive")
        self.W, self.H, self.rate, self.scale = int(W), int(H), r.numerator, r.denominator
        self.index = []  # (offset from the 'movi' tag, length) per frame
        self.end = self.MOVI + 4
        self.f = open(path, "wb")
        self.f.write(self._header())

    def _header(self):
        n, largest = len(self.index), max([size for _, size in self.index], default=0)
        strf = struct.pack("<IiiHH4sIiiII", 40, self.W, self.H, 1, 24, b"MJPG", self.W * self.H * 3, 0, 0, 0, 0)
        strh = struct.pack("<4s4sIHHIIIIIIIIhhhh", b"vids", b"MJPG", 0, 0, 0, 0, self.scale, self.rate, 0, n, largest,
                           0xFFFFFFFF, 0, 0, 0, self.W, self.H)
        avih = struct.pack("<14I", round(1e6 * self.scale / self.rate), 0, 0, 0x10, n, 0, 1, largest, self.W, self.H,
                           0, 0, 0, 0)
        chunk = lambda tag, data: tag + struct.pack("<I", len(data)) + data  # noqa: E731
        strl = chunk(b"LIST", b"strl" + chunk(b"strh", strh) + chunk(b"strf", strf))
        hdrl = chunk(b"LIST", b"hdrl" + chunk(b"avih", avih) + strl)
        riff = self.end + 8 + 16 * n  # with the index
        head = b"RIFF" + struct.pack("<I", riff - 8) + b"AVI " + hdrl + b"LIST" + struct.pack("<I", self.end - self.MOVI) + b"movi"
        assert len(head) == self.MOVI + 4
        return head

    def add(self, jpeg):
        """append one frame; jpeg: the bytes (or a buffer) of a complete JPEG file"""
        n = len(jpeg)
        padded = n + (n & 1)
        if self.end + 8 + padded + 8 + 16 * (len(self.index) + 1) > self.LIMIT:
            raise RuntimeError("ngp_pl_b200.images.AviWriter: frame %d would take the file past 2^31 - 1 bytes"
                               % len(self.index))
        self.f.write(b"00dc" + struct.pack("<I", n))
        self.f.write(jpeg)
        if n & 1:
            self.f.write(b"\0")
        self.index.append((self.end - self.MOVI, n))
        self.end += 8 + padded

    def close(self):
        if self.f is None:
            return
        self.f.write(b"idx1" + struct.pack("<I", 16 * len(self.index)))
        self.f.write(b"".join(struct.pack("<4sIII", b"00dc", 0x10, off, n) for off, n in self.index))
        self.f.seek(0)
        self.f.write(self._header())
        self.f.close()
        self.f = None


class ViewWriter:
    """Writes `{i:03d}.png` and `{i:03d}_d.png` of rendered views into a directory while the GPU renders on.

    submit(i, rgb, depth) enqueues, on the current stream, the view's images and both PNG encodes into one of `slots`
    mapped pinned host slots and records the slot's CUDA event; it never synchronises the stream. One writer thread
    waits on the events in submission order and writes the files. submit blocks only when every slot is still waiting
    to be written. close() waits for every file and joins the thread; an error of the writer is re-raised by the next
    submit or by close.

    With video_fps, the JPEG encodes of the same two images (quality video_quality) follow the PNG encodes into the
    slot, and the writer thread appends them, in submission order, to `rgb{video_tag}.avi` and `depth{video_tag}.avi`
    (AviWriter), finished by close(). png=False leaves the PNGs out; png_mode ("fixed" or "dynamic") is encode_png's
    mode."""

    def __init__(self, directory, H, W, device, slots=4, png=True, video_fps=None, video_quality=90, video_tag="",
                 png_mode="fixed"):
        _png_mode(png_mode)
        self.dir, self.H, self.W = directory, int(H), int(W)
        os.makedirs(directory, exist_ok=True)
        self.png, self.quality, self.png_mode = bool(png), int(video_quality), png_mode
        caps = [png_capacity(H, W)] * 2 * self.png + [jpeg_capacity(H, W)] * 2 * (video_fps is not None)
        self.rgb_img = torch.empty(H, W, 3, dtype=torch.uint8, device=device)
        self.depth_img = torch.empty(H, W, 3, dtype=torch.uint8, device=device)
        self.vi_ws = torch.empty(_lib.NGP_VIEW_IMAGES_WORKSPACE, dtype=torch.uint8, device=device)
        self.png_ws = png_workspace(H, W, device, png_mode) if self.png else None
        self.jpeg_ws = jpeg_workspace(H, W, device) if video_fps is not None else None
        self.videos = None if video_fps is None else [
            AviWriter(os.path.join(directory, "%s%s.avi" % (name, video_tag)), W, H, video_fps) for name in ("rgb", "depth")]
        # per slot: the files of one view, in the order [rgb PNG, depth PNG,] [rgb JPEG, depth JPEG]
        self.slots = [{"bufs": [torch.empty(cap, dtype=torch.uint8, pin_memory=True) for cap in caps],
                       "len": torch.zeros(len(caps), dtype=torch.int64, pin_memory=True),
                       "event": torch.cuda.Event()} for _ in range(slots)]
        self.free = queue.Queue()
        for k in range(slots):
            self.free.put(k)
        self.work = queue.Queue()
        self.error = None
        self.thread = threading.Thread(target=self._run, name="ngp-view-writer", daemon=True)
        self.thread.start()

    def _run(self):
        while True:
            item = self.work.get()
            if item is None:
                return
            i, k = item
            s = self.slots[k]
            try:
                if self.error is None:
                    s["event"].synchronize()
                    files = [buf[:int(n)].numpy().data for buf, n in zip(s["bufs"], s["len"])]
                    if self.png:
                        for name, data in zip(("%03d.png" % i, "%03d_d.png" % i), files):
                            with open(os.path.join(self.dir, name), "wb") as f:
                                f.write(data)
                    if self.videos is not None:
                        for video, data in zip(self.videos, files[-2:]):
                            video.add(data)
            except BaseException as e:  # handed to the submitting thread; later items are drained unwritten
                self.error = e
            finally:
                self.free.put(k)

    def _raise(self):
        if self.error is not None:
            raise RuntimeError("ngp_pl_b200.images: writing the view images failed: %r" % (self.error,)) from self.error

    def submit(self, i, rgb, depth):
        self._raise()
        k = self.free.get()
        self._raise()
        s = self.slots[k]
        view_images(rgb, depth, self.H, self.W, self.rgb_img, self.depth_img, self.vi_ws)
        j = 0
        if self.png:
            for img in (self.rgb_img, self.depth_img):
                encode_png_into(img, s["bufs"][j], s["len"][j:j + 1], self.png_ws, self.png_mode)
                j += 1
        if self.videos is not None:
            for img in (self.rgb_img, self.depth_img):
                encode_jpeg_into(img, s["bufs"][j], s["len"][j:j + 1], self.jpeg_ws, self.quality)
                j += 1
        s["event"].record(torch.cuda.current_stream(self.rgb_img.device))
        self.work.put((int(i), k))

    def close(self):
        if self.thread is not None:
            self.work.put(None)
            self.thread.join()
            self.thread = None
            for video in self.videos or ():
                video.close()
        self._raise()


@torch.no_grad()
def render_video(render_fn, poses, directions, img_wh, save_dir, fps=30, quality=90, exp_step_factor=0.0):
    """`rgb.avi` and `depth.avi` of a camera path, without ground truth: renders poses (n, 3, 4) camera-to-world in order
    and writes each view's rgb_image and depth_image as one Motion-JPEG frame of the two files in save_dir, through the
    ViewWriter the validation pass uses (the stream is never synchronised per view). render_fn(rays_o, rays_d) -> dict
    with 'rgb' (H*W, 3) and 'depth' (H*W,), or an NGP model, rendered with render(model, o, d, test_time=True,
    exp_step_factor=exp_step_factor). directions (H*W, 3) (synth.ray_directions); img_wh = (W, H)."""
    from . import synth
    if isinstance(render_fn, torch.nn.Module):
        from .models.rendering import render
        model = render_fn

        def render_fn(o, d):
            return render(model, o, d, test_time=True, exp_step_factor=exp_step_factor)
    if not isinstance(directions, torch.Tensor) or not directions.is_cuda:
        raise RuntimeError("ngp_pl_b200.images: directions must be a CUDA tensor")
    W, H = int(img_wh[0]), int(img_wh[1])
    writer = ViewWriter(save_dir, H, W, directions.device, png=False, video_fps=fps, video_quality=quality)
    try:
        for i in range(len(poses)):
            res = render_fn(*synth.get_rays(directions, poses[i]))
            writer.submit(i, res["rgb"].float().contiguous(), res["depth"].float().contiguous())
    finally:
        writer.close()
