"""Test-view images of the validation pass on the device (reference train.py:215-221): the quantised RGB image and the
turbo depth image of a render, and PNG files of both.

    rgb_image(rgb, H, W)     (rgb_pred * 255).astype(np.uint8): an (H, W, 3) uint8 device tensor
    depth_image(depth, H, W) depth2img(depth) (train.py:45-50): per-view min/max, * 255, uint8, cv2's turbo colour map;
                             an (H, W, 3) uint8 device tensor whose channels are cv2's B, G, R -- the array the reference
                             writes to its `_d.png` files, blue in the red position included
    encode_png(img)          the PNG file of an (H, W, 3) uint8 device image, as bytes
    write_png(path, img)     the same, written to `path`

The arithmetic is ngp_view_images and ngp_png_encode (csrc/images.cu); the byte stream of the PNG is specified in
include/ngp_b200.h. Tensors must live on a CUDA device, otherwise RuntimeError; there is no CPU path. metrics.evaluate
(save_dir=...) writes every view of the validation pass through `ViewWriter`.
"""
import os
import queue
import threading

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


def png_workspace(H, W, device):
    png_capacity(H, W)
    return torch.empty(_lib.lib().ngp_png_workspace(int(H), int(W)), dtype=torch.uint8, device=device)


def encode_png_into(img, out, out_len, ws):
    """One ngp_png_encode call on the current stream, no synchronisation: the file of img ((H, W, 3) uint8, device)
    into out (uint8, device or pinned host memory, at least png_capacity(H, W) bytes) and its length into out_len[0]
    (int64, device or pinned host memory). ws: png_workspace(H, W, device)."""
    img = _check_image(img)
    for t, dt in ((out, torch.uint8), (out_len, torch.int64), (ws, torch.uint8)):
        if not isinstance(t, torch.Tensor) or t.dtype != dt or not t.is_contiguous():
            raise RuntimeError("ngp_pl_b200.images: out, out_len and ws must be contiguous uint8 / int64 / uint8 tensors")
        if not (t.is_cuda or t.is_pinned()):
            raise RuntimeError("ngp_pl_b200.images: out and out_len must be CUDA or pinned host tensors")
    if not ws.is_cuda:
        raise RuntimeError("ngp_pl_b200.images: the workspace must be a CUDA tensor")
    H, W = img.shape[0], img.shape[1]
    rc = _lib.lib().ngp_png_encode(img.data_ptr(), H, W, out.data_ptr(), out.numel(), out_len.data_ptr(), ws.data_ptr(),
                                   ws.numel(), _stream(img))
    _lib.check(rc, "ngp_png_encode")


@torch.no_grad()
def encode_png(img):
    """the PNG file of an (H, W, 3) uint8 device image, as bytes (written into pinned host memory by the device, so only
    the file's bytes cross PCIe; synchronises the current stream)"""
    img = _check_image(img)
    H, W = img.shape[0], img.shape[1]
    out = torch.empty(png_capacity(H, W), dtype=torch.uint8, pin_memory=True)
    n = torch.zeros(1, dtype=torch.int64, pin_memory=True)
    encode_png_into(img, out, n, png_workspace(H, W, img.device))
    torch.cuda.current_stream(img.device).synchronize()
    return out[:int(n[0])].numpy().tobytes()


def write_png(path, img):
    """write the PNG file of an (H, W, 3) uint8 device image to path"""
    data = encode_png(img)
    with open(path, "wb") as f:
        f.write(data)


class ViewWriter:
    """Writes `{i:03d}.png` and `{i:03d}_d.png` of rendered views into a directory while the GPU renders on.

    submit(i, rgb, depth) enqueues, on the current stream, the view's images and both PNG encodes into one of `slots`
    mapped pinned host slots and records the slot's CUDA event; it never synchronises the stream. One writer thread
    waits on the events in submission order and writes the files. submit blocks only when every slot is still waiting
    to be written. close() waits for every file and joins the thread; an error of the writer is re-raised by the next
    submit or by close."""

    def __init__(self, directory, H, W, device, slots=4):
        self.dir, self.H, self.W = directory, int(H), int(W)
        os.makedirs(directory, exist_ok=True)
        cap = png_capacity(H, W)
        self.rgb_img = torch.empty(H, W, 3, dtype=torch.uint8, device=device)
        self.depth_img = torch.empty(H, W, 3, dtype=torch.uint8, device=device)
        self.vi_ws = torch.empty(_lib.NGP_VIEW_IMAGES_WORKSPACE, dtype=torch.uint8, device=device)
        self.png_ws = png_workspace(H, W, device)
        self.slots = [{"rgb": torch.empty(cap, dtype=torch.uint8, pin_memory=True),
                       "depth": torch.empty(cap, dtype=torch.uint8, pin_memory=True),
                       "len": torch.zeros(2, dtype=torch.int64, pin_memory=True),
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
                    n_rgb, n_depth = (int(v) for v in s["len"])
                    for name, buf, n in (("%03d.png" % i, s["rgb"], n_rgb), ("%03d_d.png" % i, s["depth"], n_depth)):
                        with open(os.path.join(self.dir, name), "wb") as f:
                            f.write(buf[:n].numpy().data)
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
        encode_png_into(self.rgb_img, s["rgb"], s["len"][0:1], self.png_ws)
        encode_png_into(self.depth_img, s["depth"], s["len"][1:2], self.png_ws)
        s["event"].record(torch.cuda.current_stream(self.rgb_img.device))
        self.work.put((int(i), k))

    def close(self):
        if self.thread is not None:
            self.work.put(None)
            self.thread.join()
            self.thread = None
        self._raise()
