"""Validation metrics of the reference's training loop on the device (reference metrics.py and train.py:187-237).

    psnr(image_pred, image_gt, valid_mask=None, reduction='mean')   reference metrics.py:14-15
    ssim(pred_img, gt_img, data_range=1.0)                          torchmetrics StructuralSimilarityIndexMeasure defaults
    lpips(pred_img, gt_img, net)                                    torchmetrics LearnedPerceptualImagePatchSimilarity('vgg')
                                                                    of the reference's --eval_lpips (train.py:65-68, 209-213)
    evaluate(render_fn, poses, directions, images, img_wh, ...)     the validation pass: per-view PSNR and SSIM (and LPIPS
                                                                    given an LpipsNet), gathered over the ranks as
                                                                    train.py:225-237 does; with save_dir, the test-view
                                                                    PNGs of train.py:215-221 (images.py)

The arithmetic is one kernel per view, `ngp_image_metrics` (csrc/metrics.cu), and one `ngp_lpips` chain per view
(csrc/lpips.cu). Tensors must live on a CUDA device, otherwise RuntimeError; there is no CPU path.
"""
import math

import torch

from . import _lib
from .trainer import shard_range


def _chk(*tensors):
    for t in tensors:
        if not t.is_cuda:
            raise RuntimeError("ngp_pl_b200.metrics: argument must be a CUDA tensor")


def workspace(H, W, device):
    """zero-initialised workspace of ngp_image_metrics for H x W images (any later launch on one stream may reuse it)"""
    return torch.zeros(_lib.lib().ngp_image_metrics_workspace(int(H), int(W)), dtype=torch.uint8, device=device)


def image_metrics(pred, gt, H, W, out_sse, out_ssim, ws, data_range=1.0):
    """One ngp_image_metrics launch on the current stream, no synchronisation. pred: fp32 (H*W, 3); gt: the same layout,
    fp32 or uint8 (read as v / 255). out_sse, out_ssim: float64 CUDA tensors whose first element receives the sum of
    squared errors / the mean SSIM (a slot of a per-view array, `out[v]`); out_ssim None computes the squared error
    only. ws: `workspace(H, W, device)`."""
    _chk(pred, gt, out_sse, ws)
    if out_ssim is not None:
        _chk(out_ssim)
    if pred.dtype != torch.float32 or gt.dtype not in (torch.float32, torch.uint8):
        raise RuntimeError("ngp_pl_b200.metrics: pred must be float32 and gt float32 or uint8, got %s, %s" % (pred.dtype, gt.dtype))
    if pred.numel() != 3 * H * W or gt.numel() != 3 * H * W:
        raise RuntimeError("ngp_pl_b200.metrics: expected %d x %d RGB images, got %s and %s" % (H, W, tuple(pred.shape), tuple(gt.shape)))
    if not (pred.is_contiguous() and gt.is_contiguous()):
        raise RuntimeError("ngp_pl_b200.metrics: images must be contiguous")
    for o in (out_sse, out_ssim):
        if o is not None and o.dtype != torch.float64:
            raise RuntimeError("ngp_pl_b200.metrics: outputs must be float64")
    rc = _lib.lib().ngp_image_metrics(pred.data_ptr(), gt.data_ptr(), int(gt.dtype == torch.uint8), int(H), int(W),
                                      float(data_range), out_sse.data_ptr(), None if out_ssim is None else out_ssim.data_ptr(),
                                      ws.data_ptr(), ws.numel(), torch.cuda.current_stream(pred.device).cuda_stream)
    _lib.check(rc, "ngp_image_metrics")


@torch.no_grad()
def psnr(image_pred, image_gt, valid_mask=None, reduction='mean'):
    """reference metrics.py:14-15: -10 log10(mean squared error), a float32 device scalar; +inf for identical images.
    image_gt may be uint8 (read as v / 255). The mean over all values runs in ngp_image_metrics and needs RGB data
    (a multiple of 3 values); a valid_mask or reduction='none' is plain torch indexing, as in the reference."""
    _chk(image_pred, image_gt)
    if valid_mask is not None or reduction != 'mean':
        gt = image_gt.float() / 255 if image_gt.dtype == torch.uint8 else image_gt
        value = (image_pred - gt) ** 2
        if valid_mask is not None:
            value = value[valid_mask]
        if reduction == 'mean':
            return -10 * torch.log10(torch.mean(value))
        return -10 * torch.log10(value)
    n = image_pred.numel()
    if n % 3:
        raise RuntimeError("ngp_pl_b200.metrics.psnr: the mean over all values takes RGB data (a multiple of 3 values)")
    pred, gt = image_pred.contiguous(), image_gt.contiguous()
    sse = torch.empty(1, dtype=torch.float64, device=pred.device)
    image_metrics(pred, gt, 1, n // 3, sse, None, workspace(1, n // 3, pred.device))
    return (-10 * torch.log10(sse[0] / n)).float()


def _hwc(img, what="ssim"):
    """(H, W, 3) or the reference's (1, 3, H, W) -> contiguous (H, W, 3)"""
    if img.dim() == 4 and img.shape[0] == 1 and img.shape[1] == 3:
        return img[0].permute(1, 2, 0).contiguous()
    if img.dim() == 3 and img.shape[2] == 3:
        return img.contiguous()
    raise RuntimeError("ngp_pl_b200.metrics.%s: expected one (H, W, 3) or (1, 3, H, W) image, got %s" % (what, tuple(img.shape)))


@torch.no_grad()
def ssim(pred_img, gt_img, data_range=1.0):
    """torchmetrics StructuralSimilarityIndexMeasure(data_range=data_range) of one RGB image (its defaults: Gaussian
    window 11 taps, sigma 1.5, windows wholly inside the image), a float32 device scalar. (H, W, 3) or (1, 3, H, W);
    gt_img may be uint8 (read as v / 255). H and W must be at least 11."""
    _chk(pred_img, gt_img)
    p, g = _hwc(pred_img), _hwc(gt_img)
    if p.shape != g.shape:
        raise RuntimeError("ngp_pl_b200.metrics.ssim: shapes differ: %s vs %s" % (tuple(p.shape), tuple(g.shape)))
    H, W = p.shape[0], p.shape[1]
    out = torch.empty(2, dtype=torch.float64, device=p.device)
    image_metrics(p, g, H, W, out[0], out[1], workspace(H, W, p.device), data_range)
    return out[1].float()


# LPIPS v0.1 with the VGG-16 backbone. VGG keys: torchvision's vgg16().state_dict() names (extra keys, such as the
# classifier's, are ignored). Linear-layer keys: the `lpips` package's v0.1 weight file, lin{t}.model.1.weight of shape
# (1, C, 1, 1) -- recalled from that package's sources, as are the scaling-layer constants and the 1e-10 of the
# normalisation (csrc/lpips.cu, oracle/lpips_ref.py).
LPIPS_CONVS = ((0, 3, 64), (2, 64, 64), (5, 64, 128), (7, 128, 128), (10, 128, 256), (12, 256, 256), (14, 256, 256),
               (17, 256, 512), (19, 512, 512), (21, 512, 512), (24, 512, 512), (26, 512, 512), (28, 512, 512))
LPIPS_TAP_CHANNELS = (64, 128, 256, 512, 512)


class LpipsNet:
    """The packed weights of LPIPS-VGG (the layout of ngp_lpips in include/ngp_b200.h) in one device buffer. Built from
    the caller's own files; nothing is ever downloaded."""

    def __init__(self, weights):
        self.weights = weights  # uint8 tensor of ngp_lpips_weights_bytes() bytes

    @classmethod
    def from_state_dicts(cls, vgg, lin, device):
        """vgg: a torchvision vgg16 state_dict (e.g. the ImageNet checkpoint); lin: the LPIPS v0.1 'vgg' linear layers.
        Every key and shape is checked; RuntimeError names the first mismatch (or a negative linear weight)."""
        def get(sd, key, shape):
            if key not in sd:
                raise RuntimeError("ngp_pl_b200.metrics.LpipsNet: missing key %r" % key)
            t = torch.as_tensor(sd[key])
            if tuple(t.shape) != shape:
                raise RuntimeError("ngp_pl_b200.metrics.LpipsNet: %r has shape %s, expected %s" % (key, tuple(t.shape), shape))
            return t.detach().cpu().float()
        halves, floats = [], []
        for i, cin, cout in LPIPS_CONVS:
            w = get(vgg, "features.%d.weight" % i, (cout, cin, 3, 3)).permute(0, 2, 3, 1)  # [n][ky][kx][c]: K-major
            if cin == 3:
                w = torch.nn.functional.pad(w, (0, 13))  # conv1_1 reads 16 channels, 3..15 zero
            halves.append(w.half().reshape(-1))
        biases = [get(vgg, "features.%d.bias" % i, (cout,)) for i, _, cout in LPIPS_CONVS]
        for t, c in enumerate(LPIPS_TAP_CHANNELS):
            key = "lin%d.model.1.weight" % t
            w = get(lin, key, (1, c, 1, 1)).reshape(-1)
            if not bool((w >= 0).all()):
                raise RuntimeError("ngp_pl_b200.metrics.LpipsNet: %r has negative weights" % key)
            floats.append(w)
        packed = torch.cat([torch.cat(halves).view(torch.uint8), torch.cat(biases + floats).view(torch.uint8)])
        want = _lib.lib().ngp_lpips_weights_bytes()
        if packed.numel() != want:
            raise RuntimeError("ngp_pl_b200.metrics.LpipsNet: packed %d bytes, the library expects %d" % (packed.numel(), want))
        return cls(packed.to(device))

    @classmethod
    def from_files(cls, vgg_path, lin_path, device):
        """the same from two torch.load files, e.g. torchvision's vgg16-397923af.pth and the lpips package's v0.1 vgg.pth"""
        load = lambda p: torch.load(p, map_location="cpu", weights_only=True)  # noqa: E731
        return cls.from_state_dicts(load(vgg_path), load(lin_path), device)


def lpips_workspace(H, W, device):
    """workspace of ngp_lpips for H x W images (no initialisation needed; one launch chain at a time)"""
    n = _lib.lib().ngp_lpips_workspace(int(H), int(W))
    if n == 0:
        raise RuntimeError("ngp_pl_b200.metrics.lpips: H and W must be at least 16, got %d x %d" % (H, W))
    return torch.empty(n, dtype=torch.uint8, device=device)


def lpips_metric(net, pred, gt, H, W, out, ws):
    """One ngp_lpips chain on the current stream, no synchronisation. pred: fp32 (H*W, 3) in [0, 1]; gt: the same
    layout, fp32 or uint8 (read as v / 255); out: a float64 CUDA tensor whose first element receives the LPIPS;
    ws: `lpips_workspace(H, W, device)`."""
    _chk(pred, gt, out, ws, net.weights)
    if pred.dtype != torch.float32 or gt.dtype not in (torch.float32, torch.uint8) or out.dtype != torch.float64:
        raise RuntimeError("ngp_pl_b200.metrics.lpips: pred must be float32, gt float32 or uint8 and out float64")
    if pred.numel() != 3 * H * W or gt.numel() != 3 * H * W or not (pred.is_contiguous() and gt.is_contiguous()):
        raise RuntimeError("ngp_pl_b200.metrics.lpips: expected contiguous %d x %d RGB images, got %s and %s"
                           % (H, W, tuple(pred.shape), tuple(gt.shape)))
    rc = _lib.lib().ngp_lpips(net.weights.data_ptr(), pred.data_ptr(), gt.data_ptr(), int(gt.dtype == torch.uint8), int(H),
                              int(W), out.data_ptr(), ws.data_ptr(), ws.numel(),
                              torch.cuda.current_stream(pred.device).cuda_stream)
    _lib.check(rc, "ngp_lpips")


@torch.no_grad()
def lpips(pred_img, gt_img, net):
    """LPIPS-VGG of one view, a float32 device scalar: the reference's
    LearnedPerceptualImagePatchSimilarity('vgg')(clip(pred*2-1, -1, 1), clip(gt*2-1, -1, 1)). Unlike that call, the
    images are passed in [0, 1]; the 2x - 1 and the clip happen here. (H, W, 3) or (1, 3, H, W); gt_img may be uint8
    (read as v / 255). H and W must be at least 16. net: an LpipsNet."""
    _chk(pred_img, gt_img)
    p, g = _hwc(pred_img, "lpips"), _hwc(gt_img, "lpips")
    if p.shape != g.shape:
        raise RuntimeError("ngp_pl_b200.metrics.lpips: shapes differ: %s vs %s" % (tuple(p.shape), tuple(g.shape)))
    H, W = p.shape[0], p.shape[1]
    out = torch.empty(1, dtype=torch.float64, device=p.device)
    lpips_metric(net, p, g, H, W, out, lpips_workspace(H, W, p.device))
    return out[0].float()


def gather_metrics(local, n_views, n_pixels, world_size=1, rank=0, process_group=None):
    """Summary of the validation pass from this rank's per-view rows `local` (n_local, 3) float64 = [sum of squared
    errors, SSIM, total_samples] of the views shard_range(n_views, world_size, rank), in view order; a 4th column, the
    view's LPIPS, adds {'lpips', 'lpips_per_view'} to the result. With world_size > 1
    the rows of every rank are all_gathered (as the reference's all_gather_ddp_if_available, train.py:225-237) and
    concatenated in view order; `local` must be on the device the process group's backend communicates from."""
    local = local.to(torch.float64)
    if world_size > 1:
        import torch.distributed as dist
        per = -(-n_views // world_size)  # the largest shard; smaller ones are padded
        buf = torch.zeros(per, local.shape[1], dtype=torch.float64, device=local.device)
        buf[:local.shape[0]] = local
        parts = [torch.empty_like(buf) for _ in range(world_size)]
        dist.all_gather(parts, buf, group=process_group)
        spans = [shard_range(n_views, world_size, r) for r in range(world_size)]
        local = torch.cat([p[:hi - lo] for p, (lo, hi) in zip(parts, spans)])
    rows = local.cpu().tolist()
    if len(rows) != n_views:
        raise RuntimeError("ngp_pl_b200.metrics: %d per-view rows for %d views" % (len(rows), n_views))
    psnr_v = [-10 * math.log10(r[0] / (3 * n_pixels)) if r[0] > 0 else math.inf for r in rows]
    ssim_v = [r[1] for r in rows]
    res = {"psnr": sum(psnr_v) / n_views, "ssim": sum(ssim_v) / n_views, "psnr_per_view": psnr_v, "ssim_per_view": ssim_v,
           "total_samples": int(sum(r[2] for r in rows))}
    if local.shape[1] == 4:
        lpips_v = [r[3] for r in rows]
        res["lpips"], res["lpips_per_view"] = sum(lpips_v) / n_views, lpips_v
    return res


@torch.no_grad()
def evaluate(render_fn, poses, directions, images, img_wh, world_size=1, rank=0, process_group=None, exp_step_factor=0.0,
             lpips_net=None, save_dir=None, video_fps=None, video_quality=90, png_mode="fixed"):
    """The reference's validation pass (train.py:193-237): renders this rank's share of the views
    (shard_range, the split bench.py's render_fps uses), runs ngp_image_metrics on each output on the same stream, reads
    the per-view results back once at the end and gathers them over the ranks.

    render_fn(rays_o, rays_d) -> dict with 'rgb' (H*W, 3) and 'total_samples'; an NGP model instead renders with
    render(model, o, d, test_time=True, exp_step_factor=exp_step_factor). poses (n_views, 3, 4) camera-to-world;
    directions (H*W, 3) (synth.ray_directions); images (n_views, H*W, 3) uint8 (read as v / 255) or float32, or a
    sequence of such views; img_wh = (W, H). Returns {'psnr', 'ssim'} (means over all views), {'psnr_per_view',
    'ssim_per_view'} in view order and 'total_samples' over all views. With lpips_net (an LpipsNet) each view's LPIPS
    is launched on the same stream after its PSNR and SSIM, and the result gains 'lpips' and 'lpips_per_view'.

    With save_dir (created if needed), every view of this rank's shard is also written as the reference's validation
    pass writes it (train.py:215-221): `{i:03d}.png` = (rgb * 255).astype(uint8) and `{i:03d}_d.png` = depth2img(depth),
    i the global view index. render_fn's result must then hold 'depth'. Each view's images and PNGs are enqueued on the
    render stream after its metrics, into a small ring of pinned host slots that one writer thread empties while the GPU
    renders the next view (images.ViewWriter); the stream is not synchronised per view, the call returns once every file
    is written, and the returned dict is the one without save_dir. png_mode "dynamic" (images.encode_png's mode) writes
    smaller files of the same arrays; "fixed", the default, is the faster stream.

    With video_fps as well (RuntimeError without save_dir), the same two images of every view of the shard, in view
    order, are also the frames of the Motion-JPEG videos `rgb.avi` and `depth.avi` in save_dir (the reference's rgb.mp4
    and depth.mp4, made from those PNGs; images.AviWriter), JPEG-encoded at video_quality on the render stream after the
    PNG encodes. With world_size > 1 each rank writes its shard as `rgb.rank{r}.avi` / `depth.rank{r}.avi`."""
    from . import synth
    from .images import PNG_MODES
    if png_mode not in PNG_MODES:
        raise ValueError("ngp_pl_b200.metrics.evaluate: png_mode must be one of %s, got %r" % (sorted(PNG_MODES), png_mode))
    if isinstance(render_fn, torch.nn.Module):
        from .models.rendering import render
        model = render_fn

        def render_fn(o, d):
            return render(model, o, d, test_time=True, exp_step_factor=exp_step_factor)
    W, H = int(img_wh[0]), int(img_wh[1])
    _chk(poses, directions)
    n_views = len(poses)
    lo, hi = shard_range(n_views, world_size, rank)
    dev = directions.device
    local = torch.zeros(hi - lo, 3 if lpips_net is None else 4, dtype=torch.float64, device=dev)
    ws = workspace(H, W, dev)
    ws_lpips = None if lpips_net is None else lpips_workspace(H, W, dev)
    writer = None
    if video_fps is not None and save_dir is None:
        raise RuntimeError("ngp_pl_b200.metrics.evaluate: video_fps needs save_dir")
    if save_dir is not None:
        from .images import ViewWriter
        writer = ViewWriter(save_dir, H, W, dev, video_fps=video_fps, video_quality=video_quality,
                            video_tag=".rank%d" % rank if world_size > 1 else "", png_mode=png_mode)
    try:
        for i in range(lo, hi):
            o, d = synth.get_rays(directions, poses[i])
            res = render_fn(o, d)
            pred, gt = res["rgb"].float().contiguous(), images[i].contiguous()
            image_metrics(pred, gt, H, W, local[i - lo, 0], local[i - lo, 1], ws)
            if lpips_net is not None:
                lpips_metric(lpips_net, pred, gt, H, W, local[i - lo, 3], ws_lpips)
            local[i - lo, 2] = res["total_samples"]
            if writer is not None:
                if "depth" not in res:
                    raise RuntimeError("ngp_pl_b200.metrics.evaluate: save_dir needs 'depth' in the render result")
                writer.submit(i, pred, res["depth"].float().contiguous())
    finally:
        if writer is not None:
            writer.close()
    if world_size > 1:
        import torch.distributed as dist
        if dist.get_backend(process_group) != "nccl":
            local = local.cpu()
    return gather_metrics(local, n_views, H * W, world_size, rank, process_group)
