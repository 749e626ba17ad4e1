"""Validation metrics of the reference's training loop on the device (reference metrics.py and train.py:187-237).

    psnr(image_pred, image_gt, valid_mask=None, reduction='mean')   reference metrics.py:14-15
    ssim(pred_img, gt_img, data_range=1.0)                          torchmetrics StructuralSimilarityIndexMeasure defaults
    evaluate(render_fn, poses, directions, images, img_wh, ...)     the validation pass: per-view PSNR and SSIM, gathered
                                                                    over the ranks as train.py:225-237 does

The arithmetic is one kernel per view, `ngp_image_metrics` (csrc/metrics.cu). Tensors must live on a CUDA device,
otherwise RuntimeError; there is no CPU path.
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


def _hwc(img):
    """(H, W, 3) or the reference's (1, 3, H, W) -> contiguous (H, W, 3)"""
    if img.dim() == 4 and img.shape[0] == 1 and img.shape[1] == 3:
        return img[0].permute(1, 2, 0).contiguous()
    if img.dim() == 3 and img.shape[2] == 3:
        return img.contiguous()
    raise RuntimeError("ngp_pl_b200.metrics.ssim: expected one (H, W, 3) or (1, 3, H, W) image, got %s" % (tuple(img.shape),))


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


def gather_metrics(local, n_views, n_pixels, world_size=1, rank=0, process_group=None):
    """Summary of the validation pass from this rank's per-view rows `local` (n_local, 3) float64 = [sum of squared
    errors, SSIM, total_samples] of the views shard_range(n_views, world_size, rank), in view order. With world_size > 1
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
    return {"psnr": sum(psnr_v) / n_views, "ssim": sum(ssim_v) / n_views, "psnr_per_view": psnr_v, "ssim_per_view": ssim_v,
            "total_samples": int(sum(r[2] for r in rows))}


@torch.no_grad()
def evaluate(render_fn, poses, directions, images, img_wh, world_size=1, rank=0, process_group=None, exp_step_factor=0.0):
    """The reference's validation pass (train.py:193-237) without writing images: renders this rank's share of the views
    (shard_range, the split bench.py's render_fps uses), runs ngp_image_metrics on each output on the same stream, reads
    the per-view results back once at the end and gathers them over the ranks.

    render_fn(rays_o, rays_d) -> dict with 'rgb' (H*W, 3) and 'total_samples'; an NGP model instead renders with
    render(model, o, d, test_time=True, exp_step_factor=exp_step_factor). poses (n_views, 3, 4) camera-to-world;
    directions (H*W, 3) (synth.ray_directions); images (n_views, H*W, 3) uint8 (read as v / 255) or float32, or a
    sequence of such views; img_wh = (W, H). Returns {'psnr', 'ssim'} (means over all views), {'psnr_per_view',
    'ssim_per_view'} in view order and 'total_samples' over all views."""
    from . import synth
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
    local = torch.zeros(hi - lo, 3, dtype=torch.float64, device=dev)
    ws = workspace(H, W, dev)
    for i in range(lo, hi):
        o, d = synth.get_rays(directions, poses[i])
        res = render_fn(o, d)
        image_metrics(res["rgb"].float().contiguous(), images[i].contiguous(), H, W, local[i - lo, 0], local[i - lo, 1], ws)
        local[i - lo, 2] = res["total_samples"]
    if world_size > 1:
        import torch.distributed as dist
        if dist.get_backend(process_group) != "nccl":
            local = local.cpu()
    return gather_metrics(local, n_views, H * W, world_size, rank, process_group)
