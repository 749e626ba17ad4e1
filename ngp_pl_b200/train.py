"""Train a scene from the command line on the fused trainer: the reference's `train.py`, flag for flag.

    python -m ngp_pl_b200.train --root_dir data/lego --dataset_name nerf --exp_name lego
    torchrun --nproc_per_node 4 -m ngp_pl_b200.train --root_dir ... --num_gpus 4

What a run does, in the reference's order (train.py): load the `--split` and `test` views onto the device
(`datasets.load_scene`), register the occupancy buffers and mark the cells no training camera sees
(`mark_invisible_cells`), build the `Trainer` (cosine learning rate stepped per epoch, `exp_step_factor` 1/256 for
`--scale` > 0.5, the background rule of rendering.py:153-161, `erode` for COLMAP scenes), capture the step and train
`num_epochs * epoch_steps` steps, then run the validation pass once (`metrics.evaluate`). Every step's training scalars
are recorded on the device (`Trainer(log_rows=...)`) and drained about every 100 steps without a host synchronisation.

Files, under `--out_dir` (default `.`):
  logs/{dataset_name}/{exp_name}/version_{k}/scalars.csv   header `step,loss,psnr,rm_s,vr_s,lr` (+ `distortion`), one row
                                                           per training step, then one `tag,value` row per test metric
                                                           (`test/psnr`, `test/ssim`, `test/lpips_vgg`); the same tags as
                                                           TensorBoard events there when torch.utils.tensorboard imports
  ckpts/{dataset_name}/{exp_name}/epoch={num_epochs-1}.ckpt       {'epoch', 'global_step', 'state_dict'}: the keys of
                                                           the reference's NeRFSystem (`model.*`, `directions`, `poses`)
  ckpts/{dataset_name}/{exp_name}/epoch={num_epochs-1}_slim.ckpt  what the reference's utils.slim_ckpt makes of it
  results/{dataset_name}/{exp_name}/{i:03d}.png, {i:03d}_d.png    unless --no_save_test (+ rgb.avi / depth.avi with
                                                           --video_fps)

Refused before any GPU work: the loaders that are not built (nsvf, nerfpp, rtmv), `--use_exposure`, `--optimize_ext`,
`--split trainvaltest`, `--eval_lpips` without `--lpips_vgg` / `--lpips_lin`, `--num_gpus` > 1 outside torchrun,
`--ckpt_path` without `--val_only` (resuming the optimiser state is not supported; `--weight_path` loads weights).
"""
import argparse
import csv
import json
import os
import sys
import time

DATASETS_BUILT = ("nerf", "colmap")
SPLITS_LOADED = ("train", "trainval")  # of the reference's choices, those datasets.load_scene accepts
DRAIN_EVERY = 100
LOG_ROWS = 256


def get_parser():
    p = argparse.ArgumentParser(prog="python -m ngp_pl_b200.train",
                                description="Train (or evaluate) an Instant-NGP scene on the fused H100 trainer.")
    # ---- the reference's opt.py: same names, types, defaults and choices (the default dataset excepted) ----
    p.add_argument("--root_dir", type=str, required=True, help="scene directory")
    p.add_argument("--dataset_name", type=str, default="nerf", choices=["nerf", "nsvf", "colmap", "nerfpp", "rtmv"],
                   help="scene format; 'nerf' and 'colmap' are loaded (the reference defaults to 'nsvf')")
    p.add_argument("--split", type=str, default="train", choices=["train", "trainval", "trainvaltest"],
                   help="views to train on")
    p.add_argument("--downsample", type=float, default=1.0, help="image downsample factor (<= 1)")
    p.add_argument("--scale", type=float, default=0.5, help="the scene lies in [-scale, scale]^3")
    p.add_argument("--use_exposure", action="store_true", default=False, help="HDR exposure (not supported)")
    p.add_argument("--distortion_loss_w", type=float, default=0, help="weight of the distortion loss (0 = off)")
    p.add_argument("--batch_size", type=int, default=8192, help="rays per step")
    p.add_argument("--ray_sampling_strategy", type=str, default="all_images", choices=["all_images", "same_image"],
                   help="draw a batch's pixels from all images, or from one image per batch")
    p.add_argument("--num_epochs", type=int, default=30, help="epochs of --epoch_steps steps")
    p.add_argument("--num_gpus", type=int, default=1, help="GPUs; more than one needs torchrun with as many ranks")
    p.add_argument("--lr", type=float, default=1e-2, help="initial learning rate")
    p.add_argument("--optimize_ext", action="store_true", default=False, help="camera pose refinement (not supported)")
    p.add_argument("--random_bg", action="store_true", default=False,
                   help="a random background colour per batch (real scenes only)")
    p.add_argument("--eval_lpips", action="store_true", default=False,
                   help="also LPIPS-VGG in the validation pass (needs --lpips_vgg and --lpips_lin)")
    p.add_argument("--val_only", action="store_true", default=False, help="only the validation pass of --ckpt_path")
    p.add_argument("--no_save_test", action="store_true", default=False, help="do not write the test-view images")
    p.add_argument("--exp_name", type=str, default="exp", help="experiment name")
    p.add_argument("--ckpt_path", type=str, default=None, help="checkpoint to validate (with --val_only)")
    p.add_argument("--weight_path", type=str, default=None, help="weights to start from (Lightning-shaped or slim)")
    # ---- additions ----
    p.add_argument("--seed", type=int, default=0, help="seed of the initial weights and of the device batch draws")
    p.add_argument("--out_dir", type=str, default=".", help="root of results/, ckpts/ and logs/")
    p.add_argument("--epoch_steps", type=int, default=1000, help="steps per epoch (the reference's datasets/base.py)")
    p.add_argument("--lpips_vgg", type=str, default=None, help="torchvision VGG-16 weights for --eval_lpips")
    p.add_argument("--lpips_lin", type=str, default=None, help="LPIPS v0.1 'vgg' linear layers for --eval_lpips")
    p.add_argument("--video_fps", type=float, default=None, help="also write rgb.avi / depth.avi at this frame rate")
    return p


def check_args(args, parser, environ=None):
    """The combinations this command refuses, before any GPU work: parser.error() (exit status 2) names the flag."""
    env = os.environ if environ is None else environ
    if args.dataset_name not in DATASETS_BUILT:
        parser.error("--dataset_name %s: only %s scenes are loaded here" % (args.dataset_name, " and ".join(DATASETS_BUILT)))
    if args.use_exposure:
        parser.error("--use_exposure: HDR exposure is not supported")
    if args.optimize_ext:
        parser.error("--optimize_ext: camera pose refinement is not supported")
    if args.split not in SPLITS_LOADED:
        parser.error("--split %s: the loaders take %s" % (args.split, " or ".join(SPLITS_LOADED)))
    if args.eval_lpips:
        for flag, path in (("--lpips_vgg", args.lpips_vgg), ("--lpips_lin", args.lpips_lin)):
            if not path or not os.path.isfile(path):
                parser.error("--eval_lpips needs %s, a weight file (nothing is downloaded); got %r" % (flag, path))
    world = int(env.get("WORLD_SIZE", "0") or 0)
    if args.num_gpus > 1 and world == 0:
        parser.error("--num_gpus %d: run under torchrun with %d ranks" % (args.num_gpus, args.num_gpus))
    if world and args.num_gpus != world:
        parser.error("--num_gpus %d, but torchrun started %d ranks" % (args.num_gpus, world))
    if args.num_gpus < 1:
        parser.error("--num_gpus must be at least 1")
    if args.val_only and not args.ckpt_path:
        parser.error("--val_only needs --ckpt_path")
    if args.ckpt_path and not args.val_only:
        parser.error("--ckpt_path: resuming the optimiser state is not supported; use --weight_path to start from "
                     "saved weights, or --val_only to validate the checkpoint")
    if args.batch_size < 1 or args.num_epochs < 1 or args.epoch_steps < 1:
        parser.error("--batch_size, --num_epochs and --epoch_steps must be at least 1")
    return args


def parse_args(argv=None):
    parser = get_parser()
    return check_args(parser.parse_args(argv), parser)


def trainer_settings(args):
    """Trainer keyword arguments of a run, as the reference's train.py sets its render and loss up"""
    from .trainer import CosineAnnealingLR
    exp_step_factor = 1 / 256 if args.scale > 0.5 else 0.0      # train.py:95-96
    synthetic = exp_step_factor == 0                             # rendering.py:153-161
    return dict(n_rays=args.batch_size, lr=args.lr, exp_step_factor=exp_step_factor,
                bg=(1.0, 1.0, 1.0) if synthetic else (0.0, 0.0, 0.0), random_bg=bool(args.random_bg) and not synthetic,
                erode=args.dataset_name == "colmap",             # train.py:163
                lambda_distortion=args.distortion_loss_w, ray_sampling_strategy=args.ray_sampling_strategy,
                lr_schedule=CosineAnnealingLR(args.lr, T_max=args.num_epochs, steps_per_epoch=args.epoch_steps),
                seed=args.seed)


# ---- checkpoints --------------------------------------------------------------------------------------------------------
def checkpoint(model, directions, poses, epoch, global_step):
    """what the reference's ModelCheckpoint(save_weights_only=True) keeps of its NeRFSystem"""
    sd = {"model." + k: v.detach().cpu() for k, v in model.state_dict().items()}
    sd["directions"] = directions.detach().cpu()
    sd["poses"] = poses.detach().cpu()
    return {"epoch": int(epoch), "global_step": int(global_step), "state_dict": sd}


def slim_state_dict(ckpt):
    """the reference's utils.slim_ckpt (save_poses=False) of a checkpoint dict: its state_dict without the buffers a
    trained model does not need to render"""
    drop = {"directions", "model.density_grid", "model.grid_coords", "poses"}
    return {k: v for k, v in ckpt["state_dict"].items() if k not in drop and not k.startswith("val_lpips")}


def load_weights(model, path):
    """the reference's utils.load_ckpt: a Lightning-shaped ({'state_dict': ...}) or slim file; keys under `model.` are
    loaded (prefix stripped) over the model's own state, the others ignored"""
    import torch
    ck = torch.load(path, map_location="cpu", weights_only=True)
    if "state_dict" in ck:
        ck = ck["state_dict"]
    sd = model.state_dict()
    sd.update({k[len("model."):]: v for k, v in ck.items() if k.startswith("model.")})
    model.load_state_dict(sd)


# ---- scalar log ---------------------------------------------------------------------------------------------------------
def next_version(log_root):
    ks = []
    if os.path.isdir(log_root):
        for d in os.listdir(log_root):
            if d.startswith("version_") and d[len("version_"):].isdigit():
                ks.append(int(d[len("version_"):]))
    return os.path.join(log_root, "version_%d" % (max(ks) + 1 if ks else 0))


class ScalarLog:
    """scalars.csv (+ TensorBoard events when torch.utils.tensorboard imports) of one run"""

    def __init__(self, directory, n_rays, distortion):
        os.makedirs(directory, exist_ok=True)
        self.n_rays, self.distortion = n_rays, distortion
        self.f = open(os.path.join(directory, "scalars.csv"), "w", newline="")
        self.w = csv.writer(self.f)
        self.w.writerow(["step", "loss", "psnr", "rm_s", "vr_s", "lr"] + (["distortion"] if distortion else []))
        self.tb = None
        try:
            from torch.utils.tensorboard import SummaryWriter
            self.tb = SummaryWriter(directory)
        except Exception:
            self.tb = None

    def steps(self, rows):
        for r in rows:
            vals = [r["loss"], r["psnr"], r["rm_samples"] / self.n_rays, r["vr_samples"] / self.n_rays, r["lr"]]
            if self.distortion:
                vals.append(r["distortion"])
            self.w.writerow([r["step"]] + [repr(float(v)) for v in vals])
            if self.tb is not None:
                for tag, v in zip(("train/loss", "train/psnr", "train/rm_s", "train/vr_s", "lr", "train/distortion"), vals):
                    self.tb.add_scalar(tag, v, r["step"])

    def metric(self, tag, value, step):
        self.w.writerow([tag, repr(float(value))])
        if self.tb is not None:
            self.tb.add_scalar(tag, value, step)

    def close(self):
        self.f.close()
        if self.tb is not None:
            self.tb.close()


def progress(rows, total, n_rays):
    r = rows[-1]
    k = len(rows)
    mean = lambda key: sum(x[key] for x in rows) / k  # noqa: E731
    return ("step %d/%d  loss %.5f  psnr %.2f  rm_s %.1f  vr_s %.1f  lr %.3g"
            % (r["step"] + 1, total, mean("loss"), mean("psnr"), mean("rm_samples") / n_rays, mean("vr_samples") / n_rays,
               r["lr"]))


# ---- the run --------------------------------------------------------------------------------------------------------------
def run(args):
    import torch
    from . import datasets, metrics
    from .models.networks import NGP
    from .trainer import Trainer

    world = int(os.environ.get("WORLD_SIZE", "1") or 1)
    rank = int(os.environ.get("RANK", "0") or 0)
    local = int(os.environ.get("LOCAL_RANK", "0") or 0)
    if not torch.cuda.is_available():
        raise SystemExit("ngp_pl_b200.train: no CUDA device (there is no CPU path)")
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    pg = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=dev)
        pg = dist.group.WORLD
    torch.manual_seed(args.seed)
    out = os.path.abspath(args.out_dir)
    name = (args.dataset_name, args.exp_name)
    ckpt_dir = os.path.join(out, "ckpts", *name)
    save_dir = None if args.no_save_test else os.path.join(out, "results", *name)
    lpips_net = metrics.LpipsNet.from_files(args.lpips_vgg, args.lpips_lin, dev) if args.eval_lpips else None

    test = datasets.load_scene(args.dataset_name, args.root_dir, "test", args.downsample, dev)
    settings = trainer_settings(args)
    model = NGP(scale=args.scale).to(dev)
    G = model.grid_size
    model.register_buffer("density_grid", torch.zeros(model.cascades, G ** 3, device=dev))     # train.py:72-76
    model.register_buffer("grid_coords", torch.stack(torch.meshgrid(
        *[torch.arange(G, dtype=torch.int32, device=dev)] * 3, indexing="ij"), -1).reshape(-1, 3))

    log = None
    if rank == 0:
        log_dir = next_version(os.path.join(out, "logs", *name))
        log = ScalarLog(log_dir, args.batch_size, args.distortion_loss_w > 0)
        with open(os.path.join(log_dir, "hparams.json"), "w") as f:
            shown = {k: v for k, v in settings.items() if k != "lr_schedule"}
            json.dump(dict(vars(args), trainer=shown, world_size=world), f, indent=1)
    total = args.num_epochs * args.epoch_steps
    t_train = 0.0
    try:
        if args.val_only:
            load_weights(model, args.ckpt_path)
            step = 0
        else:
            train = datasets.load_scene(args.dataset_name, args.root_dir, args.split, args.downsample, dev)
            if args.weight_path:
                load_weights(model, args.weight_path)
            model.mark_invisible_cells(train.K, train.poses, train.img_wh)                       # train.py:155-157
            ddp = ("p2p" if world <= 4 else "nvls") if world > 1 else "nccl"
            tr = Trainer(model, process_group=pg, world_size=world, rank=rank, ddp=ddp, log_rows=LOG_ROWS, **settings)
            tr.attach_bank(train)
            t0 = time.perf_counter()
            tr.capture()
            recent = []
            for step in range(total):
                tr.train_step()
                if (step + 1) % DRAIN_EVERY == 0 or step + 1 == total:
                    rows = tr.drain_log(wait=step + 1 == total)
                    if log is not None and rows:
                        log.steps(rows)
                        recent = rows
                        print(progress(recent, total, args.batch_size), flush=True)
            tr.check_exchange()
            torch.cuda.synchronize(dev)
            t_train = time.perf_counter() - t0
            tr.gather_master_params()
            step = total
            if rank == 0:
                os.makedirs(ckpt_dir, exist_ok=True)
                ck = checkpoint(model, train.directions, train.poses, args.num_epochs - 1, total)
                torch.save(ck, os.path.join(ckpt_dir, "epoch=%d.ckpt" % (args.num_epochs - 1)))
                torch.save(slim_state_dict(ck), os.path.join(ckpt_dir, "epoch=%d_slim.ckpt" % (args.num_epochs - 1)))
        t0 = time.perf_counter()
        res = metrics.evaluate(model, test.poses, test.directions, test.rgb, test.img_wh, world_size=world, rank=rank,
                               process_group=pg, exp_step_factor=settings["exp_step_factor"], lpips_net=lpips_net,
                               save_dir=save_dir, video_fps=args.video_fps)
        t_val = time.perf_counter() - t0
        if log is not None:
            log.metric("test/psnr", res["psnr"], step)
            log.metric("test/ssim", res["ssim"], step)
            if "lpips" in res:
                log.metric("test/lpips_vgg", res["lpips"], step)
            print("test/psnr %.4f  test/ssim %.4f%s" % (res["psnr"], res["ssim"],
                  "  test/lpips_vgg %.4f" % res["lpips"] if "lpips" in res else ""))
            print("time: training %.2f s (%d steps), validation %.2f s (%d views)" % (t_train, total if not args.val_only else 0,
                                                                                     t_val, len(test.poses)), flush=True)
    finally:
        if log is not None:
            log.close()
        if world > 1:
            import torch.distributed as dist
            dist.destroy_process_group()
    return res


def main(argv=None):
    args = parse_args(argv)
    run(args)
    return 0


if __name__ == "__main__":
    sys.exit(main())
