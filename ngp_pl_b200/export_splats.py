"""Export a trained checkpoint as 3D Gaussians: the 3DGS point_cloud.ply layout, for splat viewers and as the start of
a 3DGS optimisation.

    python -m ngp_pl_b200.export_splats --ckpt_path ckpts/nsvf/Lego/epoch=29.ckpt [--scale 0.5]
        [--root_dir R --dataset_name nerf|colmap [--downsample 1.0]] [--num_rays 1000000] [--min_opacity 0.5]
        [--bounds x0 y0 z0 x1 y1 z1] [--voxel G] [--nb_neighbors 20] [--std_ratio 2.0] [--keep_outliers]
        [--no_normals] [--sh_degree 3] [--directions 128] [--shape disc|sphere] [--flatness 0.1] [--ridge 1e-3]
        [--out splats.ply] [--preview DIR]

The cameras and the point flags are export_points' (same names and defaults): the points are the point cloud
export_points would write. Each point becomes one Gaussian (splats.extract_splats): SH colours of degree --sh_degree
fitted to the model's colour over --directions Fibonacci directions (weighted to the hemisphere its normal faces,
unless --no_normals), with a ridge of --ridge; a disc of tangent scale s = sqrt(mean squared distance to its 3 nearest
neighbours) and normal scale --flatness s facing the normal (--shape disc), or a sphere of scale s; opacity from the
model's density over 2 s. Positions are in the model's frame. --preview DIR (needs --root_dir, for the intrinsics)
renders every camera view through the splat rasteriser, writes `{i:03d}.png` and the model's own render
`{i:03d}_model.png` there, and prints per-view and mean PSNR of the splats against the model.
Bad arguments are refused with exit status 2 before torch is imported.
"""
import math
import sys
import time

from . import export_points


def get_parser():
    p = export_points.get_parser()
    p.prog = "python -m ngp_pl_b200.export_splats"
    p.description = "Write the 3D Gaussians of a trained Instant-NGP checkpoint as a 3DGS point_cloud.ply."
    p.add_argument("--sh_degree", type=int, default=3, help="degree of the fitted SH colours, 0..3")
    p.add_argument("--directions", type=int, default=128, help="directions the colour is fitted over, 16..1024")
    p.add_argument("--shape", type=str, default="disc", choices=["disc", "sphere"])
    p.add_argument("--flatness", type=float, default=0.1, help="normal-axis scale of a disc over its tangent scale")
    p.add_argument("--ridge", type=float, default=1e-3, help="ridge of the SH fit, >= 0")
    p.add_argument("--preview", type=str, default=None, metavar="DIR",
                   help="render the camera views through the splat rasteriser into DIR and print PSNR (needs --root_dir)")
    p.set_defaults(out="splats.ply")
    return p


def check_args(args, parser):
    """export_points' refusals, then this command's own; parser.error() (exit status 2) names the flag"""
    export_points.check_args(args, parser)
    if not 0 <= args.sh_degree <= 3:
        parser.error("--sh_degree must be in 0..3")
    if not 16 <= args.directions <= 1024:
        parser.error("--directions must be in 16..1024")
    if not (args.flatness > 0 and math.isfinite(args.flatness)):
        parser.error("--flatness must be positive and finite")
    if not (args.ridge >= 0 and math.isfinite(args.ridge)):
        parser.error("--ridge must be >= 0 and finite")
    if args.preview is not None and args.root_dir is None:
        parser.error("--preview needs --root_dir: the intrinsics and image size come from the scene")
    return args


def parse_args(argv=None):
    parser = get_parser()
    return check_args(parser.parse_args(argv), parser)


def main(argv=None):
    args = parse_args(argv)
    import torch
    from . import splats
    from .export_mesh import load_model
    poses, directions = export_points.cameras(args)
    model = load_model(args.ckpt_path, args.scale)
    bounds = None if args.bounds is None else (args.bounds[:3], args.bounds[3:])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    timings = {}
    sp = splats.extract_splats(model, poses, directions, args.num_rays, args.min_opacity, bounds, args.voxel,
                               args.nb_neighbors, args.std_ratio, args.keep_outliers, not args.no_normals,
                               args.sh_degree, args.directions, args.shape, args.flatness, args.ridge, timings=timings)
    splats.write_splats(args.out, sp)
    t1 = time.perf_counter()
    print("ngp_pl_b200.export_splats: %s: %d splats (SH degree %d, %s); %.3f s (%s)" % (
        args.out, sp.shape[0], args.sh_degree, args.shape, t1 - t0,
        ", ".join("%s %.1f ms" % kv for kv in timings.items())), flush=True)
    if args.preview is not None:
        from . import datasets
        meta = datasets.scene_meta(args.dataset_name, args.root_dir, "train", args.downsample)
        psnr = splats.preview(model, sp, meta.poses, meta.K, meta.img_wh, meta.directions, save_dir=args.preview)
        for i, v in enumerate(psnr):
            print("ngp_pl_b200.export_splats: preview view %d: PSNR %.2f dB" % (i, v), flush=True)
        print("ngp_pl_b200.export_splats: preview: mean PSNR %.2f dB over %d views (%s)" % (
            sum(psnr) / max(len(psnr), 1), len(psnr), args.preview), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
