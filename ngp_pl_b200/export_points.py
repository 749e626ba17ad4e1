"""Export a coloured point cloud with normals of a trained checkpoint as a binary PLY.

    python -m ngp_pl_b200.export_points --ckpt_path ckpts/nsvf/Lego/epoch=29.ckpt [--scale 0.5]
        [--root_dir R --dataset_name nerf|colmap [--downsample 1.0]] [--num_rays 1000000] [--min_opacity 0.5]
        [--bounds x0 y0 z0 x1 y1 z1] [--voxel G] [--nb_neighbors 20] [--std_ratio 2.0] [--keep_outliers]
        [--no_normals] [--out points.ply]

The model loads as export_mesh loads it. The cameras are the training views: from --root_dir through
datasets.scene_meta(..., 'train', downsample), which reads the metadata only and decodes no image, or else from the
`poses` and `directions` a full checkpoint of train.py stores. --num_rays rays through the training pixels (the
points.golden_step permutation, no random draw) are rendered with a black background, and every ray of opacity >=
--min_opacity whose depth lands in --bounds (default: the model's box) becomes a point coloured by the rendered colour
(points.extract_points). Then, in this order: --voxel G keeps one point per cell of a G^3 grid over the box of the
points (points.voxel_downsample); statistical outlier removal over --nb_neighbors neighbours at --std_ratio unless
--keep_outliers (points.remove_outliers); normals from the same number of neighbours, facing the cameras, unless
--no_normals (points.estimate_normals). The file is mesh.write_ply's with no faces.
Bad arguments are refused with exit status 2 before torch is imported.
"""
import argparse
import math
import sys
import time

from .export_mesh import load_model


def get_parser():
    p = argparse.ArgumentParser(prog="python -m ngp_pl_b200.export_points",
                                description="Write a coloured point cloud of a trained Instant-NGP checkpoint as a "
                                            "binary PLY.")
    p.add_argument("--ckpt_path", type=str, required=True, help="full or slim checkpoint of train.py")
    p.add_argument("--scale", type=float, default=0.5, help="scene scale the model was trained with")
    p.add_argument("--root_dir", type=str, default=None, help="the scene the model was trained on (its cameras)")
    p.add_argument("--dataset_name", type=str, default="nerf", choices=["nerf", "colmap"])
    p.add_argument("--downsample", type=float, default=1.0, help="image downsample of the cameras, in (0, 1]")
    p.add_argument("--num_rays", type=int, default=1000000, help="rays through the training pixels, 1..2^28")
    p.add_argument("--min_opacity", type=float, default=0.5, help="opacity a ray needs to become a point, in (0, 1]")
    p.add_argument("--bounds", type=float, nargs=6, default=None, metavar=("X0", "Y0", "Z0", "X1", "Y1", "Z1"),
                   help="box the points must lie in (default: the model's box [-scale, scale]^3)")
    p.add_argument("--voxel", type=int, default=None, metavar="G", help="voxel downsampling on a G^3 grid, 1..65536")
    p.add_argument("--nb_neighbors", type=int, default=20, help="neighbours of outlier removal and normals, 1..64")
    p.add_argument("--std_ratio", type=float, default=2.0, help="outlier removal keeps d <= mean + std_ratio * std")
    p.add_argument("--keep_outliers", action="store_true", help="skip the statistical outlier removal")
    p.add_argument("--no_normals", action="store_true", help="leave the normals out of the PLY")
    p.add_argument("--out", type=str, default="points.ply", help="output PLY path")
    return p


def check_args(args, parser):
    """the refusals, before torch or CUDA: parser.error() (exit status 2) names the flag"""
    try:
        with open(args.ckpt_path, "rb"):
            pass
    except OSError as e:
        parser.error("--ckpt_path %s: cannot be read (%s)" % (args.ckpt_path, e.strerror or e))
    if not (args.scale > 0 and math.isfinite(args.scale)):
        parser.error("--scale must be positive")
    if not (0 < args.downsample <= 1):
        parser.error("--downsample must be in (0, 1]")
    if not 1 <= args.num_rays <= 2 ** 28:
        parser.error("--num_rays must be in 1..2^28")
    if not (0 < args.min_opacity <= 1):
        parser.error("--min_opacity must be in (0, 1]")
    if args.bounds is not None:
        lo, hi = args.bounds[:3], args.bounds[3:]
        if not all(math.isfinite(v) for v in args.bounds) or any(a > b for a, b in zip(lo, hi)):
            parser.error("--bounds: every lower corner coordinate must be at most the upper one")
    if args.voxel is not None and not 1 <= args.voxel <= 65536:
        parser.error("--voxel must be in 1..65536")
    if not 1 <= args.nb_neighbors <= 64:
        parser.error("--nb_neighbors must be in 1..64")
    if not (args.std_ratio >= 0 and math.isfinite(args.std_ratio)):
        parser.error("--std_ratio must be >= 0 and finite")
    return args


def parse_args(argv=None):
    parser = get_parser()
    return check_args(parser.parse_args(argv), parser)


def cameras(args):
    """(poses (n, 3, 4), directions (n_pix, 3)) float32 of the training views: from --root_dir, else the checkpoint"""
    import torch
    if args.root_dir is not None:
        from . import datasets
        meta = datasets.scene_meta(args.dataset_name, args.root_dir, "train", args.downsample)
        return torch.as_tensor(meta.poses), torch.as_tensor(meta.directions)
    ck = torch.load(args.ckpt_path, map_location="cpu", weights_only=True)
    sd = ck.get("state_dict", ck)
    if "poses" not in sd or "directions" not in sd:
        print("ngp_pl_b200.export_points: %s holds no cameras (a slim checkpoint); pass --root_dir with the scene it "
              "was trained on" % args.ckpt_path, file=sys.stderr)
        raise SystemExit(2)
    return sd["poses"], sd["directions"]


def main(argv=None):
    args = parse_args(argv)
    import torch
    from . import mesh, points
    poses, directions = cameras(args)
    model = load_model(args.ckpt_path, args.scale)
    bounds = None if args.bounds is None else (args.bounds[:3], args.bounds[3:])
    times = []

    def stage(name, fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        times.append((name, time.perf_counter() - t0))
        print("ngp_pl_b200.export_points: %s: %d points" % (name, out["points"].shape[0]), flush=True)
        return out

    pts = stage("extract (%d views, %d rays)" % (poses.reshape(-1, 3, 4).shape[0], min(args.num_rays, poses.reshape(
        -1, 3, 4).shape[0] * directions.reshape(-1, 3).shape[0])),
        lambda: points.extract_points(model, poses, directions, args.num_rays, args.min_opacity, bounds))
    if args.voxel is not None:
        pts = stage("voxel %d" % args.voxel, lambda: points.voxel_downsample(pts, args.voxel))
    if not args.keep_outliers:
        pts = stage("outliers (k %d, std_ratio %g)" % (args.nb_neighbors, args.std_ratio),
                    lambda: points.remove_outliers(pts, args.nb_neighbors, args.std_ratio))
    if not args.no_normals:
        pts = stage("normals (k %d)" % args.nb_neighbors, lambda: points.estimate_normals(pts, args.nb_neighbors))
    mesh.write_ply(args.out, pts["points"], torch.empty(0, 3, dtype=torch.int64), pts["normals"], pts["colors"])
    print("ngp_pl_b200.export_points: %s: %d points; %s" % (args.out, pts["points"].shape[0], ", ".join(
        "%s %.3f s" % (n.split(" ")[0], t) for n, t in times)), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
