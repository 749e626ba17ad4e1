"""Remove floaters from a trained checkpoint's occupancy grid and write the cleaned checkpoint.

    python -m ngp_pl_b200.clean_occupancy --ckpt_path ckpts/nerf/lego/epoch=29.ckpt --out lego_clean.ckpt
        [--keep_largest K] [--min_cells N] [--scale 0.5]

The checkpoint (the full or the slim one train.py writes) is loaded into NGP(scale) with export_mesh.load_model, and
components.remove_floaters clears the occupancy of every connected piece of the grid that is not among the K largest
or has fewer than N cells. --out is written in --ckpt_path's own layout with only model.density_bitfield changed, and
model.density_grid where the file has one (its cleared cells set to -1, so a later update_density_grid keeps them
empty). show_gui, export_mesh, export_points and train --val_only take it as they take the input.
Bad arguments are refused with exit status 2 before torch is imported.
"""
import argparse
import math
import os
import sys


def get_parser():
    p = argparse.ArgumentParser(prog="python -m ngp_pl_b200.clean_occupancy",
                                description="Remove floaters from a checkpoint's occupancy grid.")
    p.add_argument("--ckpt_path", type=str, required=True, help="full or slim checkpoint of train.py")
    p.add_argument("--out", type=str, required=True, help="path of the cleaned checkpoint")
    p.add_argument("--keep_largest", type=int, default=None, metavar="K",
                   help="keep only the K largest connected pieces of the occupancy grid, >= 1")
    p.add_argument("--min_cells", type=int, default=None, metavar="N",
                   help="clear the connected pieces with fewer than N occupied cells, >= 1")
    p.add_argument("--scale", type=float, default=0.5, help="scene scale the model was trained with")
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
    if args.keep_largest is None and args.min_cells is None:
        parser.error("give --keep_largest, --min_cells, or both")
    if args.keep_largest is not None and args.keep_largest < 1:
        parser.error("--keep_largest must be >= 1")
    if args.min_cells is not None and args.min_cells < 1:
        parser.error("--min_cells must be >= 1")
    if os.path.realpath(args.out) == os.path.realpath(args.ckpt_path):
        parser.error("--out must not be --ckpt_path: the input stays as it is")
    d = os.path.dirname(os.path.abspath(args.out))
    if not os.path.isdir(d) or not os.access(d, os.W_OK):
        parser.error("--out %s: directory %s is not writable" % (args.out, d))
    return args


def parse_args(argv=None):
    parser = get_parser()
    return check_args(parser.parse_args(argv), parser)


def main(argv=None):
    args = parse_args(argv)
    import torch
    from . import components
    from .export_mesh import load_model
    model = load_model(args.ckpt_path, args.scale)
    ck = torch.load(args.ckpt_path, map_location="cpu", weights_only=True)
    sd = ck["state_dict"] if "state_dict" in ck else ck
    _, stats = components.remove_floaters(model, args.keep_largest, args.min_cells, return_stats=True)
    sd["model.density_bitfield"] = model.density_bitfield.detach().cpu()
    if "model.density_grid" in sd:
        sd["model.density_grid"] = model.density_grid.detach().cpu()
    torch.save(ck, args.out)
    print("ngp_pl_b200.clean_occupancy: %s: kept %d of %d pieces; cleared %d shell cells and %d inner cells"
          % (args.out, stats["kept"], stats["components"], stats["cleared_cells"], stats["cleared_inner"]), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
