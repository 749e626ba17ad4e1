"""Export the mesh of a trained checkpoint as a binary PLY, or as a textured OBJ.

    python -m ngp_pl_b200.export_mesh --ckpt_path ckpts/nsvf/Lego/epoch=29.ckpt [--scale 0.5] [--resolution 1024]
        [--threshold 20] [--bounds x0 y0 z0 x1 y1 z1] [--colors] [--no_normals] [--dense]
        [--keep_largest K] [--min_triangles N] [--simplify G]
        [--texture W [--texture_offset R] [--texture_samples K]] [--out mesh.ply]
        [--tsdf --root_dir R [--dataset_name nerf|colmap] [--downsample 1.0] [--min_opacity 0.5] [--tsdf_trunc T]]

The checkpoint is the full or the slim one train.py writes; it is loaded into NGP(scale) with train.load_weights. By
default the mesh is mesh.extract_mesh_sparse's: σ evaluated and marching cubes run only near the cells the model's
occupancy grid marks, so 2048^3 and 4096^3 lattices fit in memory. --dense gives mesh.extract_mesh's mesh of the whole
lattice (the notebook's mesh cell): a different mesh, which also has the surfaces the occupancy grid has culled.
--keep_largest K / --min_triangles N drop the pieces of the mesh (triangles sharing vertices) that are not among the K
largest or have fewer than N triangles, with mesh.remove_small_components: floaters and the shells of closed cavities.
--simplify G then reduces the mesh with mesh.simplify_mesh on a G^3 cluster grid over the lattice box (vertex
clustering with quadric-error placement; colours become the means of each cluster's colours).
--texture W bakes the model's colours into a W x W atlas with mesh.bake_texture and writes --out (which must end in
.obj) with mesh.write_obj, next to its .mtl and .png. The bake renders --texture_samples samples along each texel's
inward normal from --texture_offset outside the surface: by default the cluster cell with --simplify, where vertices
sit up to sqrt(3) cells off the surface they stand for, and the largest lattice step without it.
--tsdf gives fusion.extract_mesh_tsdf's mesh instead: every pixel of the training views of --root_dir (cameras from
datasets.scene_meta(--dataset_name, --root_dir, 'train', --downsample), metadata only, no image decoded) rendered with a
black background, the depth of the pixels of opacity >= --min_opacity fused into a truncated signed distance field on
the --resolution lattice over --bounds (truncation --tsdf_trunc, default 4 lattice steps), and its masked marching
cubes: only surfaces the cameras saw, no σ threshold. --colors then writes the fused colours. The state takes 24 B per
lattice point, so --tsdf takes --resolution up to 1024.
Bad arguments are refused with exit status 2 before torch is imported.
"""
import argparse
import math
import sys
import time


def get_parser():
    p = argparse.ArgumentParser(prog="python -m ngp_pl_b200.export_mesh",
                                description="Write the mesh of a trained Instant-NGP checkpoint as a binary PLY.")
    p.add_argument("--ckpt_path", type=str, required=True, help="full or slim checkpoint of train.py")
    p.add_argument("--scale", type=float, default=0.5, help="scene scale the model was trained with")
    p.add_argument("--resolution", type=int, default=1024, help="lattice points per axis, 2..8192")
    p.add_argument("--threshold", type=float, default=20.0, help="σ level of the surface, > 0")
    p.add_argument("--bounds", type=float, nargs=6, default=None, metavar=("X0", "Y0", "Z0", "X1", "Y1", "Z1"),
                   help="lattice box (default: the model's box [-scale, scale]^3)")
    p.add_argument("--colors", action="store_true", help="vertex colours from the model, seen head-on")
    p.add_argument("--no_normals", action="store_true", help="leave the normals out of the PLY")
    p.add_argument("--dense", action="store_true", help="the unculled mesh of the whole lattice (mesh.extract_mesh)")
    p.add_argument("--keep_largest", type=int, default=None, metavar="K",
                   help="keep only the K largest connected pieces of the mesh (by triangle count), >= 1")
    p.add_argument("--min_triangles", type=int, default=None, metavar="N",
                   help="drop the connected pieces of the mesh with fewer than N triangles, >= 1")
    p.add_argument("--simplify", type=int, default=None, metavar="G",
                   help="simplify on a G^3 cluster grid over the lattice box before writing, 1..65536")
    p.add_argument("--texture", type=int, default=None, metavar="W",
                   help="bake a W x W texture atlas (a power of two in 16..16384) and write an OBJ + MTL + PNG")
    p.add_argument("--texture_offset", type=float, default=None, metavar="R",
                   help="start of the bake's rays outside the surface, world units >= 0 (default: the cluster cell "
                        "with --simplify, else the largest lattice step)")
    p.add_argument("--texture_samples", type=int, default=16, metavar="K", help="samples per texel, 1..256")
    p.add_argument("--out", type=str, default="mesh.ply", help="output PLY path (.obj with --texture)")
    p.add_argument("--tsdf", action="store_true",
                   help="fuse the training views' rendered depth into a TSDF and mesh it (fusion.extract_mesh_tsdf)")
    p.add_argument("--root_dir", type=str, default=None, help="with --tsdf: the scene the model was trained on (its cameras)")
    p.add_argument("--dataset_name", type=str, default="nerf", choices=["nerf", "colmap"])
    p.add_argument("--downsample", type=float, default=1.0, help="image downsample of the cameras, in (0, 1]")
    p.add_argument("--min_opacity", type=float, default=0.5, help="with --tsdf: opacity a pixel needs to count, in (0, 1]")
    p.add_argument("--tsdf_trunc", type=float, default=None, metavar="T",
                   help="with --tsdf: truncation distance in world units, > 0 (default: 4 lattice steps)")
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
    if not 2 <= args.resolution <= 8192:
        parser.error("--resolution must be in 2..8192")
    if not (args.threshold > 0 and math.isfinite(args.threshold)):
        parser.error("--threshold must be positive (the sparse mesh fills culled space with 0)")
    if args.bounds is not None:
        lo, hi = args.bounds[:3], args.bounds[3:]
        if not all(math.isfinite(v) for v in args.bounds) or any(a >= b for a, b in zip(lo, hi)):
            parser.error("--bounds: every lower corner coordinate must be below the upper one")
    if args.keep_largest is not None and args.keep_largest < 1:
        parser.error("--keep_largest must be >= 1")
    if args.min_triangles is not None and args.min_triangles < 1:
        parser.error("--min_triangles must be >= 1")
    if args.simplify is not None and not 1 <= args.simplify <= 65536:
        parser.error("--simplify must be in 1..65536")
    if args.texture is not None:
        if not (16 <= args.texture <= 16384 and args.texture & (args.texture - 1) == 0):
            parser.error("--texture must be a power of two in 16..16384")
        if args.colors:
            parser.error("--texture and --colors exclude each other: the texture carries the colours")
        if not args.out.lower().endswith(".obj"):
            parser.error("--out must end in .obj with --texture")
    if args.texture_offset is not None and not (args.texture_offset >= 0 and math.isfinite(args.texture_offset)):
        parser.error("--texture_offset must be >= 0 and finite")
    if not 1 <= args.texture_samples <= 256:
        parser.error("--texture_samples must be in 1..256")
    if not (0 < args.downsample <= 1):
        parser.error("--downsample must be in (0, 1]")
    if not (0 < args.min_opacity <= 1):
        parser.error("--min_opacity must be in (0, 1]")
    if args.tsdf_trunc is not None and not (args.tsdf_trunc > 0 and math.isfinite(args.tsdf_trunc)):
        parser.error("--tsdf_trunc must be positive and finite")
    if args.tsdf:
        if args.root_dir is None:
            parser.error("--tsdf needs --root_dir: the fusion projects through the cameras' K and image size, which a "
                         "checkpoint does not store")
        if args.dense:
            parser.error("--tsdf and --dense exclude each other")
        if args.resolution > 1024:
            parser.error("--resolution must be at most 1024 with --tsdf (24 B of state per lattice point)")
    return args


def parse_args(argv=None):
    parser = get_parser()
    return check_args(parser.parse_args(argv), parser)


def load_model(ckpt_path, scale):
    """NGP(scale) on the current CUDA device with the checkpoint's weights, density_grid and grid_coords registered
    as train.run registers them, so the full and the slim checkpoint both load"""
    import torch
    from . import train
    from .models.networks import NGP
    if not torch.cuda.is_available():
        raise SystemExit("ngp_pl_b200.export_mesh: no CUDA device (there is no CPU path)")
    dev = torch.device("cuda", torch.cuda.current_device())
    model = NGP(scale=scale).to(dev)
    G = model.grid_size
    model.register_buffer("density_grid", torch.zeros(model.cascades, G ** 3, device=dev))
    model.register_buffer("grid_coords", torch.stack(torch.meshgrid(
        *[torch.arange(G, dtype=torch.int32, device=dev)] * 3, indexing="ij"), -1).reshape(-1, 3))
    try:
        train.load_weights(model, ckpt_path)
    except RuntimeError as e:
        raise SystemExit("ngp_pl_b200.export_mesh: %s does not fit NGP(scale=%g) (%d cascades of %d^3 cells): %s"
                         % (ckpt_path, scale, model.cascades, G, str(e).splitlines()[0]))
    return model


def texture_offset(box, resolution, simplify):
    """the default --texture_offset: the cluster cell side with --simplify, else the largest lattice step (fp32, as
    mesh.cluster_grid and mesh.lattice compute them)"""
    from . import mesh
    if simplify is not None:
        return float(mesh.cluster_grid(box[0], box[1], simplify).h)
    return float(max(mesh.lattice(resolution, box[0], box[1]).step))


def main(argv=None):
    args = parse_args(argv)
    import torch
    from . import mesh
    model = load_model(args.ckpt_path, args.scale)
    bounds = None if args.bounds is None else (args.bounds[:3], args.bounds[3:])
    normals = not args.no_normals
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    stats = None
    if args.tsdf:
        from . import datasets, fusion
        meta = datasets.scene_meta(args.dataset_name, args.root_dir, "train", args.downsample)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m = fusion.extract_mesh_tsdf(model, torch.as_tensor(meta.poses), meta.K, meta.img_wh, args.resolution, bounds,
                                     args.tsdf_trunc, args.min_opacity, normals=normals, colors=args.colors)
    elif args.dense:
        m = mesh.extract_mesh(model, args.resolution, bounds, args.threshold, normals=normals, colors=args.colors)
    else:
        m, stats = mesh.extract_mesh_sparse(model, args.resolution, bounds, args.threshold, normals=normals,
                                            colors=args.colors, return_stats=True)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    line = "ngp_pl_b200.export_mesh: %s: %d vertices, %d triangles at %d^3 in %.3f s" % (
        args.out, m["vertices"].shape[0], m["triangles"].shape[0], args.resolution, dt)
    if stats is not None:
        line += " (bricks: %d active, %d visited, %d surface)" % (stats["active"], stats["visited"], stats["surface"])
    box = bounds if bounds is not None else (model._xyz_min_host, model._xyz_max_host)
    if args.keep_largest is not None or args.min_triangles is not None:
        t0 = time.perf_counter()
        m, cs = mesh.remove_small_components(m, args.keep_largest, args.min_triangles, return_stats=True)
        torch.cuda.synchronize()
        line += "; kept %d of %d pieces, %d vertices, %d triangles in %.3f s" % (
            cs["kept"], cs["components"], m["vertices"].shape[0], m["triangles"].shape[0], time.perf_counter() - t0)
    if args.simplify is not None:
        t0 = time.perf_counter()
        m = mesh.simplify_mesh(m, args.simplify, box)
        torch.cuda.synchronize()
        line += "; simplified at grid %d to %d vertices, %d triangles in %.3f s" % (
            args.simplify, m["vertices"].shape[0], m["triangles"].shape[0], time.perf_counter() - t0)
    if args.texture is None:
        mesh.write_ply(args.out, **m)
    else:
        r = args.texture_offset
        if r is None:
            r = texture_offset(box, args.resolution, args.simplify)
        t0 = time.perf_counter()
        tex = mesh.bake_texture(model, m, args.texture, r, args.texture_samples, return_texels=True)
        torch.cuda.synchronize()
        S = int(tex["squares"][:, 2].max()) if tex["squares"].shape[0] else args.texture
        line += "; baked a %d^2 atlas (S = %d, %d texels, offset %.6g, %d samples) in %.3f s" % (
            args.texture, S, tex["texel"].shape[0], r, args.texture_samples, time.perf_counter() - t0)
        mesh.write_obj(args.out, m["vertices"], m["triangles"], m["normals"], tex["uv"], tex["texture"])
    print(line, flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
