"""ctypes binding of libngp_b200.so (the C-ABI declared in include/ngp_b200.h).

There is NO fallback: if the library is missing or a symbol is absent this module raises, and every
operator built on it raises with it. (The CPU oracle under /oracle is test infrastructure and is never
imported from here.)
"""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libngp_b200.so")
ABI_VERSION = 15  #NGP_ABI_VERSION in include/ngp_b200.h

NGP_MAX_LEVELS = 16
NGP_DENSITY_MLP_PARAMS = 3072
NGP_RGB_MLP_PARAMS = 7168
NGP_MC_SLAB_POINTS = 1 << 20
NGP_MESH_BRICK = 8
NGP_MESH_MAX_N = 8192
NGP_MESH_CHUNK_BRICKS = 1 << 16
NGP_SIMPLIFY_MAX_GRID = 65536
NGP_TEXTURE_MIN_SIZE = 16
NGP_TEXTURE_MAX_SIZE = 16384
NGP_TEXTURE_MIN_SQUARE = 4
NGP_TEXTURE_MARGIN = 1
NGP_TEXTURE_MAX_SAMPLES = 256
NGP_TEXTURE_CHUNK_SAMPLES = 1 << 22
NGP_POINTS_MAX_K = 64
NGP_POINTS_KNN_MAX_CELLS = 1 << 22
NGP_TSDF_GROUP = 64
NGP_SPLAT_FLOATS = 62
NGP_SPLAT_MIN_DIRS = 16
NGP_SPLAT_MAX_DIRS = 1024
NGP_SPLAT_SPHERE = 0
NGP_SPLAT_DISC = 1
NGP_SPLAT_VIEW_FLOATS = 19
NGP_SPLAT_MAX_SIDE = 16384
NGP_SPLAT_PIVOT_RTOL = 1e-10
NGP_VIEW_IMAGES_WORKSPACE = 4096
NGP_PNG_FIXED = 0
NGP_PNG_DYNAMIC = 1
# ngp_render_infer_layout's fields, in the order of NGP_INFER_T_CUR .. NGP_INFER_COUNTERS
NGP_INFER_FIELDS = ("t_cur", "t_end", "alive0", "alive1", "ray_start", "ray_n", "ray_idx", "ts", "deltas", "sigmas",
                    "rgbs", "counters")
NGP_INFER_STATE_OFFSET = 32
NGP_INFER_TOTAL_OFFSET = 64


class NgpGridMeta(C.Structure):
    _fields_ = [
        ("n_levels", C.c_int32),
        ("hashed_mask", C.c_uint32),
        ("offset", C.c_uint32 * (NGP_MAX_LEVELS + 1)),
        ("res", C.c_uint32 * NGP_MAX_LEVELS),
        ("scale", C.c_float * NGP_MAX_LEVELS),
    ]


class NgpNet(C.Structure):
    _fields_ = [
        ("enc_params_h", C.c_void_p),
        ("rgb_params_h", C.c_void_p),
        ("meta", NgpGridMeta),
        ("xyz_min", C.c_float * 3),
        ("xyz_max", C.c_float * 3),
        ("rgb_act", C.c_int32),
    ]


class NgpSamples(C.Structure):
    _fields_ = [
        ("xyzs", C.c_void_p),
        ("dirs", C.c_void_p),
        ("rays_o", C.c_void_p),
        ("rays_d", C.c_void_p),
        ("ray_idx", C.c_void_p),
        ("ts", C.c_void_p),
        ("n", C.c_int64),
        ("n_dev", C.c_void_p),
        ("live_idx", C.c_void_p),
        ("n_live_dev", C.c_void_p),
    ]


class NgpLattice(C.Structure):
    """Mirror of NgpLattice in include/ngp_b200.h."""
    _fields_ = [
        ("n", C.c_int32 * 3),
        ("lo", C.c_float * 3),
        ("step", C.c_float * 3),
    ]


class NgpClusterGrid(C.Structure):
    """Mirror of NgpClusterGrid in include/ngp_b200.h."""
    _fields_ = [
        ("lo", C.c_float * 3),
        ("h", C.c_float),
        ("n", C.c_int32 * 3),
    ]


class NgpTrainCfg(C.Structure):
    """Mirror of NgpTrainCfg in include/ngp_b200.h."""
    _fields_ = [
        ("n_rays", C.c_int32),
        ("cascades", C.c_int32),
        ("grid_size", C.c_int32),
        ("max_samples", C.c_int32),
        ("scale", C.c_float),
        ("exp_step_factor", C.c_float),
        ("T_threshold", C.c_float),
        ("near_distance", C.c_float),
        ("center", C.c_float * 3),
        ("half_size", C.c_float * 3),
        ("bg", C.c_float * 3),
        ("lambda_opacity", C.c_float),
        ("max_total_samples", C.c_int64),
    ]


class NgpInferCfg(C.Structure):
    """Mirror of NgpInferCfg in include/ngp_b200.h."""
    _fields_ = [
        ("n_rays", C.c_int32),
        ("cascades", C.c_int32),
        ("grid_size", C.c_int32),
        ("max_samples", C.c_int32),
        ("scale", C.c_float),
        ("exp_step_factor", C.c_float),
        ("T_threshold", C.c_float),
        ("near_distance", C.c_float),
        ("center", C.c_float * 3),
        ("half_size", C.c_float * 3),
        ("bg", C.c_float * 3),
        ("sample_budget", C.c_int32),
        ("max_round_samples", C.c_int64),
    ]


class NgpViewCfg(C.Structure):
    """Mirror of NgpViewCfg in include/ngp_b200.h."""
    _fields_ = [
        ("mode", C.c_int32),
        ("quality", C.c_int32),
        ("H", C.c_int32),
        ("W", C.c_int32),
    ]


class NgpTrainBuffers(C.Structure):
    """Mirror of NgpTrainBuffers in include/ngp_b200.h."""
    _fields_ = [(n, C.c_void_p) for n in (
        "rays_o", "rays_d", "noise", "density_bitfield",
        "stage_t", "stage_dt", "n_samples", "offsets", "counters", "rgb", "opacity", "depth",
        "ray_idx", "ts", "deltas", "sigmas", "rgbs", "ws", "dsigmas", "drgbs", "live_idx", "feat_save", "scalars",
        "scan_temp")] + [("scan_temp_bytes", C.c_size_t), ("bwd_workspace", C.c_void_p), ("bwd_workspace_bytes", C.c_size_t),
                                  ("bg_dev", C.c_void_p)]


_P = C.c_void_p
_i = C.c_int
_i64 = C.c_int64
_f = C.c_float
_sz = C.c_size_t

# name -> (restype, argtypes). Every symbol include/ngp_b200.h declares must be listed here;
# tests/test_abi.py checks header <-> table <-> library agreement.
SIGNATURES = {
    "ngp_abi_version": (_i, []),
    "ngp_launch_count": (C.c_ulonglong, []),
    "ngp_trace_set": (_i, [_P]),
    "ngp_ray_aabb_intersect": (_i, [_P, _P, _P, _P, _i, _i, _i, _P, _P, _P, _P]),
    "ngp_ray_sphere_intersect": (_i, [_P, _P, _P, _P, _i, _i, _i, _P, _P, _P, _P]),
    "ngp_packbits": (_i, [_P, _i, _i64, _f, _P, _P, _P]),
    "ngp_morton3D": (_i, [_P, _i, _P, _P]),
    "ngp_morton3D_invert": (_i, [_P, _i, _P, _P]),
    "ngp_raymarching_train_workspace": (_sz, [_i]),
    "ngp_raymarching_train_workspace2": (_sz, [_i, _i]),
    "ngp_raymarching_train": (_i, [_P, _P, _P, _P, _i, _f, _f, _P, _i, _i, _i, _P, _P, _P, _P, _P, _P, _P, _sz, _P]),
    "ngp_raymarching_test": (_i, [_P, _P, _P, _P, _P, _i, _f, _f, _i, _i, _i, _i, _P, _P, _P, _P, _P, _P]),
    "ngp_composite_train_fw": (_i, [_P, _P, _P, _P, _P, _f, _i, _i64, _P, _P, _P, _P, _P, _P]),
    "ngp_composite_train_bw": (_i, [_P] * 13 + [_f, _i, _i64, _P, _P, _P]),
    "ngp_composite_test_fw": (_i, [_P, _P, _P, _P, _P, _P, _f, _P, _i, _i, _P, _P, _P, _P]),
    "ngp_distortion_loss_fw": (_i, [_P, _P, _P, _P, _i, _i64, _P, _P, _P, _P]),
    "ngp_distortion_loss_bw": (_i, [_P, _P, _P, _P, _P, _P, _P, _i, _i64, _P, _P]),
    "ngp_grid_meta": (C.c_uint32, [_i, _i, _i, _f, C.POINTER(NgpGridMeta)]),
    "ngp_cast_params": (_i, [_P, _P, _i64, _P]),
    "ngp_net_forward": (_i, [C.POINTER(NgpNet), C.POINTER(NgpSamples), _i, _P, _P, _P, _P, _P]),
    "ngp_net_backward_workspace": (_sz, [_i64]),
    "ngp_net_backward": (_i, [C.POINTER(NgpNet), C.POINTER(NgpSamples), _P, _P, _P, _P, _P, _P, _P, _sz, _P]),
    "ngp_net_backward_mlp": (_i, [C.POINTER(NgpNet), C.POINTER(NgpSamples), _P, _P, _P, _P, _P, _P, _P, _sz, _P]),
    "ngp_net_backward_scatter": (_i, [C.POINTER(NgpNet), C.POINTER(NgpSamples), _P, _P, _P, _sz, _P]),
    "ngp_sh_encode": (_i, [_P, _i64, _P, _P]),
    "ngp_mlp_rgb_forward": (_i, [_P, _P, _i64, _i, _P, _P]),
    "ngp_mlp_rgb_backward": (_i, [_P, _P, _P, _i64, _i, _P, _P, _P, _P]),
    "ngp_enc_backward": (_i, [C.POINTER(NgpNet), C.POINTER(NgpSamples), _P, _P, _P, _P, _P, _sz, _P]),
    "ngp_grad_scale": (_i, [_P, _P, _P, _i64, _P, _P, _P]),
    "ngp_train_scan_temp_bytes": (_sz, [_i]),
    "ngp_render_train_fwd": (_i, [C.POINTER(NgpNet), C.POINTER(NgpTrainCfg), C.POINTER(NgpTrainBuffers), _P]),
    "ngp_render_train_march": (_i, [C.POINTER(NgpTrainCfg), C.POINTER(NgpTrainBuffers), _P]),
    "ngp_render_train_net": (_i, [C.POINTER(NgpNet), C.POINTER(NgpTrainCfg), C.POINTER(NgpTrainBuffers), _P]),
    "ngp_render_train_step": (_i, [C.POINTER(NgpNet), C.POINTER(NgpTrainCfg), C.POINTER(NgpTrainBuffers), _P, _P, _P, _P]),
    "ngp_render_train_bwd": (_i, [C.POINTER(NgpNet), C.POINTER(NgpTrainCfg), C.POINTER(NgpTrainBuffers),
                                  _P, _P, _P, _P, _P, _P, _P]),
    "ngp_nerf_loss_grad": (_i, [C.POINTER(NgpTrainCfg), C.POINTER(NgpTrainBuffers), _P, _P, _P, _P]),
    "ngp_adam_step": (_i, [_P, _P, _P, _P, _P, _i64, _P, _P, _f, _f, _f, _f, _i, _P]),
    "ngp_adam_step_p2p": (_i, [_i, _i, _P, _P, _P, _P, _P, _i64, _P, _P, _f, _f, _f, _i, _P]),
    "ngp_adam_step_fused": (_i, [_i, _i, _P, _P, _P, C.c_uint64, C.c_uint64, _P, _P, _P, _i64, _P, _P, _P, _P, _f, _f, _f, _i, _P]),
    "ngp_train_log_step": (_i, [_P, _P, _P, _P, _P, _i64, _P, _i, _P]),
    "ngp_gen_rays": (_i, [_P, _P, _P, _P, _P, _i64, _i, _P, _P, _P, _P]),
    "ngp_sample_rays": (_i, [_P, _P, _P, _i, _i64, _i, C.c_uint32, C.c_uint32, _P, _P, _P, _P, _P, _P]),
    "ngp_sample_rays_ex": (_i, [_P, _P, _P, _i, _i, _i, _i64, _i, C.c_uint32, C.c_uint32, _P, _P, _P, _P, _P, _P]),
    "ngp_stage_image": (_i, [_P, _i, _i, _i, _i, _i, _i, _P, _P]),
    "ngp_render_infer_workspace": (_sz, [_i, _i64]),
    "ngp_render_infer_layout": (_sz, [_i, _i64, _P]),
    "ngp_render_infer": (_i, [C.POINTER(NgpNet), C.POINTER(NgpInferCfg), _P, _P, _P, _P, _P, _P, _P, _i, _i, _i, _P,
                              _P, _sz, _P]),
    "ngp_render_infer_frame": (_i, [C.POINTER(NgpNet), C.POINTER(NgpInferCfg), _P, _P, _P, _P, _P, _P, _P, _P, _sz, _P]),
    "ngp_render_view_workspace": (_sz, [C.POINTER(NgpInferCfg), C.POINTER(NgpViewCfg)]),
    "ngp_render_view_frame": (_i, [C.POINTER(NgpNet), C.POINTER(NgpInferCfg), C.POINTER(NgpViewCfg)] + [_P] * 9 +
                              [_sz, _P, _P, _sz, _P]),
    "ngp_update_grid_workspace": (_sz, [_i, _i]),
    "ngp_update_density_grid": (_i, [C.POINTER(NgpNet), _P, _P, _P, _i, _i, _f, _f, _i, _f, C.c_uint32, _P, _sz, _P]),
    "ngp_update_density_grid_pick": (_i, [_P, _i, _i, _f, _f, _i, C.c_uint32, _P, _sz, _P]),
    "ngp_update_density_grid_eval": (_i, [C.POINTER(NgpNet), _P, _P, _P, _i, _i, _f, _i, _f, _P, _sz, _P]),
    "ngp_image_metrics_workspace": (_sz, [_i, _i]),
    "ngp_image_metrics": (_i, [_P, _P, _i, _i, _i, _f, _P, _P, _P, _sz, _P]),
    "ngp_lpips_weights_bytes": (_sz, []),
    "ngp_lpips_workspace": (_sz, [_i, _i]),
    "ngp_lpips": (_i, [_P, _P, _P, _i, _i, _i, _P, _P, _sz, _P]),
    "ngp_density_lattice": (_i, [C.POINTER(NgpNet), C.POINTER(NgpLattice), _P, _P]),
    "ngp_marching_cubes_workspace": (_sz, [C.POINTER(NgpLattice)]),
    "ngp_marching_cubes_count": (_i, [_P, C.POINTER(NgpLattice), _f, _P, _P, _sz, _P]),
    "ngp_marching_cubes_emit": (_i, [_P, C.POINTER(NgpLattice), _f, _P, _P, _P, _i64, _i64, _P, _sz, _P]),
    "ngp_mesh_bricks_bytes": (_sz, [C.POINTER(NgpLattice)]),
    "ngp_mesh_brick_mask": (_i, [_P, _i, _i, _f, C.POINTER(NgpLattice), _P, _P]),
    "ngp_density_bricks": (_i, [C.POINTER(NgpNet), C.POINTER(NgpLattice), _P, _i64, _i, _P, _P, _P]),
    "ngp_mesh_sparse_workspace": (_sz, [C.POINTER(NgpLattice)]),
    "ngp_mesh_sparse_bricks": (_i, [C.POINTER(NgpNet), C.POINTER(NgpLattice), _f, _P, _P, _P, _sz, _P]),
    "ngp_mesh_surface_workspace": (_sz, [C.POINTER(NgpLattice), _i64]),
    "ngp_mesh_sparse_count": (_i, [C.POINTER(NgpNet), C.POINTER(NgpLattice), _f, _P, _i64, _P, _P, _sz, _P, _sz, _P]),
    "ngp_mesh_sparse_emit": (_i, [C.POINTER(NgpLattice), _f, _i64, _P, _P, _P, _i64, _i64, _P, _sz, _P]),
    "ngp_mesh_simplify_workspace": (_sz, [_i64, _i64]),
    "ngp_mesh_simplify_count": (_i, [_P, _i64, _P, _i64, C.POINTER(NgpClusterGrid), _P, _P, _sz, _P]),
    "ngp_mesh_simplify_emit": (_i, [_P, _i64, _i64, _P, _P, _P, _P, _P, _P, _i64, _i64, _P, _sz, _P]),
    "ngp_mesh_texture_workspace": (_sz, [_i64, _i64, _i]),
    "ngp_mesh_texture_atlas": (_i, [_P, _i64, _P, _i64, _i, _P, _P, _P, _P, _sz, _P]),
    "ngp_mesh_texture_texels": (_i, [_P, _P, _i64, _P, _i64, _i, _P, _i64, _P, _P, _P, _P, _P, _sz, _P]),
    "ngp_mesh_texture_bake_workspace": (_sz, [_i]),
    "ngp_mesh_texture_bake": (_i, [C.POINTER(NgpNet), _i, _i64, _P, _P, _P, _f, _i, _P, _P, _sz, _P]),
    "ngp_points_workspace": (_sz, [_i64]),
    "ngp_points_rays": (_i, [_i64, _i64, _i64, _i64, _i, _P, _P, _P, _P, _P, _P, _P]),
    "ngp_points_backproject": (_i, [_P, _P, _P, _P, _P, _i64, _f, _P, _P, _P, _P, _P, _P, _sz, _P]),
    "ngp_points_voxel": (_i, [_P, _P, _P, _i64, C.POINTER(NgpClusterGrid), _P, _P, _P, _P, _P, _P, _P, _sz, _P]),
    "ngp_points_knn": (_i, [_P, _i64, _i, _P, _P, _P, _sz, _P]),
    "ngp_points_outliers": (_i, [_P, _P, _P, _i64, _i, _P, C.c_double, _P, _P, _P, _P, _P, _P, _P, _sz, _P]),
    "ngp_points_normals": (_i, [_P, _P, _i64, _i, _P, _P, _P]),
    "ngp_tsdf_integrate": (_i, [C.POINTER(NgpLattice), _f, _i, _P, _P, _i, _i, _P, _P, _P, _P, _f, _P, _P, _P, _P, _P]),
    "ngp_tsdf_mc_workspace": (_sz, [C.POINTER(NgpLattice)]),
    "ngp_tsdf_mc_count": (_i, [_P, _P, C.POINTER(NgpLattice), _P, _P, _sz, _P]),
    "ngp_tsdf_mc_emit": (_i, [_P, _P, _P, _P, C.POINTER(NgpLattice), _P, _P, _P, _P, _i64, _i64, _P, _sz, _P]),
    "ngp_splat_colors": (_i, [C.POINTER(NgpNet), _P, _i64, _P, _i, _P, _P, _P, _P]),
    "ngp_splat_fit": (_i, [_P, _i64, _i, _P, _P, _P, _i, C.c_double, _P, _P]),
    "ngp_splat_geometry": (_i, [_P, _P, _P, _P, _i, _i64, _i, _f, _P, _P]),
    "ngp_splat_render_workspace": (_sz, [_i64, _i, _i, _i64]),
    "ngp_splat_render": (_i, [_P, _i64, _P, _i, _i, _i64, _P, _P, _P, _P, _sz, _P]),
    "ngp_grid_components": (_i, [_P, _i, _i, _f, _P, _P, _P]),
    "ngp_grid_components_clean": (_i, [_P, _P, _i, _i, _f, _P, _P, _P, _P, _P]),
    "ngp_components_select_workspace": (_sz, [_i64]),
    "ngp_components_select": (_i, [_P, _P, _i64, _i64, _i64, _P, _P, _P, _sz, _P]),
    "ngp_mesh_components_workspace": (_sz, [_i64, _i64]),
    "ngp_mesh_components": (_i, [_P, _i64, _i64, _P, _P, _P, _sz, _P]),
    "ngp_mesh_filter_workspace": (_sz, [_i64, _i64]),
    "ngp_mesh_filter_count": (_i, [_P, _i64, _i64, _P, _P, _P, _P, _sz, _P]),
    "ngp_mesh_filter_emit": (_i, [_P, _P, _P, _P, _i64, _i64, _P, _P, _P, _P, _i64, _i64, _P, _sz, _P]),
    "ngp_view_images": (_i, [_P, _P, _i, _i, _P, _P, _P, _sz, _P]),
    "ngp_png_workspace": (_sz, [_i, _i]),
    "ngp_png_capacity": (_sz, [_i, _i]),
    "ngp_png_encode": (_i, [_P, _i, _i, _P, _sz, _P, _P, _sz, _P]),
    "ngp_png_workspace_mode": (_sz, [_i, _i, _i]),
    "ngp_png_encode_mode": (_i, [_P, _i, _i, _i, _P, _sz, _P, _P, _sz, _P]),
    "ngp_jpeg_workspace": (_sz, [_i, _i]),
    "ngp_jpeg_capacity": (_sz, [_i, _i]),
    "ngp_jpeg_encode": (_i, [_P, _i, _i, _i, _P, _sz, _P, _P, _sz, _P]),
}

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                "ngp_pl_b200: %s is missing. Build it with `python -m ngp_pl_b200.build` (needs nvcc). "
                "There is no CPU or PyTorch fallback for this path." % LIB_PATH)
        h = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(h, name)  # AttributeError if the symbol is not exported
            fn.restype = res
            fn.argtypes = args
        if h.ngp_abi_version() != ABI_VERSION:
            raise RuntimeError("ngp_pl_b200: ABI version mismatch, rebuild libngp_b200.so")
        _lib = h
    return _lib


def check(rc, what):
    if rc != 0:
        raise RuntimeError("ngp_pl_b200.%s failed with code %d%s" % (
            what, rc, " (invalid argument)" if rc == -22 else " (cudaError_t)"))


def infer_layout(n_rays, max_round_samples):
    """byte offsets of the wavefront's workspace arrays, {field: offset}, and the workspace size"""
    off = (C.c_int64 * len(NGP_INFER_FIELDS))()
    size = lib().ngp_render_infer_layout(int(n_rays), int(max_round_samples), off)
    if size == 0:
        raise ValueError("ngp_render_infer_layout: n_rays and max_round_samples must be >= 1")
    return dict(zip(NGP_INFER_FIELDS, off)), int(size)


def grid_meta(n_levels, log2_hashmap_size, base_resolution, per_level_scale):
    m = NgpGridMeta()
    total = lib().ngp_grid_meta(int(n_levels), int(log2_hashmap_size), int(base_resolution),
                                float(per_level_scale), C.byref(m))
    if total == 0:
        raise RuntimeError("ngp_grid_meta: unsupported grid configuration")
    return m, int(total)
