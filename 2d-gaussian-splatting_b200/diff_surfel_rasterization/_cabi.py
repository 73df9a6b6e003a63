"""ctypes binding of libsurfel_b200.so (C ABI: include/surfel_rasterizer.h).

This is the stub a maintainer of the reference would add in place of upstream's pybind11 `_C`
module (see INTEGRATION.md).  It fails loudly when the CUDA library is missing: there is no CPU or
PyTorch fallback behind this boundary.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SURFEL_LIB") or os.path.join(os.path.dirname(_HERE), "lib", "libsurfel_b200.so")

c_void_p, c_int, c_uint32, c_size_t, c_float = (ctypes.c_void_p, ctypes.c_int, ctypes.c_uint32,
                                                ctypes.c_size_t, ctypes.c_float)


class SurfelSettings(ctypes.Structure):
    """struct surfel_settings (include/surfel_rasterizer.h)."""
    _fields_ = [
        ("image_height", ctypes.c_int32), ("image_width", ctypes.c_int32),
        ("tanfovx", c_float), ("tanfovy", c_float), ("scale_modifier", c_float),
        ("sh_degree", ctypes.c_int32), ("prefiltered", ctypes.c_int32), ("debug", ctypes.c_int32),
        ("tile_row_begin", ctypes.c_int32), ("tile_row_end", ctypes.c_int32),
        ("bg", c_void_p), ("viewmatrix", c_void_p), ("projmatrix", c_void_p), ("campos", c_void_p),
        ("out_plane_stride", ctypes.c_int64), ("grad_plane_stride", ctypes.c_int64),
        ("out_replica_count", ctypes.c_int32), ("sh_grad_deferred", ctypes.c_int32),
        ("out_replica_base", ctypes.c_uint64 * 8),
    ]


class AdamGroup(ctypes.Structure):
    """struct surfel_adam_group (include/surfel_rasterizer.h)."""
    _fields_ = [("param", c_void_p), ("grad", c_void_p), ("exp_avg", c_void_p), ("exp_avg_sq", c_void_p),
                ("n", ctypes.c_longlong), ("step_size", c_float), ("bias2_sqrt", c_float),
                ("aligned16", ctypes.c_int)]


ADAM_MAX_GROUPS = 8


class DensifyGroup(ctypes.Structure):
    """struct surfel_densify_group (include/surfel_rasterizer.h)."""
    _fields_ = [("param", c_void_p), ("exp_avg", c_void_p), ("exp_avg_sq", c_void_p),
                ("out_param", c_void_p), ("out_exp_avg", c_void_p), ("out_exp_avg_sq", c_void_p),
                ("row_floats", c_int), ("kind", c_int)]


DENSIFY_MAX_GROUPS = 8
DENSIFY_COPY, DENSIFY_XYZ, DENSIFY_SCALING, DENSIFY_ROTATION = 0, 1, 2, 3


class TsdfFrame(ctypes.Structure):
    """struct surfel_tsdf_frame (include/surfel_rasterizer.h)."""
    _fields_ = [("full_proj_transform", c_float * 16), ("height", ctypes.c_int32), ("width", ctypes.c_int32),
                ("offset", ctypes.c_int64)]


# name -> (restype, argtypes); every symbol include/surfel_rasterizer.h declares
SIGNATURES = {
    "surfel_abi_version": (c_int, []),
    "surfel_last_error": (ctypes.c_char_p, []),
    "surfel_accepts_capacity": (c_int, []),
    "surfel_set_variant": (c_int, [ctypes.c_char_p, ctypes.c_char_p]),
    "surfel_geom_bytes": (c_size_t, [c_int]),
    "surfel_image_bytes": (c_size_t, [c_int, c_int]),
    "surfel_binning_bytes": (c_size_t, [c_size_t, c_int, c_int]),
    "surfel_geom_offsets": (c_int, [c_int, ctypes.POINTER(c_size_t)]),
    "surfel_binning_offsets": (c_int, [c_size_t, c_int, c_int, ctypes.POINTER(c_size_t)]),
    "surfel_image_offsets": (c_int, [c_int, c_int, ctypes.POINTER(c_size_t)]),
    "surfel_forward_preprocess": (c_int, [ctypes.POINTER(SurfelSettings), c_int, c_int] + [c_void_p] * 11 + [c_void_p]),
    "surfel_forward_render": (c_int, [ctypes.POINTER(SurfelSettings), c_int, c_uint32] + [c_void_p] * 4 + [c_int, c_void_p, c_void_p, c_void_p]),
    "surfel_bin_duplicate": (c_int, [ctypes.POINTER(SurfelSettings), c_int, c_uint32, c_void_p, c_void_p, c_void_p, c_void_p]),
    "surfel_bin_sort": (c_int, [ctypes.POINTER(SurfelSettings), c_uint32, c_void_p, c_void_p]),
    "surfel_bin_bucket": (c_int, [ctypes.POINTER(SurfelSettings), c_int, c_uint32, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "surfel_render_forward": (c_int, [ctypes.POINTER(SurfelSettings), c_uint32] + [c_void_p] * 5 + [c_void_p]),
    "surfel_grad_scratch_floats": (c_int, []),
    "surfel_backward": (c_int, [ctypes.POINTER(SurfelSettings), c_int, c_int, c_uint32] + [c_void_p] * 5 + [c_int]
                        + [c_void_p] * 15 + [c_int, c_void_p]),
    "surfel_sh_grad_expand": (c_int, [c_int, c_int, c_int] + [c_void_p] * 4 + [c_void_p]),
    "surfel_mark_visible": (c_int, [c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "surfel_sort_temp_bytes": (c_size_t, [c_size_t]),
    "surfel_post_forward": (c_int, [c_int, c_int, c_float] + [c_void_p] * 6 + [c_void_p]),
    "surfel_post_backward": (c_int, [c_int, c_int, c_float] + [c_void_p] * 9 + [c_void_p]),
    "surfel_post_reg_partials_bytes": (c_size_t, [c_int, c_int]),
    "surfel_post_reg_forward": (c_int, [c_int, c_int, c_float, ctypes.c_double, ctypes.c_double] + [c_void_p] * 6
                                + [c_void_p]),
    "surfel_post_reg_backward": (c_int, [c_int, c_int, c_float, ctypes.c_double, ctypes.c_double] + [c_void_p] * 6
                                 + [c_void_p]),
    "surfel_l1_ssim_forward": (c_int, [c_int, c_int, c_int] + [c_void_p] * 6 + [c_void_p]),
    "surfel_l1_ssim_backward": (c_int, [c_int, c_int, c_int] + [c_void_p] * 7 + [c_void_p]),
    "surfel_adam_step": (c_int, [c_int, ctypes.POINTER(AdamGroup), ctypes.c_double, ctypes.c_double, ctypes.c_double, c_void_p]),
    "surfel_densify_stats": (c_int, [c_int] + [c_void_p] * 5 + [c_void_p]),
    "surfel_ply_unpack": (c_int, [c_int, c_int, c_void_p, ctypes.POINTER(ctypes.c_int32), c_int] + [c_void_p] * 5 + [c_void_p]),
    "surfel_ply_pack": (c_int, [c_int] + [c_void_p] * 7 + [c_void_p]),
    "surfel_knn_workspace_bytes": (c_size_t, [c_int]),
    "surfel_knn_mean_sq_dist": (c_int, [c_int, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "surfel_densify_workspace_bytes": (c_size_t, [c_int]),
    "surfel_densify_plan": (c_int, [c_int] + [c_void_p] * 4 + [ctypes.c_double] * 4 + [c_int, ctypes.c_double]
                            + [c_void_p, c_size_t, c_void_p, c_void_p]),
    "surfel_densify_apply": (c_int, [c_int, c_int, c_int, c_int, ctypes.POINTER(DensifyGroup), c_void_p, c_void_p,
                                     c_size_t, c_void_p]),
    "surfel_tsdf_eval": (c_int, [ctypes.c_longlong, c_void_p, c_int, ctypes.POINTER(TsdfFrame), ctypes.c_longlong,
                                 c_void_p, c_void_p, ctypes.POINTER(c_float), ctypes.c_double, ctypes.c_double,
                                 c_void_p, c_void_p]),
    "surfel_tsdf_eval_grid": (c_int, [c_int, ctypes.POINTER(ctypes.c_double), c_int, ctypes.POINTER(TsdfFrame),
                                      ctypes.c_longlong, c_void_p, ctypes.POINTER(c_float), ctypes.c_double,
                                      ctypes.c_double, c_void_p, c_void_p]),
    "surfel_mcubes_crop_workspace_bytes": (c_size_t, [c_int]),
    "surfel_mcubes_crop_count": (c_int, [c_int, c_void_p, ctypes.POINTER(c_int), c_int, c_void_p, c_size_t, c_void_p,
                                         c_void_p]),
    "surfel_mcubes_crop_emit": (c_int, [c_int, c_void_p, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(c_int),
                                        c_int, c_void_p, c_size_t, ctypes.c_longlong, ctypes.c_longlong, c_void_p,
                                        c_void_p, c_void_p, c_void_p]),
    "surfel_mcubes_merge_workspace_bytes": (c_size_t, [ctypes.c_longlong]),
    "surfel_mcubes_merge": (c_int, [ctypes.c_longlong, c_void_p, c_void_p, ctypes.c_longlong, c_void_p, c_int,
                                    ctypes.POINTER(c_float), ctypes.c_double, c_void_p, c_size_t, c_void_p, c_void_p,
                                    c_void_p, c_void_p]),
    "surfel_meshpost_workspace_bytes": (c_size_t, [ctypes.c_longlong, ctypes.c_longlong]),
    "surfel_meshpost_clusters": (c_int, [ctypes.c_longlong, ctypes.c_longlong, c_void_p, c_void_p, c_size_t, c_void_p,
                                         c_void_p, c_void_p, c_void_p]),
    "surfel_meshpost_compact": (c_int, [ctypes.c_longlong, ctypes.c_longlong, c_void_p, c_void_p, c_void_p,
                                        ctypes.c_longlong, ctypes.c_longlong, c_void_p, c_size_t, c_void_p, c_void_p,
                                        c_void_p, c_void_p]),
    "surfel_chamfer_max_points": (ctypes.c_longlong, []),
    "surfel_chamfer_sample_workspace_bytes": (c_size_t, [ctypes.c_longlong]),
    "surfel_chamfer_sample_count": (c_int, [ctypes.c_longlong, ctypes.c_longlong, c_void_p, c_void_p,
                                            ctypes.c_double, c_void_p, c_size_t, c_void_p, c_void_p]),
    "surfel_chamfer_sample_emit": (c_int, [ctypes.c_longlong, ctypes.c_longlong, c_void_p, c_void_p, ctypes.c_double,
                                           c_void_p, c_size_t, ctypes.c_longlong, c_void_p, c_void_p]),
    "surfel_chamfer_workspace_bytes": (c_size_t, [ctypes.c_longlong, ctypes.c_longlong]),
    "surfel_chamfer_downsample": (c_int, [ctypes.c_longlong, ctypes.c_longlong, c_void_p, ctypes.c_double, c_void_p,
                                          c_size_t, ctypes.POINTER(c_int), c_void_p]),
    "surfel_chamfer_select": (c_int, [ctypes.c_longlong, ctypes.c_longlong, c_void_p, c_void_p]
                              + [ctypes.POINTER(ctypes.c_double)] * 3 + [ctypes.c_double, c_void_p,
                                                                         ctypes.POINTER(c_int),
                                                                         ctypes.POINTER(ctypes.c_double), c_void_p,
                                                                         c_size_t] + [c_void_p] * 8),
    "surfel_chamfer_distances": (c_int, [ctypes.c_longlong, ctypes.c_longlong, c_void_p, ctypes.c_longlong,
                                         ctypes.c_longlong, c_void_p, ctypes.c_longlong, c_void_p, c_void_p,
                                         ctypes.c_longlong, c_void_p, c_void_p, ctypes.c_double, ctypes.c_double,
                                         c_void_p, c_size_t] + [c_void_p] * 6),
    "surfel_cull_max_views": (c_int, []),
    "surfel_cull_max_radius": (c_int, []),
    "surfel_cull_workspace_bytes": (c_size_t, [ctypes.c_longlong, c_int, c_int, ctypes.c_longlong,
                                               ctypes.c_longlong]),
    "surfel_cull_dilate": (c_int, [c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p]),
    "surfel_cull_vertices": (c_int, [ctypes.c_longlong, c_void_p, ctypes.c_longlong, c_void_p, c_int, c_void_p,
                                     c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p,
                                     c_void_p]),
    "surfel_cull_emit": (c_int, [ctypes.c_longlong, c_void_p, ctypes.c_longlong, c_void_p,
                                 ctypes.POINTER(ctypes.c_double), c_void_p, ctypes.c_longlong, c_void_p, c_size_t,
                                 ctypes.c_longlong, ctypes.c_longlong, c_void_p, c_void_p, c_void_p, c_void_p]),
    "surfel_metrics_min_side": (c_int, []),
    "surfel_metrics_max_side": (c_int, []),
    "surfel_metrics_partials_count": (c_size_t, [c_int]),
    "surfel_metrics_lpips_input": (c_int, [c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "surfel_metrics_pack_conv": (c_int, [c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "surfel_metrics_conv3x3": (c_int, [c_int, c_int, c_int, c_int, c_int] + [c_void_p] * 5),
    "surfel_metrics_maxpool": (c_int, [c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "surfel_metrics_lpips_tap": (c_int, [c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "surfel_metrics_lpips_finish": (c_int, [ctypes.POINTER(ctypes.c_longlong)] + [c_void_p] * 4),
    "surfel_metrics_psnr": (c_int, [c_int, ctypes.c_longlong] + [c_void_p] * 5),
    "surfel_launch_count":(ctypes.c_ulonglong, []),
    "surfel_profile_enable": (None, [c_int]),
    "surfel_profile_num_stages": (c_int, []),
    "surfel_profile_stage_name": (ctypes.c_char_p, [c_int]),
    "surfel_profile_read": (c_int, [ctypes.POINTER(ctypes.c_double), ctypes.POINTER(c_int)]),
    "surfel_sort_pairs": (c_int, [c_void_p] * 4 + [c_size_t, c_int, c_void_p, ctypes.POINTER(c_int), c_void_p]),
}

_lib = None


def load():
    """Load the CUDA library; raise (never fall back) if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH) and not os.environ.get("SURFEL_LIB"):
        # not built yet (fresh checkout): compile it in-tree with nvcc.  This is a BUILD step, not a
        # fallback: if it fails there is no other implementation to fall back to.
        try:
            import importlib.util
            spec = importlib.util.spec_from_file_location("surfel_b200_build", os.path.join(os.path.dirname(_HERE), "build.py"))
            mod = importlib.util.module_from_spec(spec)
            spec.loader.exec_module(mod)
            mod.build()
        except Exception as ex:   # noqa: BLE001
            raise ImportError(f"could not build {LIB_PATH} with nvcc: {ex}") from ex
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found: build the sm_90a CUDA library first "
            "(python 2d-gaussian-splatting_b200/build.py, or __graft_entry__.build()). "
            "diff_surfel_rasterization has no CPU fallback.")
    _lib = load_handle(LIB_PATH)
    return _lib


def load_handle(path):
    """Open a build of the library at `path` (the main one, or a test variant under lib/variants/) as a separate
    handle with every signature of SIGNATURES configured on it; the global handle of load() is left alone."""
    if not os.path.exists(path):
        raise ImportError(f"{path} not found: build it first (python 2d-gaussian-splatting_b200/build.py)")
    lib = ctypes.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the symbol is not exported
        fn.restype, fn.argtypes = res, args
    if lib.surfel_abi_version() != 3:
        raise ImportError(f"{path}: ABI version mismatch")
    return lib


def check(status, lib=None):
    """Raise on a non-zero status, with the error string of the library handle that returned it (default: the
    global one)."""
    if status != 0:
        raise RuntimeError("surfel rasterizer: " + (lib or load()).surfel_last_error().decode())
