"""ctypes binding of include/neuralbody_b200.h -- the binding a reference maintainer would
add next to lib/networks/renderer/ (see INTEGRATION.md).  There is NO fallback: if the
shared library is missing or does not load, importing/using the product path raises."""
import ctypes as C
import os

from . import _build

NB_OK = 0
NB_DTYPE_F32, NB_DTYPE_F16 = 0, 1
NB_PRECISION_FP32, NB_PRECISION_TC_FP16, NB_PRECISION_TC_FP16X3, NB_PRECISION_TC_TF32X3 = 0, 1, 2, 3
NB_NUM_LEVELS = 4

EXPORTS = ["nb_abi_version", "nb_last_error", "nb_has_precision", "nb_packed_volume_bytes", "nb_packed_volume_level_offset",
           "nb_pack_volume", "nb_packed_weights_bytes", "nb_pack_weights", "nb_render_fwd",
           "nb_render_fwd_launches", "nb_render_fwd_workspace_bytes", "nb_render_bwd", "nb_render_bwd_frame", "nb_render_bwd_rays",
           "nb_render_bwd_maps", "nb_render_bwd_inputs", "nb_render_save_bytes",
           "nb_render_bwd_workspace_bytes", "nb_render_save_bytes_for", "nb_render_bwd_workspace_bytes_for", "nb_debug_gemm_tf32x3", "nb_debug_composite",
           "nb_debug_composite_bwd", "nb_decode_density", "nb_decode_density_workspace_bytes",
           "nb_decode_density_list", "nb_sample_pdf", "nb_sample_pdf_src",
           "nb_mcubes_workspace_bytes", "nb_mcubes_count", "nb_mcubes_emit", "nb_mesh_inside",
           "nb_mesh_inside_f64", "nb_image_rays_workspace_bytes", "nb_image_rays", "nb_image_rays_f64",
           "nb_train_rays_workspace_bytes", "nb_train_rays", "nb_item_images", "nb_mask_views_workspace_bytes",
           "nb_mask_views", "nb_eval_image_workspace_bytes",
           "nb_eval_image", "nb_vis_frame_workspace_bytes", "nb_vis_frame", "nb_mesh_ply_bytes", "nb_mesh_ply",
           "nb_image_loss_workspace_bytes", "nb_image_loss_fwd", "nb_image_loss_bwd", "nb_spconv_workspace_bytes",
           "nb_spconv_fwd", "nb_spconv_bwd"]


class nb_volume_level(C.Structure):
    _fields_ = [("data", C.c_void_p), ("C", C.c_int), ("D", C.c_int), ("H", C.c_int), ("W", C.c_int)]


class nb_decoder_weights(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in (
        "fc0_w", "fc0_b", "fc1_w", "fc1_b", "fc2_w", "fc2_b", "alpha_w", "alpha_b", "feature_w", "feature_b",
        "latent_w", "latent_b", "view_w", "view_b", "rgb_w", "rgb_b", "latent", "latent_index")] + \
        [("num_train_frame", C.c_int), ("batch", C.c_int)]


LevelDims = (C.c_int * 4) * NB_NUM_LEVELS


class nb_render_args(C.Structure):
    _fields_ = [
        ("batch", C.c_int), ("n_rays", C.c_int), ("n_samples", C.c_int),
        ("ray_o", C.c_void_p), ("ray_d", C.c_void_p), ("near", C.c_void_p), ("far", C.c_void_p),
        ("t_vals", C.c_void_p), ("t_rand", C.c_void_p),
        ("R", C.c_void_p), ("Th", C.c_void_p), ("bounds", C.c_void_p),
        ("voxel_size", C.c_float * 3), ("out_sh", C.c_int * 3), ("level_dims", LevelDims),
        ("volume_blob", C.c_void_p), ("volume_dtype", C.c_int),
        ("weights_blob", C.c_void_p),
        ("white_bkgd", C.c_int), ("precision", C.c_int),
        ("rgb_map", C.c_void_p), ("disp_map", C.c_void_p), ("acc_map", C.c_void_p), ("weights", C.c_void_p),
        ("depth_map", C.c_void_p), ("raw", C.c_void_p), ("out_ray_stride", C.c_int),
        ("mask_msks", C.c_void_p), ("mask_RT", C.c_void_p), ("mask_Ks", C.c_void_p),
        ("mask_nv", C.c_int), ("mask_H", C.c_int), ("mask_W", C.c_int), ("mask_R0", C.c_void_p), ("mask_Th0", C.c_void_p),
        ("skip_empty", C.c_int), ("stats", C.c_void_p), ("save", C.c_void_p),
        ("trace", C.c_void_p), ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t), ("z_vals", C.c_void_p),
    ]


class nb_importance_args(C.Structure):
    _fields_ = [("n_rays_total", C.c_int), ("n_samples", C.c_int), ("n_importance", C.c_int),
                ("near", C.c_void_p), ("far", C.c_void_p), ("t_vals", C.c_void_p), ("t_rand", C.c_void_p),
                ("weights", C.c_void_p), ("u", C.c_void_p), ("z_out", C.c_void_p), ("z_samples", C.c_void_p)]


class nb_mcubes_args(C.Structure):
    _fields_ = [("grid", C.c_void_p), ("nx", C.c_int), ("ny", C.c_int), ("nz", C.c_int), ("isovalue", C.c_double),
                ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t), ("counts", C.c_void_p),
                ("vertices", C.c_void_p), ("triangles", C.c_void_p)]


class nb_mesh_inside_args(C.Structure):
    _fields_ = [("x", C.c_void_p), ("y", C.c_void_p), ("z", C.c_void_p), ("nx", C.c_int), ("ny", C.c_int), ("nz", C.c_int),
                ("msks", C.c_void_p), ("RT", C.c_void_p), ("Ks", C.c_void_p), ("nv", C.c_int), ("H", C.c_int), ("W", C.c_int),
                ("inside", C.c_void_p)]


NB_SCALAR_F32, NB_SCALAR_F64 = 0, 1
NB_TRAIN_CAM_DOUBLES = 30
NB_TRAIN_CLASS_BODY, NB_TRAIN_CLASS_FACE, NB_TRAIN_CLASS_BOUND = 1, 2, 4
NB_TRAIN_RAYS_OK, NB_TRAIN_RAYS_ROUNDS, NB_TRAIN_RAYS_EMPTY, NB_TRAIN_RAYS_REPLAY = 0, 1, 2, 3
NB_TRAIN_RAYS_MAX_ROUNDS = 64


class nb_train_rays_args(C.Structure):
    _fields_ = [("B", C.c_int), ("H", C.c_int), ("W", C.c_int), ("n_rays", C.c_int), ("body_ratio", C.c_double),
                ("face_ratio", C.c_double), ("k_kind", C.c_int), ("rt_kind", C.c_int), ("class_map", C.c_void_p),
                ("image", C.c_void_p), ("cams", C.c_void_p), ("draws", C.c_void_p), ("draw_offset", C.c_void_p),
                ("key", C.c_ulonglong * 2), ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t),
                ("ray_o", C.c_void_p), ("ray_d", C.c_void_p), ("near", C.c_void_p), ("far", C.c_void_p), ("rgb", C.c_void_p),
                ("coord", C.c_void_p), ("rounds", C.c_void_p), ("status", C.c_void_p)]


NB_ITEM_CAM_DOUBLES = 17
NB_ITEM_MAX_W = 4096
NB_ITEM_BKGD_NONE, NB_ITEM_BKGD_BLACK, NB_ITEM_BKGD_WHITE = 0, 1, 2
NB_ITEM_CLASS_NONE, NB_ITEM_CLASS_H36M, NB_ITEM_CLASS_SNAPSHOT = 0, 1, 2


class nb_item_images_args(C.Structure):
    _fields_ = [("B", C.c_int), ("H0", C.c_int), ("W0", C.c_int), ("H", C.c_int), ("W", C.c_int), ("n_dist", C.c_int),
                ("bkgd", C.c_int), ("class_rule", C.c_int), ("img_u8", C.c_void_p), ("msk_u8", C.c_void_p),
                ("cams", C.c_void_p), ("bound", C.c_void_p), ("img", C.c_void_p), ("msk", C.c_void_p),
                ("class_map", C.c_void_p)]


class nb_mask_views_args(C.Structure):
    _fields_ = [("nv", C.c_int), ("H0", C.c_int), ("W0", C.c_int), ("H", C.c_int), ("W", C.c_int), ("n_dist", C.c_int),
                ("binarise", C.c_int), ("dilate", C.c_int), ("msk_u8", C.c_void_p), ("cams", C.c_void_p),
                ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t), ("msks", C.c_void_p)]


NB_EVAL_OK, NB_EVAL_COUNT, NB_EVAL_SMALL = 0, 1, 2


class nb_eval_image_result(C.Structure):
    _fields_ = [("status", C.c_int), ("count", C.c_int), ("box", C.c_int * 4), ("sq_sum", C.c_double), ("mse", C.c_double),
                ("psnr", C.c_double), ("ssim", C.c_double), ("ssim_channel", C.c_double * 3)]


class nb_eval_image_args(C.Structure):
    _fields_ = [("n", C.c_int), ("H", C.c_int), ("W", C.c_int), ("white_bkgd", C.c_int), ("eval_whole_img", C.c_int),
                ("rgb_pred", C.c_void_p), ("rgb_gt", C.c_void_p), ("mask_at_box", C.c_void_p), ("workspace", C.c_void_p),
                ("workspace_bytes", C.c_size_t), ("result", C.c_void_p), ("crop_pred", C.c_void_p),
                ("crop_gt", C.c_void_p)]


NB_VIS_OK, NB_VIS_COUNT = 0, 1


class nb_vis_frame_result(C.Structure):
    _fields_ = [("status", C.c_int), ("count", C.c_int)]


class nb_vis_frame_args(C.Structure):
    _fields_ = [("n", C.c_int), ("H", C.c_int), ("W", C.c_int), ("white_bkgd", C.c_int), ("rgb_map", C.c_void_p),
                ("mask_at_box", C.c_void_p), ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t),
                ("result", C.c_void_p), ("frame", C.c_void_p)]


NB_MESH_PLY_OK, NB_MESH_PLY_FACE = 0, 1
NB_MESH_PLY_BODY_OFFSET = 16


class nb_mesh_ply_result(C.Structure):
    _fields_ = [("status", C.c_int), ("reserved", C.c_int * 3)]


class nb_mesh_ply_args(C.Structure):
    _fields_ = [("nv", C.c_longlong), ("nf", C.c_longlong), ("vertices", C.c_void_p), ("faces", C.c_void_p),
                ("out", C.c_void_p), ("out_bytes", C.c_size_t)]


class nb_image_loss_args(C.Structure):
    _fields_ = [("rays", C.c_int), ("pred", C.c_void_p), ("gt", C.c_void_p), ("mask", C.c_void_p), ("workspace", C.c_void_p),
                ("workspace_bytes", C.c_size_t), ("loss", C.c_void_p), ("count", C.c_void_p)]


NB_SPCONV_LAYERS = 17
_SpLayers = C.c_void_p * NB_SPCONV_LAYERS


class nb_spconv_args(C.Structure):
    _fields_ = [("batch", C.c_int), ("n_points", C.c_int), ("n_vert", C.c_int), ("out_sh", C.c_int * 3),
                ("coord", C.c_void_p), ("code", C.c_void_p), ("weight", _SpLayers), ("bn_weight", _SpLayers),
                ("bn_bias", _SpLayers), ("running_mean", _SpLayers), ("running_var", _SpLayers),
                ("num_batches_tracked", _SpLayers), ("training", C.c_int), ("momentum", C.c_float), ("eps", C.c_float),
                ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t), ("volumes", C.c_void_p * NB_NUM_LEVELS),
                ("row_counts", C.c_void_p)]


class nb_spconv_grads(C.Structure):
    _fields_ = [("d_volumes", C.c_void_p * NB_NUM_LEVELS), ("d_code", C.c_void_p), ("d_weight", _SpLayers),
                ("d_bn_weight", _SpLayers), ("d_bn_bias", _SpLayers)]


class nb_image_rays_args(C.Structure):
    _fields_ = [("H", C.c_int), ("W", C.c_int), ("bounds", C.c_float * 6), ("workspace", C.c_void_p),
                ("workspace_bytes", C.c_size_t), ("ray_o", C.c_void_p), ("ray_d", C.c_void_p), ("near", C.c_void_p),
                ("far", C.c_void_p), ("mask_at_box", C.c_void_p), ("count", C.c_void_p), ("image", C.c_void_p),
                ("rgb", C.c_void_p), ("k_f32", C.c_int), ("rank", C.c_int), ("world", C.c_int), ("chunk", C.c_int),
                ("n_local", C.c_int)]


class nb_render_bwd_args(C.Structure):
    _fields_ = [
        ("fwd", C.POINTER(nb_render_args)), ("save", C.c_void_p), ("raw", C.c_void_p),
        ("d_rgb_map", C.c_void_p), ("d_depth_map", C.c_void_p), ("d_acc_map", C.c_void_p),
        ("weights", C.POINTER(nb_decoder_weights)), ("grads", C.POINTER(nb_decoder_weights)),
        ("d_volumes", C.c_void_p * NB_NUM_LEVELS), ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t),
    ]


class nb_render_input_grads(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("d_R", "d_Th", "d_ray_o", "d_ray_d", "d_near", "d_far", "d_z_vals", "d_bounds")]


_lib = None


def load(path=None):
    """dlopen libneuralbody_b200.so and declare every prototype. Raises if absent."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    path = path or os.environ.get("NB_LIB_PATH") or _build.LIB_PATH
    if not os.path.exists(path):
        raise RuntimeError(
            "libneuralbody_b200.so not found at %s -- run `python -c 'import __graft_entry__ as g; g.build()'`; "
            "there is no CPU fallback for the render path" % path)
    lib = C.CDLL(path)
    lib.nb_abi_version.restype = C.c_int
    lib.nb_last_error.restype = C.c_char_p
    lib.nb_has_precision.restype = C.c_int
    lib.nb_has_precision.argtypes = [C.c_int]
    lib.nb_packed_volume_bytes.restype = C.c_size_t
    lib.nb_packed_volume_bytes.argtypes = [LevelDims, C.c_int, C.c_int]
    lib.nb_packed_volume_level_offset.restype = C.c_size_t
    lib.nb_packed_volume_level_offset.argtypes = [LevelDims, C.c_int, C.c_int, C.c_int]
    lib.nb_pack_volume.restype = C.c_int
    lib.nb_pack_volume.argtypes = [nb_volume_level * NB_NUM_LEVELS, C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]
    lib.nb_packed_weights_bytes.restype = C.c_size_t
    lib.nb_packed_weights_bytes.argtypes = [C.c_int]
    lib.nb_pack_weights.restype = C.c_int
    lib.nb_pack_weights.argtypes = [C.POINTER(nb_decoder_weights), C.c_void_p, C.c_size_t, C.c_void_p]
    lib.nb_render_fwd.restype = C.c_int
    lib.nb_render_fwd.argtypes = [C.POINTER(nb_render_args), C.c_void_p]
    lib.nb_render_fwd_launches.restype = C.c_int
    lib.nb_render_fwd_launches.argtypes = [C.c_int]
    lib.nb_render_fwd_workspace_bytes.restype = C.c_size_t
    lib.nb_render_fwd_workspace_bytes.argtypes = [C.c_int, C.c_int, C.c_int]
    lib.nb_render_bwd.restype = C.c_int
    lib.nb_render_bwd.argtypes = [C.POINTER(nb_render_bwd_args), C.c_void_p]
    lib.nb_render_bwd_frame.restype = C.c_int
    lib.nb_render_bwd_frame.argtypes = [C.POINTER(nb_render_bwd_args), C.c_void_p, C.c_void_p, C.c_void_p]
    lib.nb_render_bwd_rays.restype = C.c_int
    lib.nb_render_bwd_rays.argtypes = [C.POINTER(nb_render_bwd_args), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p]
    lib.nb_render_bwd_maps.restype = C.c_int
    lib.nb_render_bwd_maps.argtypes = [C.POINTER(nb_render_bwd_args), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p]
    lib.nb_render_bwd_inputs.restype = C.c_int
    lib.nb_render_bwd_inputs.argtypes = [C.POINTER(nb_render_bwd_args), C.c_void_p, C.c_void_p,
                                         C.POINTER(nb_render_input_grads), C.c_void_p]
    lib.nb_render_save_bytes.restype = C.c_size_t
    lib.nb_render_save_bytes.argtypes = [C.c_int, C.c_int, C.c_int]
    lib.nb_render_bwd_workspace_bytes.restype = C.c_size_t
    lib.nb_render_bwd_workspace_bytes.argtypes = [C.c_int, C.c_int, C.c_int]
    lib.nb_render_save_bytes_for.restype = C.c_size_t
    lib.nb_render_save_bytes_for.argtypes = [C.POINTER(nb_render_args)]
    lib.nb_render_bwd_workspace_bytes_for.restype = C.c_size_t
    lib.nb_render_bwd_workspace_bytes_for.argtypes = [C.POINTER(nb_render_args)]
    lib.nb_debug_gemm_tf32x3.restype = C.c_int
    lib.nb_debug_gemm_tf32x3.argtypes = [C.c_void_p] * 3 + [C.c_int] * 6 + [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    lib.nb_debug_composite.restype = C.c_int
    lib.nb_debug_composite.argtypes = [C.POINTER(nb_render_args), C.c_void_p, C.c_void_p]
    lib.nb_debug_composite_bwd.restype = C.c_int
    lib.nb_debug_composite_bwd.argtypes = [C.POINTER(nb_render_args)] + [C.c_void_p] * 7 + [C.POINTER(nb_render_input_grads),
                                                                                            C.c_void_p, C.c_void_p]
    lib.nb_decode_density.restype = C.c_int
    lib.nb_decode_density.argtypes = [C.POINTER(nb_render_args), C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    lib.nb_decode_density_workspace_bytes.restype = C.c_size_t
    lib.nb_decode_density_workspace_bytes.argtypes = [C.c_int, C.c_int]
    lib.nb_decode_density_list.restype = C.c_int
    lib.nb_decode_density_list.argtypes = [C.POINTER(nb_render_args), C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    lib.nb_sample_pdf.restype = C.c_int
    lib.nb_sample_pdf.argtypes = [C.POINTER(nb_importance_args), C.c_void_p]
    lib.nb_sample_pdf_src.restype = C.c_int
    lib.nb_sample_pdf_src.argtypes = [C.POINTER(nb_importance_args), C.c_void_p, C.c_void_p]
    lib.nb_mcubes_workspace_bytes.restype = C.c_size_t
    lib.nb_mcubes_workspace_bytes.argtypes = [C.c_int] * 3
    lib.nb_mcubes_count.restype = C.c_int
    lib.nb_mcubes_count.argtypes = [C.POINTER(nb_mcubes_args), C.c_void_p]
    lib.nb_mcubes_emit.restype = C.c_int
    lib.nb_mcubes_emit.argtypes = [C.POINTER(nb_mcubes_args), C.c_void_p]
    lib.nb_mesh_inside.restype = C.c_int
    lib.nb_mesh_inside.argtypes = [C.POINTER(nb_mesh_inside_args), C.c_void_p]
    lib.nb_mesh_inside_f64.restype = C.c_int
    lib.nb_mesh_inside_f64.argtypes = [C.POINTER(nb_mesh_inside_args), C.c_void_p, C.c_void_p, C.c_void_p]
    lib.nb_image_rays_workspace_bytes.restype = C.c_size_t
    lib.nb_image_rays_workspace_bytes.argtypes = [C.c_int, C.c_int]
    lib.nb_image_rays.restype = C.c_int
    lib.nb_image_rays.argtypes = [C.POINTER(nb_image_rays_args)] + [C.POINTER(C.c_float)] * 4 + [C.c_void_p]
    lib.nb_image_rays_f64.restype = C.c_int
    lib.nb_image_rays_f64.argtypes = [C.POINTER(nb_image_rays_args)] + [C.POINTER(C.c_double)] * 4 + [C.c_void_p]
    lib.nb_train_rays_workspace_bytes.restype = C.c_size_t
    lib.nb_train_rays_workspace_bytes.argtypes = [C.c_int, C.c_int, C.c_int]
    lib.nb_train_rays.restype = C.c_int
    lib.nb_train_rays.argtypes = [C.POINTER(nb_train_rays_args), C.c_void_p]
    lib.nb_item_images.restype = C.c_int
    lib.nb_item_images.argtypes = [C.POINTER(nb_item_images_args), C.c_void_p]
    lib.nb_mask_views_workspace_bytes.restype = C.c_size_t
    lib.nb_mask_views_workspace_bytes.argtypes = [C.c_int] * 3
    lib.nb_mask_views.restype = C.c_int
    lib.nb_mask_views.argtypes = [C.POINTER(nb_mask_views_args), C.c_void_p]
    lib.nb_eval_image_workspace_bytes.restype = C.c_size_t
    lib.nb_eval_image_workspace_bytes.argtypes = [C.c_int, C.c_int, C.c_int]
    lib.nb_eval_image.restype = C.c_int
    lib.nb_eval_image.argtypes = [C.POINTER(nb_eval_image_args), C.c_void_p]
    lib.nb_vis_frame_workspace_bytes.restype = C.c_size_t
    lib.nb_vis_frame_workspace_bytes.argtypes = [C.c_int, C.c_int]
    lib.nb_vis_frame.restype = C.c_int
    lib.nb_vis_frame.argtypes = [C.POINTER(nb_vis_frame_args), C.c_void_p]
    lib.nb_mesh_ply_bytes.restype = C.c_size_t
    lib.nb_mesh_ply_bytes.argtypes = [C.c_longlong, C.c_longlong]
    lib.nb_mesh_ply.restype = C.c_int
    lib.nb_mesh_ply.argtypes = [C.POINTER(nb_mesh_ply_args), C.c_void_p]
    lib.nb_image_loss_workspace_bytes.restype = C.c_size_t
    lib.nb_image_loss_workspace_bytes.argtypes = []
    lib.nb_image_loss_fwd.restype = C.c_int
    lib.nb_image_loss_fwd.argtypes = [C.POINTER(nb_image_loss_args), C.c_void_p]
    lib.nb_image_loss_bwd.restype = C.c_int
    lib.nb_image_loss_bwd.argtypes = [C.POINTER(nb_image_loss_args), C.c_void_p, C.c_void_p, C.c_void_p]
    lib.nb_spconv_workspace_bytes.restype = C.c_size_t
    lib.nb_spconv_workspace_bytes.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_int)]
    lib.nb_spconv_fwd.restype = C.c_int
    lib.nb_spconv_fwd.argtypes = [C.POINTER(nb_spconv_args), C.c_void_p]
    lib.nb_spconv_bwd.restype = C.c_int
    lib.nb_spconv_bwd.argtypes = [C.POINTER(nb_spconv_args), C.POINTER(nb_spconv_grads), C.c_void_p]
    if lib.nb_abi_version() != 6:
        raise RuntimeError("libneuralbody_b200.so ABI version mismatch")
    if path in (_build.LIB_PATH, os.environ.get("NB_LIB_PATH")):
        _lib = lib
    return lib


def check(status, what):
    if status != NB_OK:
        msg = load().nb_last_error().decode("utf-8", "replace")
        raise RuntimeError("%s failed (status %d): %s" % (what, status, msg))
