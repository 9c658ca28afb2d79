"""ctypes binding of the C-ABI library (include/read_b200.h).

The product path fails LOUDLY when the CUDA library is missing or the device is not an H100 (sm_90):
there is no CPU or eager-PyTorch fallback anywhere in this package.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# READ_B200_LIB: load another build of the library (e.g. the -DREAD_DIAG build: python -m read_b200.build --diag)
LIB_PATH = os.environ.get("READ_B200_LIB") or os.path.join(_HERE, "libread_b200.so")

c_int, c_i64, c_u32 = ctypes.c_int, ctypes.c_int64, ctypes.c_uint32
c_vp = ctypes.c_void_p

MAX_SRC = 4

# enums (mirror include/read_b200.h)
FEAT_NCHW_F32, FEAT_NHWC_F32, FEAT_NHWC_BF16 = 0, 1, 2
TEXACT = {"none": 0, "sigmoid": 1, "tanh": 2}
ACT_F32, ACT_BF16 = 0, 1
SRC_IDENTITY, SRC_NEAREST_DOWN, SRC_NEAREST_UP, SRC_BILINEAR_UP4 = 0, 1, 2, 3
OUT_NHWC, OUT_NCHW_F32, OUT_RAW_NHWC = 0, 1, 2
CONV_AUTO, CONV_GENERIC, CONV_TCGEN05, CONV_TCGEN05_GATHER = 0, 1, 2, 3   # names kept from the ABI; 2 / 3 are the wgmma kernels


class ReadSrc(ctypes.Structure):
    _fields_ = [("ptr", c_vp), ("C", ctypes.c_int32), ("H", ctypes.c_int32), ("W", ctypes.c_int32),
                ("mode", ctypes.c_int32), ("factor", ctypes.c_int32)]


class ReadConvDesc(ctypes.Structure):
    _fields_ = [
        ("act_dtype", ctypes.c_int32), ("n_src", ctypes.c_int32), ("src", ReadSrc * MAX_SRC),
        ("mul", c_vp),
        ("B", ctypes.c_int32), ("Hin", ctypes.c_int32), ("Win", ctypes.c_int32), ("Cin", ctypes.c_int32),
        ("Hout", ctypes.c_int32), ("Wout", ctypes.c_int32), ("Cout", ctypes.c_int32),
        ("k", ctypes.c_int32), ("stride", ctypes.c_int32), ("pad", ctypes.c_int32), ("elu", ctypes.c_int32),
        ("w_generic", c_vp), ("w_tc", c_vp),
        ("bias_f", c_vp), ("bias_m", c_vp), ("bn_scale", c_vp), ("bn_shift", c_vp),
        ("residual", c_vp), ("out", c_vp), ("out_mode", ctypes.c_int32),
        ("out2", c_vp), ("out2_mul", c_vp), ("impl", ctypes.c_int32),
        ("addin", c_vp), ("addin_H", ctypes.c_int32), ("addin_W", ctypes.c_int32),
    ]


MAX_TEX_SLOTS, MAX_TEX_ITEMS = 16, 64
MAX_SEGMENTS = 128           # READ_MAX_SEGMENTS: segments per read_raster_project_segments launch
MAX_SEGMENTS_CULLED = 4096   # READ_MAX_SEGMENTS_CULLED: segments per read_raster_project_segments_culled launch


class ReadTexTable(ctypes.Structure):
    _fields_ = [("tex_nd", c_vp * MAX_TEX_SLOTS), ("N", c_i64 * MAX_TEX_SLOTS), ("grad_nd", c_vp * MAX_TEX_SLOTS),
                ("touched", c_vp * MAX_TEX_SLOTS), ("n_slots", ctypes.c_int32), ("n_items", ctypes.c_int32),
                ("slot", ctypes.c_uint8 * MAX_TEX_ITEMS)]


MAX_LEVELS = 8              # READ_MAX_LEVELS
MAX_POINT_SIZE = 64         # READ_MAX_POINT_SIZE: widest point sprite, in pixels


class ReadSpriteDesc(ctypes.Structure):
    _fields_ = [("size", ctypes.c_float * MAX_LEVELS), ("relative", ctypes.c_int32 * MAX_LEVELS), ("point_sizes", c_vp)]


PANORAMA_MAX_WIDTH = 65536  # READ_PANORAMA_MAX_WIDTH


class ReadPanoramaDesc(ctypes.Structure):
    _fields_ = [("theta_half", ctypes.c_float), ("k_w", ctypes.c_float), ("t_hi", ctypes.c_float), ("k_h", ctypes.c_float),
                ("znear", ctypes.c_float), ("zfar", ctypes.c_float), ("width", ctypes.c_int32), ("margin", ctypes.c_int32),
                ("full", ctypes.c_int32)]


VIEW_MODES = {"color": 0, "normals": 1, "depth": 2, "uv": 3, "xyz": 4, "label": 5}   # READ_VIEW_*


class ReadPointViewDesc(ctypes.Structure):
    _fields_ = [("mode", ctypes.c_int32), ("submode", ctypes.c_int32), ("colors", c_vp), ("normals", c_vp), ("xyz", c_vp),
                ("n", c_i64), ("total_m", ctypes.c_float * 16), ("m_view", ctypes.c_float * 16), ("cam", ctypes.c_float * 3),
                ("lo", ctypes.c_float * 3), ("hi", ctypes.c_float * 3), ("clear", ctypes.c_float * 4),
                ("flip_vertical", ctypes.c_int32)]


class ReadHaloDesc(ctypes.Structure):
    _fields_ = [("src_up", c_vp), ("src_dn", c_vp), ("peer_up_slot", c_vp), ("peer_dn_slot", c_vp),
                ("peer_up_flag", c_vp), ("peer_dn_flag", c_vp), ("slot_from_up", c_vp), ("slot_from_dn", c_vp),
                ("flag_from_up", c_vp), ("flag_from_dn", c_vp), ("dst_top", c_vp), ("dst_bot", c_vp),
                ("bytes", c_i64), ("epoch", c_vp), ("cta_counter", c_vp)]


_SIGS = {
    "read_version": (c_int, []),
    "read_last_error": (ctypes.c_char_p, []),
    "read_device_ok": (c_int, []),
    "read_set_option": (c_int, [ctypes.c_char_p, c_int]),
    "read_pyramid_entries": (c_i64, [c_int, c_int, c_int, c_int]),
    "read_pyramid_level_offset": (c_i64, [c_int, c_int, c_int, c_int]),
    "read_level_size": (None, [c_int, c_int, c_int, ctypes.POINTER(c_int), ctypes.POINTER(c_int)]),
    "read_zbuf_clear": (c_int, [c_vp, c_i64, c_vp]),
    "read_raster_project": (c_int, [c_vp, c_i64, c_i64, c_vp, c_int, c_int, c_int, c_int, c_vp, c_vp]),
    "read_raster_project_direct": (c_int, [c_vp, c_i64, c_i64, c_vp, c_int, c_int, c_int, c_int, c_vp, c_vp]),
    "read_raster_derive_levels": (c_int, [c_int, c_int, c_int, c_int, c_vp, c_vp]),
    "read_raster_project_sorted": (c_int, [c_vp, c_i64, c_vp, c_int, c_int, c_int, c_vp, c_vp]),
    "read_raster_project_sorted_views": (c_int, [c_vp, c_i64, c_vp, c_int, c_int, c_int, c_int, c_vp, c_vp]),
    "read_raster_project_segments": (c_int, [c_vp, c_i64, c_vp, c_vp, c_vp, c_int, c_vp, c_int, c_int, c_int, c_int, c_vp,
                                             c_vp]),
    "read_raster_cull_workspace_bytes": (c_i64, [c_i64]),
    "read_raster_project_segments_culled": (c_int, [c_vp, c_i64, c_vp, c_int, c_i64, c_vp, c_vp, c_vp, c_vp, c_i64, c_int, c_int,
                                                    c_int, c_int, c_vp, c_vp]),
    "read_gather_backward_sparse": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_int, c_i64, c_vp, c_vp, c_vp]),
    "read_sparse_rmsprop_step": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_int, c_int, ctypes.c_float, ctypes.c_float,
                                         ctypes.c_float, ctypes.c_float, c_vp]),
    "read_square_avg_dense": (c_int, [c_vp, c_vp, c_i64, c_int, c_int, ctypes.c_float, c_vp, c_vp]),
    "read_compact_touched": (c_int, [c_vp, c_vp, c_i64, c_int, c_vp, c_int, c_vp, c_vp, c_vp]),
    "read_scatter_pairs": (c_int, [c_vp, c_vp, c_int, c_int, c_i64, c_vp, c_vp, c_vp]),
    # the L2 regulariser of PointTexture without a dense gradient (read_b200.train._RegLoss)
    "read_reg_loss_workspace_bytes": (c_i64, [c_int, c_i64]),
    "read_reg_loss": (c_int, [c_vp, c_int, c_i64, ctypes.c_double, c_vp, c_vp, c_vp]),
    "read_sparse_rmsprop_step_reg": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_int, c_int, ctypes.c_float, ctypes.c_float,
                                             ctypes.c_float, ctypes.c_float, c_vp, c_vp]),
    "read_ipc_alloc": (c_int, [c_i64, ctypes.POINTER(c_vp), ctypes.c_char_p]),
    "read_ipc_open": (c_int, [ctypes.c_char_p, ctypes.POINTER(c_vp)]),
    "read_ipc_close": (c_int, [c_vp]),
    "read_ipc_free": (c_int, [c_vp]),
    "read_epoch_bump": (c_int, [c_vp, c_vp]),
    "read_halo_exchange": (c_int, [ctypes.POINTER(ReadHaloDesc), c_vp]),
    "read_stage_net_inputs": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_int, c_int, c_vp, c_vp]),
    "read_raster_direct_mask": (c_u32, [c_int, c_int, c_int]),
    "read_raster_sprites_sorted": (c_int, [c_vp, c_i64, c_vp, c_int, c_int, c_int, c_int, ctypes.POINTER(ReadSpriteDesc), c_vp, c_vp]),
    "read_raster_sprites_segments": (c_int, [c_vp, c_i64, c_vp, c_vp, c_vp, c_int, c_vp, c_int, c_int, c_int, c_int,
                                             ctypes.POINTER(ReadSpriteDesc), c_vp, c_vp]),
    "read_raster_sprites_segments_culled": (c_int, [c_vp, c_i64, c_vp, c_int, c_i64, c_vp, c_vp, c_vp, c_vp, c_i64, c_int, c_int,
                                                    c_int, c_int, ctypes.POINTER(ReadSpriteDesc), c_vp, c_vp]),
    "read_raster_panorama_sorted": (c_int, [c_vp, c_i64, c_vp, c_int, c_int, c_int, c_int, ctypes.POINTER(ReadPanoramaDesc), c_vp,
                                            c_vp]),
    "read_raster_panorama_segments_culled": (c_int, [c_vp, c_i64, c_vp, c_int, c_i64, c_vp, c_vp, c_vp, c_vp, c_i64, c_int, c_int,
                                                     c_int, c_int, ctypes.POINTER(ReadPanoramaDesc), c_vp, c_vp]),
    "read_zbuf_resolve": (c_int, [c_vp, c_i64, c_vp, c_vp, c_vp]),
    "read_pcpr_forward": (c_int, [c_vp, c_i64, c_vp, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_vp]),
    "read_texture_to_point_major": (c_int, [c_vp, c_int, c_i64, c_vp, c_vp]),
    "read_texture_to_channel_major": (c_int, [c_vp, c_int, c_i64, c_vp, c_vp]),
    "read_gather_from_index": (c_int, [c_vp, c_int, c_i64, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp]),
    "read_gather_from_zbuf": (c_int, [c_vp, c_int, c_i64, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp]),
    "read_pyramid_resolve_gather": (c_int, [c_vp, c_int, c_i64, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                            ctypes.POINTER(c_vp), c_int, c_vp]),
    "read_gather_backward": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_int, c_i64, c_vp, c_vp]),
    "read_gather_from_index_items": (c_int, [ctypes.POINTER(ReadTexTable), c_vp, c_int, c_int, c_int, c_int, c_vp, c_vp]),
    "read_gather_backward_items": (c_int, [c_vp, c_vp, ctypes.POINTER(ReadTexTable), c_int, c_int, c_vp]),
    "read_gather_backward_sparse_items": (c_int, [c_vp, c_vp, ctypes.POINTER(ReadTexTable), c_int, c_int, c_vp]),
    "read_gather_backward_items_det": (c_int, [c_vp, c_vp, ctypes.POINTER(ReadTexTable), c_int, c_int, c_vp, c_vp]),
    "read_gather_backward_sparse_items_det": (c_int, [c_vp, c_vp, ctypes.POINTER(ReadTexTable), c_int, c_int, c_vp, c_vp]),
    "read_generic_npad": (c_int, [c_int]),
    "read_pack_weights_generic": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_vp, c_vp]),
    "read_tc_weight_elems": (c_i64, [c_int, c_int, c_int]),
    "read_pack_weights_tc": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_vp, c_vp]),
    "read_pack_weights_tc_strided": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp, c_vp]),
    "read_pack_weights_tc_for": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp]),
    "read_pack_weights_tc_dgrad": (c_int, [c_vp, c_vp, c_int, c_int, c_vp, c_vp]),
    "read_pack_weights_tc_dgrad1x1": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp, c_vp]),
    "read_gate_backward": (c_int, [c_vp, c_vp, c_i64, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                   c_vp]),
    "read_conv3x3_wgrad": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp]),
    "read_conv3x3_dgrad_cin8": (c_int, [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp, c_vp]),
    "read_conv_wgrad": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp]),
    "read_pack_weights_dgrad_s2": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_vp, c_vp]),
    "read_conv_dgrad_s2": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp]),
    "read_bn_workspace_bytes": (c_i64, [c_int]),
    "read_bn_batch_stats": (c_int, [c_vp, c_i64, c_int, c_int, c_vp, c_vp, ctypes.c_float, ctypes.c_float, c_vp, c_vp, c_vp, c_vp,
                                    c_vp, c_vp, c_vp, c_vp, c_vp]),
    "read_bn_apply": (c_int, [c_vp, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "read_bn_backward_reduce": (c_int, [c_vp, c_vp, c_i64, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "read_gate_backward_batch_stats": (c_int, [c_vp, c_vp, c_i64, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                               c_vp, c_vp]),
    "read_bn_workspace_bytes_items": (c_i64, [c_int, c_int]),
    "read_bn_batch_stats_items": (c_int, [c_vp, c_int, c_i64, c_int, c_int, c_vp, c_vp, ctypes.c_float, ctypes.c_float, c_vp, c_vp,
                                          c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "read_bn_apply_items": (c_int, [c_vp, c_int, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "read_bn_backward_reduce_items": (c_int, [c_vp, c_vp, c_int, c_i64, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "read_gate_backward_batch_stats_items": (c_int, [c_vp, c_vp, c_int, c_i64, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                                     c_vp, c_vp, c_vp, c_vp]),
    "read_vgg_workspace_bytes": (c_i64, []),
    "read_vgg_normalize": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_vp]),
    "read_vgg_post": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_vp, c_int, c_vp, c_vp, c_vp, ctypes.c_double, c_vp, c_vp]),
    "read_vgg_dgrad_in": (c_int, [c_vp, c_int, c_vp, c_int, c_int, c_int, c_int, c_vp, ctypes.c_float, c_vp, c_vp]),
    "read_vgg_image_grad": (c_int, [c_vp, c_int, c_int, c_int, c_vp, c_vp, c_vp]),
    "read_vgg_normalize_masked": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "read_vgg_post_partial": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_vp, ctypes.c_double, c_vp, c_vp]),
    "read_vgg_dgrad_in_partial": (c_int, [c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_vp, ctypes.c_float, c_vp, c_vp]),
    "read_vgg_image_grad_masked": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_vp, c_vp, c_vp]),
    "read_gather_backward_det_workspace_bytes": (c_i64, [c_int, c_int, c_int, c_int, c_i64]),
    "read_gather_backward_det": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_int, c_i64, c_vp, c_vp, c_vp]),
    "read_gather_backward_sparse_det": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_int, c_i64, c_vp, c_vp, c_vp, c_vp]),
    "read_gate_det_workspace_bytes": (c_i64, [c_int, c_int]),
    "read_gate_backward_det": (c_int, [c_vp, c_vp, c_i64, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                       c_vp, c_vp]),
    "read_bn_backward_reduce_det": (c_int, [c_vp, c_vp, c_i64, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "read_gate_backward_batch_stats_det": (c_int, [c_vp, c_vp, c_i64, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                                   c_vp, c_vp, c_vp, c_vp]),
    "read_bn_backward_reduce_items_det": (c_int, [c_vp, c_vp, c_int, c_i64, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                                  c_vp]),
    "read_gate_backward_batch_stats_items_det": (c_int, [c_vp, c_vp, c_int, c_i64, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                                         c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "read_conv_wgrad_det_workspace_bytes": (c_i64, [c_int, c_int, c_int, c_int, c_int, c_int, c_int]),
    "read_conv_wgrad_det": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp,
                                    c_vp]),
    "read_conv_tc_supported": (c_int, [ctypes.POINTER(ReadConvDesc)]),
    "read_conv_tcg_supported": (c_int, [ctypes.POINTER(ReadConvDesc)]),
    "read_tcg_weight_elems": (c_i64, [c_int, c_int, c_int]),
    "read_pack_weights_tcg": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_vp, c_vp]),
    "read_conv_plan_create": (c_int, [ctypes.POINTER(ReadConvDesc), ctypes.POINTER(c_vp)]),
    "read_conv_plan_launch": (c_int, [c_vp, c_vp]),
    "read_conv_plan_impl": (c_int, [c_vp]),
    "read_conv_plan_set_max_ctas": (c_int, [c_vp, c_int]),
    "read_conv_plan_set_tile_order": (c_int, [c_vp, c_int]),
    "read_conv_plan_destroy": (None, [c_vp]),
    "read_upsample_bilinear4": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp]),
    "read_frame_to_rgba": (c_int, [c_vp, c_int, c_int, c_int, ctypes.c_float, c_vp, c_vp]),
    "read_point_view": (c_int, [c_vp, c_int, c_int, ctypes.POINTER(ReadPointViewDesc), c_vp, c_vp]),
    "read_nchw_f32_to_nhwc": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp]),
    "read_nhwc_to_nchw_f32": (c_int, [c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_vp]),
    "read_launch_count": (c_i64, []),
}
# int32 index maps (clouds of more than 2^24 + 1 points): each float entry point's twin is bound like it (the map is a pointer)
for _name in ("read_zbuf_resolve", "read_gather_from_index", "read_gather_from_index_items", "read_gather_backward",
              "read_gather_backward_sparse", "read_gather_backward_items", "read_gather_backward_sparse_items",
              "read_gather_backward_det", "read_gather_backward_sparse_det", "read_gather_backward_items_det",
              "read_gather_backward_sparse_items_det"):
    _SIGS[_name + "_i32"] = _SIGS[_name]

EXPORTS = tuple(sorted(_SIGS))
_lib = None


def load():
    """Load libread_b200.so (built by ``python -m read_b200.build`` / ``__graft_entry__.build()``)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"read_b200: CUDA library not built ({LIB_PATH} missing). Run `python -m read_b200.build`. "
            "There is no CPU fallback.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in _SIGS.items():
        fn = getattr(lib, name)          # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    # READ_B200_OPTIONS="name=value,name=value": tuning options (read_set_option, INTEGRATION.md section 3) applied at load time
    for item in filter(None, os.environ.get("READ_B200_OPTIONS", "").split(",")):
        name, _, value = item.partition("=")
        if lib.read_set_option(name.strip().encode(), int(value)) != 0:
            raise RuntimeError(f"read_b200: READ_B200_OPTIONS: unknown option {name!r}")
    return lib


def check(rc):
    if rc != 0:
        msg = load().read_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"read_b200: {msg} (code {rc})")


_device_checked = set()


def require_device(device_index=None):
    """Raise unless torch sees a CUDA device of compute capability 9.0 (H100): the kernels are built for sm_90a only."""
    import torch
    if not torch.cuda.is_available():
        raise RuntimeError("read_b200: no CUDA device; this package has no CPU fallback")
    idx = torch.cuda.current_device() if device_index is None else device_index
    if idx in _device_checked:
        return
    major, minor = torch.cuda.get_device_capability(idx)
    if (major, minor) != (9, 0):
        raise RuntimeError(f"read_b200: kernels are built for sm_90a only, device {idx} is sm_{major}{minor}")
    _device_checked.add(idx)


def stream_ptr():
    import torch
    return torch.cuda.current_stream().cuda_stream


def ptr(t):
    return None if t is None else t.data_ptr()
