"""ctypes binding of the C ABI in include/lanefit_b200.h.

The shared library is built in-tree (``python -m lanedetection_end2end_b200.csrc.build``
or ``__graft_entry__.build()``) as ``lanedetection_end2end_b200/liblanefit_b200.so``.
There is NO fallback: if the library is missing, every device op raises.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "liblanefit_b200.so")

LF_OK = 0
LF_F32, LF_BF16 = 0, 1
ACT_IDS = {"none": 0, "square": 1, "abs": 2, "relu": 3, "sigmoid": 4, "softplus": 5}
SOLVER_INVERSE, SOLVER_CHOLESKY = 0, 1
STATUS_SINGULAR, STATUS_NONFINITE, STATUS_NOT_POSDEF = 1, 2, 4
MAX_ORDER = 4
PACK_INDEX_MASK, PACK_TF32_HI, PACK_TF32_LO = 0x1fffffff, 0x20000000, 0x40000000   # LfPackJob index flags

_c_void_p = ctypes.c_void_p
_c_int = ctypes.c_int
_c_double = ctypes.c_double
_c_float = ctypes.c_float
_c_size_t = ctypes.c_size_t

# name -> (restype, argtypes); every symbol include/lanefit_b200.h declares
PROTOTYPES = {
    "lf_version": (_c_int, []),
    "lf_set_pdl": (None, [_c_int]),
    "lf_get_pdl": (_c_int, []),
    "lf_error_string": (ctypes.c_char_p, [_c_int]),
    "lf_last_cuda_error": (ctypes.c_char_p, []),
    "lf_lsq_workspace_bytes": (_c_size_t, [_c_int] * 5),
    "lf_lsq_fwd": (_c_int, [_c_void_p, _c_int, _c_void_p, _c_void_p, _c_void_p,
                            _c_int, _c_int, _c_int, _c_int, _c_int, _c_int, _c_int, _c_double, _c_int,
                            _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_size_t, _c_void_p]),
    "lf_lsq_bwd": (_c_int, [_c_void_p, _c_int, _c_void_p, _c_void_p, _c_void_p,
                            _c_int, _c_int, _c_int, _c_int, _c_int, _c_int, _c_int,
                            _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p]),
    "lf_lsq_plan": (_c_int, [_c_int] * 11 + [_c_void_p]),
}
LSQ_PLAN_INFO = 7       # LF_LSQ_PLAN_INFO: entries lf_lsq_plan fills
LSQ_PLAN_FIELDS = ("rowsep", "act_t", "nl", "groups", "nchunks", "ctas_per_sm", "align")

MAX_TAPS = 9

_i = ctypes.c_int
_p = ctypes.c_void_p


class LfConvArgs(ctypes.Structure):
    _fields_ = [("inp", _p), ("wmat", _p), ("bias", _p), ("out", _p), ("mask_src", _p), ("add_src", _p),
                ("add_mask", _p),
                ("N", _i), ("Hin", _i), ("Win", _i), ("Cin", _i), ("in_cstride", _i),
                ("Hout", _i), ("Wout", _i), ("out_cstride", _i), ("out_coff", _i), ("Cout", _i), ("CoutPad", _i),
                ("Hs", _i), ("Ws", _i), ("osy", _i), ("osx", _i), ("oy0", _i), ("ox0", _i), ("isy", _i), ("isx", _i),
                ("ntaps", _i), ("dy", _i * MAX_TAPS), ("dx", _i * MAX_TAPS), ("wtap", _i * MAX_TAPS),
                ("relu", _i)]


class LfConvTcArgs(ctypes.Structure):
    _fields_ = [("inp", _p), ("wpack", _p), ("bias", _p), ("out", _p), ("mask_src", _p), ("add_src", _p),
                ("add_mask", _p), ("colsum_partial", _p), ("stats_partial", _p), ("mask_scale", _p), ("mask_shift", _p), ("N", _i), ("H", _i), ("W", _i), ("C", _i), ("dy", _i * 3),
                ("dx", _i * 3), ("relu", _i), ("in_dtype", _i), ("out_dtype", _i), ("mask_dtype", _i)]


TC_PLAN_INFO = 12       # LF_TC_PLAN_INFO: entries lf_conv1d_tc_plan fills
TC_PLAN_FIELDS = ("slab", "res", "stages", "n_lo", "lo_stg", "lo_bytes", "TA", "TB", "vertical", "m_ctas", "smem_bytes",
                  "a_bytes")


class LfConvTcFp8Args(ctypes.Structure):
    _fields_ = [("conv", LfConvTcArgs), ("x_amax", _p), ("w_scale", _p), ("out_amax", _p)]


class LfWgradArgs(ctypes.Structure):
    _fields_ = [("P", _p), ("Q", _p), ("partial", _p), ("qsum_partial", _p),
                ("N", _i), ("Hs", _i), ("Ws", _i),
                ("Hp", _i), ("Wp", _i), ("Cp", _i), ("p_cstride", _i), ("p_coff", _i), ("psy", _i), ("psx", _i),
                ("Hq", _i), ("Wq", _i), ("Cq", _i), ("q_cstride", _i), ("q_coff", _i), ("qsy", _i), ("qsx", _i),
                ("ntaps", _i), ("pdy", _i * MAX_TAPS), ("pdx", _i * MAX_TAPS), ("qdy", _i * MAX_TAPS),
                ("qdx", _i * MAX_TAPS),
                ("CpPad", _i), ("CqPad", _i), ("nsplit", _i)]


TCG_MAX_TAPS = 9
_ll = ctypes.c_longlong


class LfTcgView(ctypes.Structure):
    _fields_ = [("ptr", _p), ("H", _i), ("W", _i), ("sn", _ll), ("sy", _ll), ("sx", _ll)]


class LfConvTcgArgs(ctypes.Structure):
    _fields_ = [("a", LfTcgView * 2), ("wg", _p), ("bias", _p), ("out", _p), ("osn", _ll), ("osy", _ll), ("osx", _ll),
                ("oy_mul", _i), ("oy0", _i), ("N", _i), ("Hs", _i), ("Ws", _i), ("Kc", _i), ("Ng", _i), ("ntaps", _i),
                ("map", _i * TCG_MAX_TAPS), ("dy", _i * TCG_MAX_TAPS), ("dx", _i * TCG_MAX_TAPS), ("precision", _i), ("relu", _i)]


REDUCE_MAX_JOBS = 8


class LfReduceJob(ctypes.Structure):
    _fields_ = [("partial", _p), ("dst", _p), ("nsplit", _i), ("ntaps", _i), ("Cp", _i), ("Cq", _i), ("CpPad", _i),
                ("CqPad", _i), ("st", _i), ("sp", _i), ("sq", _i)]


WGRAD_TCG_MAX_BLOCKS = 24


class LfWgradTcgArgs(ctypes.Structure):
    _fields_ = [("a", LfTcgView * 2), ("b", LfTcgView), ("partial", _p), ("N", _i), ("Hs", _i), ("Ws", _i), ("Ka", _i),
                ("Nn", _i), ("nblocks", _i), ("map", _i * WGRAD_TCG_MAX_BLOCKS), ("dy", _i * WGRAD_TCG_MAX_BLOCKS),
                ("dx", _i * WGRAD_TCG_MAX_BLOCKS), ("cblk", _i * WGRAD_TCG_MAX_BLOCKS), ("nctas", _i), ("precision", _i),
                ("a_dtype", _i)]


OPTIM_ADAM, OPTIM_SGD, OPTIM_RMSPROP = 0, 1, 2
OPTIM_CHUNK = 2048


class LfOptimSeg(ctypes.Structure):
    _fields_ = [("param", _p), ("grad", _p), ("state0", _p), ("state1", _p), ("numel", _ll), ("chunk0", _ll)]


class LfOptimHyper(ctypes.Structure):
    _fields_ = [("lr", _c_double), ("beta1", _c_double), ("beta2", _c_double), ("eps", _c_double),
                ("weight_decay", _c_double), ("momentum", _c_double)]


class LfOptimState(ctypes.Structure):
    _fields_ = [("step", _ll), ("skipped", _ll), ("ticket", ctypes.c_ulonglong)]


OPTIM_PP_SCALAR_BYTES = 48


class LfOptimSegPP(ctypes.Structure):
    _fields_ = [("seg", LfOptimSeg), ("slot", _i), ("reserved", _i)]


class LfGradClip(ctypes.Structure):
    _fields_ = [("max_norm", _c_float), ("total_norm", _c_float), ("clip_coef", _c_float), ("nonfinite", _i),
                ("nonfinite_skipped", _ll), ("ticket", ctypes.c_ulonglong)]


STATUS_JPEG_CORRUPT = 8
JPEG_PIECE_BYTES = 128
JPEG_MAX_BPM = 6


class LfJpegHuff(ctypes.Structure):
    _fields_ = [("look", ctypes.c_ushort * 512), ("maxcode", _i * 18), ("valoff", _i * 18), ("val", ctypes.c_ubyte * 256)]


class LfJpegImage(ctypes.Structure):
    _fields_ = [("ecs_off", _ll), ("ecs_len", _i), ("W", _i), ("H", _i), ("ncomp", _i), ("mcux", _i), ("mcuy", _i), ("bpm", _i),
                ("restart", _i), ("nint", _i), ("hs", _i * 3), ("vs", _i * 3), ("comp_w", _i * 3), ("comp_h", _i * 3),
                ("qtab", _i * 3), ("blk_comp", _i * JPEG_MAX_BPM), ("blk_dx", _i * JPEG_MAX_BPM), ("blk_dy", _i * JPEG_MAX_BPM),
                ("blk_dc", _i * JPEG_MAX_BPM), ("blk_ac", _i * JPEG_MAX_BPM),
                ("stream_off", _ll), ("x_off", _ll), ("b_off", _ll), ("us_off", _ll), ("pb_off", _ll), ("plane_off", _ll * 3),
                ("block_off", _ll), ("plane_stride", _i * 3), ("npieces_max", _i), ("qt", (ctypes.c_ushort * 64) * 4),
                ("dc", LfJpegHuff * 4), ("ac", LfJpegHuff * 4)]


STATUS_PNG_CORRUPT = 16


class LfPngImage(ctypes.Structure):
    _fields_ = [("zoff", _ll), ("zlen", _i), ("W", _i), ("H", _i), ("depth", _i), ("rowbytes", _i), ("reserved", _i),
                ("raw_off", _ll)]


TUSIMPLE_MAX_GT = 8
TUSIMPLE_MAX_S = 64
DRAW_MAX_LANES, DRAW_MAX_RADIUS = 8, 16
LOADER_LANES, LOADER_POINTS = 4, 56
LOADER_BEV_COEFFS = 3

_NET_PROTOS = {
    "lf_loader_stage": (_i, [_p, _p, _i, _i, _i, _i, _i, _p, _p, _i, _p, _p, _i, _p, _p, _i, _i, _p, _p, _p, _p]),
    "lf_loader_assemble": (_i, [_p, _p, _i, _i, _i, _i, _p, _i, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "lf_loader_label_rows": (_i, [_p, _i, _i, _i, _p, _p, _p, _p]),
    "lf_loader_assemble_bev": (_i, [_p, _p, _i, _i, _i, _p, _i, _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "lf_tusimple_score": (_i, [_p, _p, _p, _i, _i, _i, _p, _p, _p, _i, _i, _p, _p, _p, _p]),
    "lf_bev_lane_score": (_i, [_p, _p, _p, _p, _i, _i, _p, _p, _p, _p, _p, _p, _i, _i, _ll, _p, _p, _p, _p]),
    "lf_png_workspace_bytes": (_c_size_t, [_p, _i]),
    "lf_png_decode": (_i, [_p, _i, _i, _i, _p, _p, _p, _c_size_t, _p]),
    "lf_label_preprocess": (_i, [_p, _i, _i, _i, _i, _p, _p, _i, _i, _i, _p, _p, _p]),
    "lf_jpeg_workspace_bytes": (_c_size_t, [_p, _i, _p]),
    "lf_jpeg_decode": (_i, [_p, _i, _i, _i, _p, _p, _p, _c_size_t, _p, _c_size_t, _p]),
    "lf_jpeg_quality_tables": (_i, [_i, _i, _p]),
    "lf_jpeg_encode_bound": (_ll, [_i, _i, _i, _i]),
    "lf_jpeg_encode_workspace_bytes": (_c_size_t, [_i, _i, _i, _i, _i]),
    "lf_jpeg_encode": (_i, [_p, _i, _i, _i, _i, _i, _p, _p, _ll, _p, _p, _p]),
    "lf_draw_lane_points": (_i, [_p, _i, _i, _i, _p, _i, _i, _p, _p, _i, _p]),
    "lf_optim_step": (_i, [_i, _p, _i, _ll, _p, _p, _p, _p]),
    "lf_optim_step_pp": (_i, [_i, _p, _p, _i, _ll, _p, _p, _i, _p, _p, _p, _p]),
    "lf_grad_norm_workspace_bytes": (_c_size_t, [_ll]),
    "lf_grad_norm": (_i, [_p, _i, _ll, _p, _p, _c_size_t, _p]),
    "lf_grad_norm_pp": (_i, [_p, _i, _ll, _p, _p, _c_size_t, _p]),
    "lf_optim_step_clip": (_i, [_i, _p, _i, _ll, _p, _p, _p, _p, _p]),
    "lf_optim_step_pp_clip": (_i, [_i, _p, _p, _i, _ll, _p, _p, _i, _p, _p, _p, _p, _p]),
    "lf_wgrad_tcg_ctas": (_i, [_i, _i, _i, _i, _i, _i, _i]),
    "lf_wgrad_tcg": (_i, [ctypes.POINTER(LfWgradTcgArgs), _p]),
    "lf_reduce_multi": (_i, [ctypes.POINTER(LfReduceJob), _i, _p]),
    "lf_conv_tcg_supported": (_i, [_i, _i, _i, _i, _i]),
    "lf_conv_tcg": (_i, [ctypes.POINTER(LfConvTcgArgs), _p]),
    "lf_conv_f32": (_i, [ctypes.POINTER(LfConvArgs), _p]),
    "lf_wgrad_f32": (_i, [ctypes.POINTER(LfWgradArgs), _p]),
    "lf_wgrad_f32_nsplit": (_i, [ctypes.POINTER(LfWgradArgs)]),
    "lf_conv1d_tc": (_i, [ctypes.POINTER(LfConvTcArgs), _p]),
    "lf_conv1d_tc_supported": (_i, [_i, _i, _i, _i]),
    "lf_conv1d_tc_x3": (_i, [ctypes.POINTER(LfConvTcArgs), _p]),
    "lf_conv1d_tc_bf16": (_i, [ctypes.POINTER(LfConvTcArgs), _p]),
    "lf_conv1d_tc_fp8": (_i, [ctypes.POINTER(LfConvTcFp8Args), _p]),
    "lf_amax_per_image": (_i, [_p, _i, ctypes.c_longlong, _i, _p, _p]),
    "lf_conv1d_tc_x3_rows": (_i, [_i, _i, _i, _i, _i, _i]),
    "lf_conv1d_tc_set_variant": (None, [_i]),
    "lf_conv1d_tc_slab_ok": (_i, [_i, _i, _i, _i, _i, _i]),
    "lf_conv1d_tc_plan": (_i, [_i, _i, _i, _i, _i, _i, _p, _p, _p]),
    "lf_wgrad_reduce": (_i, [_p, _i, _i, _i, _i, _i, _i, _p, _i, _i, _i, _p]),
    "lf_vec_reduce": (_i, [_p, _i, _i, _i, _p, _p]),
    "lf_colsum_blocks": (_i, [ctypes.c_longlong]),
    "lf_colsum": (_i, [_p, ctypes.c_longlong, _i, _i, _i, _p, _i, _p]),
    "lf_maxpool2_fwd": (_i, [_p, _i, _i, _i, _i, _i, _p, _i, _i, _p]),
    "lf_maxpool2_affine_relu": (_i, [_p, _i, _i, _i, _i, _i, _p, _p, _p, _i, _i, _p]),
    "lf_maxpool2_bwd": (_i, [_p, _i, _i, _i, _i, _i, _p, _i, _i, _p, _i, _i, _p]),
    "lf_bn_blocks": (_i, [ctypes.c_longlong, _i]),
    "lf_bn_stats": (_i, [_p, ctypes.c_longlong, _i, _p, _p]),
    "lf_bn_finalize": (_i, [_p, _i, ctypes.c_longlong, _i, _p, _p, ctypes.c_float, ctypes.c_float, _p, _p, _p, _p, _p,
                            _p, _p]),
    "lf_bn_eval_prepare": (_i, [_i, _p, _p, ctypes.c_float, _p, _p, _p, _p, _p]),
    "lf_bn_apply": (_i, [_p, ctypes.c_longlong, _i, _i, _p, _p, _p, _p, _i, _p, _p]),
    "lf_bn_apply_bf16": (_i, [_p, ctypes.c_longlong, _i, _i, _p, _p, _p, _p, _i, _p, _p]),
    "lf_bn_bwd_reduce": (_i, [_p, _p, _p, _p, ctypes.c_longlong, _i, _i, _p, _p, _p, _p]),
    "lf_bn_bwd_finalize": (_i, [_p, _i, ctypes.c_longlong, _i, _p, _p, _p, _p, _p]),
    "lf_bn_bwd_apply": (_i, [_p, _p, _p, _p, ctypes.c_longlong, _i, _i, _p, _p, _p, _p, _p, _p, _p]),
    "lf_bn_bwd_apply_gated": (_i, [_p, _p, _p, _p, ctypes.c_longlong, _i, _i, _p, _p, _p, _p, _p, _p, _p, _p]),
    "lf_outconv_fwd": (_i, [_p, _p, _p, _i, _i, _i, _i, _i, _p, _p]),
    "lf_outconv_bwd_data": (_i, [_p, _p, _i, _i, _i, _i, _i, _p, _p]),
    "lf_outconv_wgrad_blocks": (_i, [ctypes.c_longlong]),
    "lf_outconv_bwd_weight": (_i, [_p, _p, _i, _i, _i, _i, _i, _p, _p]),
    "lf_nchw_to_nhwc_pad": (_i, [_p, _i, _i, _i, _i, _i, _p, _p]),
    "lf_nhwc_to_nchw": (_i, [_p, _i, _i, _i, _i, _p, _p]),
    "lf_nchw_to_nhwc": (_i, [_p, _i, _i, _i, _i, _p, _p]),
    "lf_pack_gather": (_i, [_p, _i, _i, _p]),
    "lf_backproj_loss": (_i, [_p, _p, _p, _p, _p, _p, _i, _i, _i, _p, _p, _p, _p, _p, _p]),
    "lf_backproj_loss_host": (_i, [_p, _p, _p, _p, _p, _p, _i, _i, _i, _p, _p, _p, _p]),
    "lf_backproj_loss_dev": (_i, [_p, _p, _p, _p, _p, _i, _i, _i, _p, _p, _p, _p, _p, _p, _p, _p]),
    "lf_backproj_loss_dev_host": (_i, [_p, _p, _p, _p, _p, _i, _i, _i, _p, _p, _p, _p, _p]),
    "lf_lsq_fwd_rowsums": (_i, [_p, _i, _p, _p, _i, _i, _i, _i, _i, _i, _i, ctypes.c_double, _i, _p, _p, _p, _p, _p, _p,
                                ctypes.c_size_t, _p]),
    "lf_lsq_grid_grad": (_i, [_p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _p, _p]),
    "lf_lsq_fwd_keep": (_i, [_p, _i, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, ctypes.c_double, _i, _p, _p, _p, _p, _p,
                             ctypes.c_size_t, _p]),
    "lf_lsq_fwd_rowsums_keep": (_i, [_p, _i, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, ctypes.c_double, _i, _p, _p, _p, _p,
                                     _p, _p, ctypes.c_size_t, _p]),
    "lf_lsq_bwd_keep": (_i, [_p, _i, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _p, _p, _p, _p, _p]),
    "lf_homography_tables": (_i, [_p, _i, _i, ctypes.c_double, _p, _p, _p, _p, _p, _p, _p, _p]),
    "lf_homography_bwd": (_i, [_p, _i, _i, _p, _p, _p, _p, _p]),
    "lf_homography_host": (_i, [_p, _i, _p, _p, _p]),
    "lf_homography_bwd_host": (_i, [_p, _i, _i, _p, _p, _p, _p]),
    "lf_predicted_homography_tables": (_i, [_p, _i, _i, _i, ctypes.c_double, _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "lf_predicted_homography_bwd": (_i, [_p, _i, _i, _i, _p, _p, _p, _p, _p]),
    "lf_predicted_homography_host": (_i, [_p, _i, _p, _p, _p]),
    "lf_predicted_homography_bwd_host": (_i, [_p, _i, _i, _p, _p, _p, _p]),
    "lf_predicted_homography_source_tables": (_i, [_p, _i, _i, _i, ctypes.c_double, _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "lf_predicted_homography_source_bwd": (_i, [_p, _i, _i, _i, _p, _p, _p, _p, _p, _p]),
    "lf_predicted_homography_source_host": (_i, [_p, _i, _p, _p, _p, _p]),
    "lf_predicted_homography_source_bwd_host": (_i, [_p, _i, _i, _p, _p, _p, _p, _p]),
    "lf_lsq_fwd_per_image": (_i, [_p, _i, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, ctypes.c_double, _i, _p, _p, _p, _p, _p,
                                  _p, ctypes.c_size_t, _p]),
    "lf_lsq_bwd_per_image": (_i, [_p, _i, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _p, _p, _p, _p, _p]),
    "lf_lsq_grid_grad_per_image": (_i, [_p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _p, _p]),
    # prefix fits of a lane curriculum: the entry point's arguments with Lmap after L
    "lf_lsq_fwd_lanes": (_i, [_p, _i, _p, _p, _p] + [_i] * 8 + [ctypes.c_double, _i, _p, _p, _p, _p, _p, ctypes.c_size_t,
                                                                 _p]),
    "lf_lsq_fwd_keep_lanes": (_i, [_p, _i, _p, _p, _p, _p] + [_i] * 8 + [ctypes.c_double, _i, _p, _p, _p, _p, _p,
                                                                         ctypes.c_size_t, _p]),
    "lf_lsq_fwd_rowsums_lanes": (_i, [_p, _i, _p, _p] + [_i] * 8 + [ctypes.c_double, _i, _p, _p, _p, _p, _p, _p,
                                                                    ctypes.c_size_t, _p]),
    "lf_lsq_fwd_rowsums_keep_lanes": (_i, [_p, _i, _p, _p, _p] + [_i] * 8 + [ctypes.c_double, _i, _p, _p, _p, _p, _p, _p,
                                                                             ctypes.c_size_t, _p]),
    "lf_lsq_bwd_lanes": (_i, [_p, _i, _p, _p, _p] + [_i] * 8 + [_p, _p, _p, _p, _p]),
    "lf_lsq_bwd_keep_lanes": (_i, [_p, _i, _p, _p, _p, _p] + [_i] * 8 + [_p, _p, _p, _p, _p]),
    "lf_lsq_fwd_per_image_lanes": (_i, [_p, _i, _p, _p, _p] + [_i] * 8 + [ctypes.c_double, _i, _p, _p, _p, _p, _p, _p,
                                                                          ctypes.c_size_t, _p]),
    "lf_lsq_bwd_per_image_lanes": (_i, [_p, _i, _p, _p, _p] + [_i] * 8 + [_p, _p, _p, _p, _p]),
    "lf_backproj_loss_per_image_scratch": (ctypes.c_size_t, [_i, _i]),
    "lf_backproj_loss_per_image": (_i, [_p, _p, _p, _p, _p, _i, _i, _i, _p, _p, _p, _p, _p, _p, _p, _p]),
    "lf_area_loss": (_i, [_p, _p, _i, _i, _i, _p, _p, _p, _p, _p]),
    "lf_area_loss_host": (_i, [_p, _p, _i, _i, _i, _p, _p, _p, _p]),
    "lf_seg_lane_maps": (_i, [_p, _i, _i, _i, _i, _i, _i, _p, _p]),
    "lf_seg_lane_maps_line": (_i, [_p, _i, _i, _i, _i, _i, _i, _p, _p, _p]),
    "lf_ce2d_blocks": (_i, [_i, _i, _i]),
    "lf_ce2d_fwd": (_i, [_p, _p, _p, _i, _i, _i, _i, _p, _p, _p, _p]),
    "lf_ce2d_bwd": (_i, [_p, _p, _p, _i, _i, _i, _i, _p, _p, _p, _p]),
    "lf_seg_confusion": (_i, [_p, _p, _i, _i, _i, _i, _p, _p, _p]),
    "lf_frame_preprocess": (_i, [_p, _i, _i, _i, _i, _i, _p, _p, _i, _p, _p, _i, _i, _i, _p, _i, _p, _p]),
    "lf_linear_chunks": (_i, [_i]),
    "lf_rowmean_fwd": (_i, [_p, _i, _i, _i, _i, _p, _p]),
    "lf_rowmean_bwd": (_i, [_p, _i, _i, _i, _i, _p, _p]),
    "lf_linear_fwd": (_i, [_p, _p, _p, _i, _i, _i, _i, _p, _p, _p]),
    "lf_linear_bwd_data": (_i, [_p, _p, _p, _i, _i, _i, _p, _p]),
    "lf_linear_bwd_weight": (_i, [_p, _p, _p, _i, _i, _i, _p, _p, _p]),
    "lf_bn_bwd_finalize_sx": (_i, [_p, _i, ctypes.c_longlong, _i, _i, _p, _p, _p, _p, _p, _p, _p]),
    "lf_bn_collapse": (_i, [_p, _i, _i, _i, ctypes.c_longlong, _p, _p, _p]),
    "lf_bn_finalize_tot": (_i, [_p, _i, _p, _p, ctypes.c_float, ctypes.c_float, _p, _p, _p, _p, _p, _p, _p]),
    "lf_bn_bwd_finalize_tot": (_i, [_p, _p, _p, _i, _p, _p, _p, _p, _p]),
    "lf_bn_bwd_finalize_sx_tot": (_i, [_p, _p, _p, _i, _p, _p, _p, _p, _p, _p, _p]),
}
PROTOTYPES.update(_NET_PROTOS)


_lib = None


class LanefitError(RuntimeError):
    pass


def lib():
    """Load (once) and return the ctypes handle; raises if the library was not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise LanefitError(
                "liblanefit_b200.so not found at %s -- build it with "
                "`python -m lanedetection_end2end_b200.csrc.build` (there is no CPU/eager fallback)" % LIB_PATH)
        h = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in PROTOTYPES.items():
            fn = getattr(h, name)   # AttributeError if the .so is stale
            fn.restype = res
            fn.argtypes = args
        _lib = h
    return _lib


def check(rc, what):
    if rc != LF_OK:
        h = lib()
        msg = h.lf_error_string(rc).decode()
        if rc == -4:
            msg += ": " + h.lf_last_cuda_error().decode()
        raise LanefitError("%s failed: %s (code %d)" % (what, msg, rc))


LAUNCHES = 0          # kernels launched through the C ABI since import (every call below = 1 launch)
TRACE = None          # set to a list to record (label, start_event, end_event, flops, bytes) per launch


def call(name, *args, flops=0, nbytes=0, label=None):
    """Invoke one launching entry point: counts it, optionally brackets it with CUDA events on
    the current stream (bench.py's per-kernel roofline), and raises on a non-zero return.
    label: the name the launch is traced under (default: the entry point's)."""
    global LAUNCHES
    fn = getattr(lib(), name)
    if TRACE is None:
        rc = fn(*args)
    else:
        import torch
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        rc = fn(*args)
        e1.record()
        TRACE.append((label or name, e0, e1, flops, nbytes))
    LAUNCHES += 1
    check(rc, name)


def ptr(t):
    """Device pointer of a tensor (or None)."""
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def stream_ptr():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def dtype_id(t):
    import torch
    if t.dtype == torch.float32:
        return LF_F32
    if t.dtype == torch.bfloat16:
        return LF_BF16
    raise LanefitError("unsupported dtype %s (float32 or bfloat16 expected)" % t.dtype)


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise LanefitError(
                "lanedetection_end2end_b200 runs on CUDA (sm_90a) only; got a %s tensor. "
                "There is no CPU fallback by design." % t.device)
