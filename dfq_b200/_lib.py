"""ctypes binding of libdfq_sm90.so (the C ABI declared in include/dfq_b200.h).

There is no CPU fallback: if the library is missing and cannot be built, or a call fails, this module
raises.  The descriptor structs mirror include/dfq_b200.h field for field (numpy structured dtypes
with C alignment, so whole tables are passed as one pointer).
"""
from __future__ import annotations

import contextlib
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("DFQ_LIB") or os.path.join(_HERE, "libdfq_sm90.so")   # DFQ_LIB: a tuning build

ABI_VERSION = 11


LAYER_COLS_READY = 1   # DfqLayer.flags
LAYER_FOLD_PENDING = 2
LAYER_ROWS_READY = 4
ROWS_FULL, ROWS_STREAMED, ROWS_UNDECIDED, ROWS_HOST_FULL = 0, 1, 2, 3   # DfqCleResult.rows_streamed
FOLD_FULL, FOLD_DEFER, FOLD_APPLY = 0, 1, 2   # DfqFold.mode
BC_PREPARED = 4        # DfqBcLayer.flags


class DfqError(RuntimeError):
    pass


# ---- struct mirrors -------------------------------------------------------------------------------
LAYER_DT = np.dtype([
    ("w_off", np.int64), ("bias_off", np.int64),
    ("rows", np.int32), ("cols", np.int32), ("kk", np.int32),
    ("rel_in", np.int32), ("rel_out", np.int32), ("col_mode", np.int32), ("group", np.int32), ("flags", np.int32),
    ("cmin_off", np.int64), ("cmax_off", np.int64), ("fold_off", np.int64), ("rext_off", np.int64),
    ("rext_rows", np.int32), ("_pad", np.int32),
], align=True)

RELATION_DT = np.dtype([
    ("first", np.int32), ("second", np.int32), ("channels", np.int32),
    ("groups", np.int32), ("gi", np.int32), ("go", np.int32),
    ("bn_w_off", np.int64), ("bn_b_off", np.int64),
    ("s_acc_off", np.int64), ("s_step_off", np.int64), ("inv_off", np.int64),
], align=True)

CLE_PARAMS_DT = np.dtype([
    ("s_lo", np.float32), ("s_hi", np.float32), ("inv_lo", np.float32), ("inv_hi", np.float32),
    ("eps", np.float32), ("signed_mode", np.int32),
    ("converge_thres", np.float64), ("converge_count", np.int32), ("max_sweeps", np.int32),
    ("apply_only", np.int32), ("_pad", np.int32),
], align=True)

CLE_RESULT_DT = np.dtype([
    ("n_sweeps", np.int32), ("converged", np.int32), ("last_diff", np.float64),
    ("diffs", np.float64, (64,)), ("fused_sweeps", np.int32), ("bc_prepared", np.int32),
    ("rows_streamed", np.int32), ("_pad", np.int32),
], align=True)

FOLD_DT = np.dtype([
    ("layer", np.int32), ("bn_eps", np.float32),
    ("gamma_off", np.int64), ("beta_off", np.int64), ("mean_off", np.int64), ("var_off", np.int64),
    ("fake_w_off", np.int64), ("fake_b_off", np.int64),
    ("scan_go", np.int32), ("scan_gi", np.int32), ("mode", np.int32), ("scan_rows", np.int32), ("fac_off", np.int64),
    ("row_prefix", np.int32), ("_pad", np.int32),
], align=True)

TERM_DT = np.dtype([
    ("bn_w_off", np.int64), ("bn_b_off", np.int64),
    ("n", np.int32), ("relu", np.int32), ("dst_off", np.int32), ("accumulate", np.int32),
], align=True)

BC_LAYER_DT = np.dtype([
    ("layer", np.int32), ("signed_mode", np.int32), ("term_begin", np.int32), ("term_end", np.int32),
    ("expect_len", np.int32), ("flags", np.int32),
    ("expect_off", np.int64), ("delta_off", np.int64), ("next_bn_b_off", np.int64), ("minmax_off", np.int64),
    ("colmin_off", np.int64), ("colmax_off", np.int64), ("n_col", np.int32), ("_pad", np.int32),
], align=True)

QUANT_TASK_DT = np.dtype([
    ("off", np.int64), ("n", np.int64), ("num_bits", np.int32), ("symmetric", np.int32),
    ("minmax_off", np.int64),
], align=True)

I8_CONV_DT = np.dtype([(f, np.int32) for f in (
    "N", "C", "H", "W", "O", "kh", "kw", "stride_h", "stride_w", "pad_h", "pad_w", "dil_h", "dil_w", "groups",
    "OH", "OW", "Cpad", "_pad")], align=True)

I8_EPILOGUE_DT = np.dtype([("residual", np.uint64), ("y", np.uint64), ("yq", np.uint64)] +
                          [(f, np.float32) for f in ("out_scale", "pre_lo", "pre_hi", "post_lo", "post_hi")], align=True)

I8_POOL_DT = np.dtype([(f, np.int32) for f in (
    "N", "C", "H", "W", "kh", "kw", "stride_h", "stride_w", "pad_h", "pad_w", "dil_h", "dil_w", "ceil_mode", "OH", "OW",
    "Cpad")], align=True)

I8_RESIZE_DT = np.dtype([(f, np.int32) for f in ("N", "C", "H", "W", "OH", "OW", "align_corners", "coff", "cstride")] +
                        [(f, np.float32) for f in ("out_scale", "lo", "hi")], align=True)

I8_AFFINE_DT = np.dtype([(f, np.float64) for f in ("kP", "kA", "kW", "kN")], align=True)

I8_AFFINE_EPILOGUE_DT = np.dtype([(f, np.uint64) for f in ("residual", "y", "yq", "S")] +
                                 [("out_min", np.float32), ("out_max", np.float32), ("out_bits", np.int32)] +
                                 [(f, np.float32) for f in ("pre_lo", "pre_hi", "post_lo", "post_hi")], align=True)

I8_AFFINE_OBSERVE_DT = np.dtype([("obs_min", np.float32), ("obs_max", np.float32), ("obs_bits", np.int32),
                                 ("res_min", np.float32), ("res_max", np.float32), ("res_bits", np.int32)], align=True)

I8_AFFINE_LAYOUT_DT = np.dtype([(f, np.int32) for f in ("coff", "cstride", "S_accumulate", "pad_code_on", "pad_code")],
                               align=True)

I8_AFFINE_RESIZE_DT = np.dtype([(f, np.int32) for f in ("N", "C", "H", "W", "OH", "OW", "align_corners", "coff", "cstride")] +
                               [("pre_lo", np.float32), ("pre_hi", np.float32), ("obs_min", np.float32),
                                ("obs_max", np.float32), ("obs_bits", np.int32), ("post_lo", np.float32),
                                ("post_hi", np.float32), ("out_min", np.float32), ("out_max", np.float32),
                                ("out_bits", np.int32)], align=True)

I8_AFFINE_ROWS_DT = np.dtype([("y", np.uint64), ("off", np.int64), ("img_stride", np.int64)] +
                             [(f, np.float32) for f in ("pre_lo", "pre_hi", "post_lo", "post_hi", "obs_min", "obs_max")] +
                             [("obs_bits", np.int32), ("tail_min", np.float32), ("tail_max", np.float32),
                              ("tail_bits", np.int32)], align=True)

SSD_NMS_DT = np.dtype([(f, np.int32) for f in ("N", "P", "C", "prior_batch")] +
                      [(f, np.float32) for f in ("center_variance", "size_variance", "prob_threshold", "iou_threshold")] +
                      [("candidate_size", np.int32), ("top_k", np.int32)], align=True)

SEG_ARGMAX_DT = np.dtype([(f, np.int32) for f in ("N", "C", "H", "W", "OH", "OW", "align_corners", "label_type")],
                         align=True)
SEG_LABEL_U8, SEG_LABEL_I64, SEG_LABEL_F32 = 0, 1, 2
# DfqSegArgmax is struct-size index 19, checked on its own: EXPECTED_SIZES stays the table of indices 0 .. 18
SEG_ARGMAX_INDEX, SEG_ARGMAX_SIZE = 19, 32

PRE_IMAGE_DT = np.dtype([(f, np.int64) for f in ("src", "label", "xtap", "ytap", "xnear", "ynear")] +
                        [(f, np.int32) for f in ("H", "W", "xk", "yk")], align=True)
PRE_RESAMPLE_DT = np.dtype([(f, np.int32) for f in ("n", "out_h", "out_w", "filter", "norm", "_pad")] +
                           [("blob_bytes", np.int64), ("mean", np.float32, (3,)), ("std", np.float32, (3,)),
                            ("mean64", np.float64, (3,)), ("std64", np.float64, (3,))], align=True)
PRE_PIL_BILINEAR, PRE_CV_LINEAR = 0, 1
PRE_NORM_F32, PRE_NORM_F64, PRE_NORM_SUB_DIV = 0, 1, 2
# struct-size indices of DfqPreImage and DfqPreResample, checked on their own like DfqSegArgmax's; index 20 stays -1
PRE_SIZES = {21: (PRE_IMAGE_DT, 64), 22: (PRE_RESAMPLE_DT, 104)}

JPEG_IMAGE_DT = np.dtype([("dst", np.int64), ("tables", np.int64)] +
                         [(f, np.int32) for f in ("H", "W", "ncomp", "hs", "vs", "mcux", "mcuy", "_pad")], align=True)
JPEG_SEGMENT_DT = np.dtype([("begin", np.int64), ("end", np.int64)] +
                           [(f, np.int32) for f in ("image", "mcu0", "mcus", "_pad")], align=True)
JPEG_DECODE_DT = np.dtype([("n", np.int32), ("nseg", np.int32), ("blob_bytes", np.int64), ("call", np.uint64)], align=True)
JPEG_HUFF_DT = np.dtype([("maxcode", np.int32, (18,)), ("valoff", np.int32, (18,)), ("look", np.uint16, (512,)),
                         ("vals", np.uint8, (256,))], align=True)
JPEG_TABLES_DT = np.dtype([("q", np.int32, (3, 64)), ("dc", JPEG_HUFF_DT, (3,)), ("ac", JPEG_HUFF_DT, (3,))], align=True)
JPEG_BAD_CODE, JPEG_BAD_RUN, JPEG_SHORT_SCAN = 1, 2, 4    # reason bits of dfq_jpeg_decode's error word
# struct-size indices of the JPEG decoder's structs, checked on their own like PRE_SIZES
JPEG_SIZES = {23: (JPEG_IMAGE_DT, 48), 24: (JPEG_SEGMENT_DT, 32), 25: (JPEG_DECODE_DT, 24), 26: (JPEG_HUFF_DT, 1424),
              27: (JPEG_TABLES_DT, 9312)}

PNG_IMAGE_DT = np.dtype([(f, np.int64) for f in ("src", "src_end", "work", "dst")] + [("H", np.int32), ("W", np.int32)],
                        align=True)
PNG_DECODE_DT = np.dtype([("n", np.int32), ("_pad", np.int32), ("blob_bytes", np.int64), ("call", np.uint64)], align=True)
# reason bits of dfq_png_decode's error word
PNG_BAD_BLOCK, PNG_BAD_CODESET, PNG_BAD_CODE, PNG_FAR, PNG_STORED_LEN, PNG_SHORT, PNG_BAD_FILTER, PNG_ADLER = \
    1, 2, 4, 8, 16, 32, 64, 128
# struct-size indices of the PNG decoder's structs, checked on their own like JPEG_SIZES
PNG_SIZES = {29: (PNG_IMAGE_DT, 40), 30: (PNG_DECODE_DT, 24)}

MAP_IGNORED, MAP_TP, MAP_FP = 0, 1, 2                  # verdicts of dfq_map_match
MAP_ERR_DET_LABEL, MAP_ERR_GT_LABEL, MAP_ERR_DET_OFFSETS, MAP_ERR_GT_OFFSETS = 1, 2, 4, 8   # its device error bits

# dfq_bias_correct_absorb_clip's relation table (include/dfq_b200.h), struct-size index 28
ABSORB_DT = np.dtype([("first", np.int32), ("second", np.int32), ("n", np.int32), ("_pad", np.int32),
                      ("bn_w_off", np.int64), ("bn_b_off", np.int64), ("c_off", np.int64)], align=True)
ABSORB_SIZES = {28: (ABSORB_DT, 40)}

# sizes the C side uses (checked in tests against sizeof via the header's layout rules)
EXPECTED_SIZES = {
    "DfqLayer": (LAYER_DT, 88), "DfqRelation": (RELATION_DT, 64), "DfqCleParams": (CLE_PARAMS_DT, 48),
    "DfqCleResult": (CLE_RESULT_DT, 544), "DfqFold": (FOLD_DT, 88), "DfqExpectTerm": (TERM_DT, 32),
    "DfqBcLayer": (BC_LAYER_DT, 80), "DfqQuantTask": (QUANT_TASK_DT, 32), "DfqI8Conv": (I8_CONV_DT, 72),
    "DfqI8Epilogue": (I8_EPILOGUE_DT, 48), "DfqI8Pool": (I8_POOL_DT, 64), "DfqI8Resize": (I8_RESIZE_DT, 48),
    "DfqI8Affine": (I8_AFFINE_DT, 32), "DfqI8AffineEpilogue": (I8_AFFINE_EPILOGUE_DT, 64),
    "DfqI8AffineObserve": (I8_AFFINE_OBSERVE_DT, 24), "DfqI8AffineLayout": (I8_AFFINE_LAYOUT_DT, 20),
    "DfqI8AffineResize": (I8_AFFINE_RESIZE_DT, 76), "DfqI8AffineRows": (I8_AFFINE_ROWS_DT, 64),
    "DfqSsdNms": (SSD_NMS_DT, 40),
}

_PF = C.c_void_p   # device float*


class _Momentum(object):
    """ctypes argument type of the EMA momentum, a C double since ABI 2.  A Python number is passed as is, so 1 - m is formed
    from the same double the reference uses; a c_float or c_double (what callers of ABI 1 pass) is widened exactly."""

    @classmethod
    def from_param(cls, v):
        return C.c_double(v.value if isinstance(v, (C.c_float, C.c_double)) else float(v))


_I64 = C.c_int64
_I32 = C.c_int32
_ST = C.c_void_p   # cudaStream_t

# name -> argtypes, in the order of include/dfq_b200.h
SIGNATURES = {
    "dfq_abi_version": [],
    "dfq_struct_size": [C.c_int],
    "dfq_device_info": [C.POINTER(C.c_int), C.POINTER(C.c_int)],
    "dfq_cle_run": [_PF, _I64, C.c_void_p, _I32, C.c_void_p, _I32, C.c_void_p, C.c_void_p, _I32,
                    C.c_void_p, C.c_void_p, _I32, C.c_void_p, _ST],
    "dfq_cle_run_bc": [_PF, _I64, C.c_void_p, _I32, C.c_void_p, _I32, C.c_void_p, C.c_void_p, _I32,
                       C.c_void_p, C.c_void_p, _I32, C.c_void_p, C.c_void_p, _I32, C.c_void_p, _I32, _I32, _ST],
    "dfq_cle_takes_stack": [C.c_void_p, _I32, C.c_void_p, _I32, C.c_void_p, C.c_void_p, _I32, _I32, C.c_void_p],
    "dfq_bn_fold": [_PF, _I64, C.c_void_p, _I32, C.c_void_p, _I32, _ST],
    "dfq_bias_correct": [_PF, _I64, C.c_void_p, _I32, C.c_void_p, _I32, C.c_void_p, _I32, C.c_void_p, _I32, _I32, _ST],
    "dfq_bias_correct_absorb_clip": [_PF, _I64, C.c_void_p, _I32, C.c_void_p, _I32, C.c_void_p, _I32, C.c_void_p, _I32, _I32,
                                     C.c_void_p, _I32, C.c_float, _I32, C.c_float, C.c_float, _ST],
    "dfq_quantize_tensors": [_PF, _I64, C.c_void_p, _I32, C.c_int, _ST],
    "dfq_minmax": [_PF, _I64, _PF, _ST],
    "dfq_quant_dequant": [_PF, _PF, _I64, C.c_float, C.c_double, C.c_float, C.c_float, C.c_int, _PF, _ST],
    "dfq_quant_dequant_dev": [_PF, _PF, _I64, _PF, _PF, C.c_int, C.c_int, C.c_int, C.c_int, _PF, _ST],
    "dfq_act_minmax_per_sample": [_PF, _I64, _I64, _PF, _PF, _ST],
    "dfq_observer_update": [_PF, _PF, _PF, C.c_int, _Momentum, _ST],
    "dfq_observe_quant": [_PF, _PF, _I64, _I64, _PF, _PF, _PF, C.c_int, _Momentum, C.c_int, C.c_int, C.c_int, C.c_int, _ST],
    "dfq_bnstat_loss_fwd": [_PF, _I64, _I64, _I64, _PF, _PF, C.c_float, _PF, _PF, C.c_void_p, _ST],
    "dfq_bnstat_loss_bwd": [_PF, _PF, _I64, _I64, _I64, _PF, _PF, C.c_float, _PF, _PF, _PF, C.c_int, _ST],
    "dfq_range_rows": [_PF, _I64, _I64, _PF, _PF, _ST],
    "dfq_range_cols": [_PF, _I64, _I64, _I64, _I64, _PF, _PF, _ST],
    "dfq_mean_abs_diff": [_PF, _PF, _I64, C.c_void_p, _ST],
    "dfq_quant_error": [_PF, _PF, _I64, _PF, C.c_int, C.c_int, _ST],
    "dfq_selftest_bc_arithmetic": [_PF, _PF, _PF, _I64, _PF, C.c_int, C.c_int, C.c_void_p, _ST],
    "dfq_clamp": [_PF, _I64, C.c_float, C.c_float, _ST],
    "dfq_host_copy_segments": [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int],
    "dfq_i8_quantize_nhwc": [_PF, C.c_void_p, _I32, _I32, _I32, _I32, _I32, C.c_float, _ST],
    "dfq_i8_pack_weights": [_PF, _PF, C.c_void_p, C.c_void_p, _ST],
    "dfq_i8_conv": [C.c_void_p, C.c_void_p, _PF, _PF, _PF, C.c_void_p, C.c_void_p, _ST],
    "dfq_i8_conv_requant": [C.c_void_p, C.c_void_p, _PF, _PF, C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_void_p, _ST],
    "dfq_i8_conv_fused": [C.c_void_p, C.c_void_p, _PF, _PF, C.c_void_p, C.c_void_p, _ST],
    "dfq_i8_conv_slice": [C.c_void_p, C.c_void_p, _PF, _PF, C.c_void_p, _I32, _I32, C.c_void_p, _ST],
    "dfq_i8_conv_nhwc": [C.c_void_p, C.c_void_p, _PF, _PF, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, _ST],
    "dfq_i8_maxpool": [C.c_void_p, _PF, _PF, C.c_void_p, C.c_float, C.c_void_p, _ST],
    "dfq_i8_upsample_bilinear": [_PF, _PF, C.c_void_p, C.c_void_p, _ST],
    "dfq_i8_affine_quantize": [_PF, C.c_void_p, C.c_void_p, _I32, _I32, _I32, _I32, _I32, C.c_float, C.c_float, _I32, _ST],
    "dfq_i8_affine_pack": [_PF, C.c_float, C.c_float, _I32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, _ST],
    "dfq_i8_affine_conv": [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, _PF, _PF, C.c_void_p, C.c_void_p,
                           _ST],
    "dfq_i8_affine_conv_fused": [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, _PF, C.c_void_p, C.c_void_p,
                                 _ST],
    "dfq_i8_affine_conv_observed": [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, _PF, C.c_void_p,
                                    C.c_void_p, C.c_void_p, _ST],
    "dfq_i8_affine_conv_layout": [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, _PF, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.c_void_p, _ST],
    "dfq_i8_affine_upsample_bilinear": [_PF, C.c_void_p, C.c_void_p, C.c_void_p, _ST],
    "dfq_i8_affine_conv_rows": [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, _PF, C.c_void_p, C.c_void_p,
                                _ST],
    "dfq_i8_affine_maxpool": [C.c_void_p, _PF, _PF, C.c_void_p, C.c_void_p, C.c_float, C.c_float, _I32, C.c_void_p, _ST],
    "dfq_i8_pack_codes": [C.c_void_p, C.c_void_p, C.c_void_p, _ST],
    "dfq_i8_unpack_codes": [C.c_void_p, C.c_void_p, C.c_void_p, _ST],
    "dfq_i8_plane_mean": [_PF, _PF, C.c_void_p, _I64, _I32, _I64, _I32, C.c_float, _ST],
    "dfq_ssd_decode": [_PF, _PF, _PF, C.c_void_p, _ST],
    "dfq_ssd_nms": [_PF, _PF, _PF, _PF, C.c_void_p, C.c_void_p, C.c_void_p, _ST],
    "dfq_ssd_compact": [_PF, _PF, C.c_void_p, C.c_void_p, _PF, _PF, C.c_void_p, _PF, C.c_void_p, _ST],
    "dfq_ssd_soft_nms": [_PF, _PF, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, _ST],
    "dfq_ssd_soft_compact": [_PF, _PF, C.c_void_p, C.c_void_p, _PF, _PF, C.c_void_p, _PF, C.c_void_p, C.c_float, _ST],
    "dfq_seg_argmax": [_PF, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, _ST],
    "dfq_cls_count": [_PF, C.c_void_p, C.c_void_p, C.c_void_p, _I64, _I32, _ST],
    "dfq_map_match": [_PF, C.c_void_p, _PF, C.c_void_p, _I64, _PF, C.c_void_p, C.c_void_p, C.c_void_p, _I64, _I32, _I32,
                      C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, _ST],
    "dfq_map_curve": [C.c_void_p, C.c_void_p, _I64, _I32, C.c_void_p, _I32, C.c_void_p, _I64, C.c_void_p, _ST],
    "dfq_pre_resample": [C.c_void_p, C.c_void_p, C.c_void_p, _PF, _PF, _ST],
    "dfq_jpeg_decode": [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, _ST],
    "dfq_png_decode": [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, _ST],
}

_lib = None


def load(build_if_missing: bool = True) -> C.CDLL:
    """Load (building first if needed) the CUDA library.  Raises DfqError when unavailable."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        if not build_if_missing:
            raise DfqError("libdfq_sm90.so not built (run python -m dfq_b200._build)")
        from . import _build
        _build.build()
    try:
        lib = C.CDLL(LIB_PATH)
    except OSError as e:  # pragma: no cover
        raise DfqError("cannot load %s: %s" % (LIB_PATH, e)) from e
    for name, argtypes in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError = ABI mismatch: fail loudly
        fn.argtypes = argtypes
        fn.restype = C.c_int
    lib.dfq_last_error.restype = C.c_char_p
    lib.dfq_last_error.argtypes = []
    if lib.dfq_abi_version() != ABI_VERSION:
        raise DfqError("libdfq_sm90.so ABI %d != binding %d" % (lib.dfq_abi_version(), ABI_VERSION))
    _lib = lib
    return lib


def check(rc: int, what: str):
    if rc != 0:
        msg = load().dfq_last_error().decode("utf-8", "replace")
        raise DfqError("%s failed (%d): %s" % (what, rc, msg))


def table_ptr(arr: np.ndarray) -> C.c_void_p:
    assert arr.flags["C_CONTIGUOUS"]
    return C.c_void_p(arr.ctypes.data)


def require_cuda():
    """The product path needs a GPU; never degrade to the CPU."""
    import torch
    if not torch.cuda.is_available():
        raise DfqError("dfq_b200 requires a CUDA device (H100, sm_90a); no CPU fallback exists")


def stream_ptr():
    """The current device's current stream.  The package launches through launch(), which makes its tensors' device
    current first; this raw form is for direct ABI calls made on the current device."""
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _device_index(o) -> int:
    """CUDA device index of a tensor or device; -1 for the CPU."""
    import torch
    if isinstance(o, torch.Tensor):
        return o.get_device()
    d = torch.device(o)
    if d.type != "cuda":
        return -1
    return torch.cuda.current_device() if d.index is None else d.index


@contextlib.contextmanager
def launch(*on):
    """The launch context of library calls: `with launch(x, y) as st:` makes the one CUDA device of `on` (tensors,
    torch.devices or None, which are skipped) the current device and yields that device's current stream.  Every library
    call of the package is made inside one, so a call follows its tensors as torch's own ops do: tensors on cuda:1 run on
    cuda:1's current stream even when cuda:0 is current, the library's stream-ordered allocations come from cuda:1, and
    its per-device host state (DESIGN.md, "Launch context") is cuda:1's.  Tensors on two devices raise DfqError naming
    both, before anything is entered or launched.  CPU tensors enter no device: the entry points refuse them before their
    library calls, except under the host-side twins the tests run them through."""
    import torch
    idx = []
    for o in on:
        if o is not None and _device_index(o) not in idx:
            idx.append(_device_index(o))
    if len(idx) != 1:
        raise DfqError("a library call takes its tensors on one device, got %s"
                       % (" and ".join("cpu" if i < 0 else "cuda:%d" % i for i in idx) if idx else "none"))
    if idx[0] < 0:
        yield stream_ptr()
        return
    with torch.cuda.device(idx[0]):
        yield stream_ptr()
