"""ctypes binding of the C ABI declared in ``include/slowfast_b200.h``.

The product path has no CPU fallback: if the native library is missing, or is asked to run without a CUDA
device, the call fails loudly (``NativeLibraryError``).
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

from .build import lib_path


class NativeLibraryError(RuntimeError):
    pass


class ConvDesc(C.Structure):
    """Mirror of ``sfb_conv_desc`` (include/slowfast_b200.h)."""

    _fields_ = [
        ("a_hi", C.c_void_p), ("a_lo", C.c_void_p),
        ("n", C.c_int32), ("d", C.c_int32), ("h", C.c_int32), ("w", C.c_int32), ("c", C.c_int32),
        ("c_pitch", C.c_int64),
        ("b_hi", C.c_void_p), ("b_lo", C.c_void_p),
        ("cout", C.c_int32),
        ("kt", C.c_int32), ("kh", C.c_int32), ("kw", C.c_int32),
        ("dil_t", C.c_int32), ("dil_h", C.c_int32), ("dil_w", C.c_int32),
        ("str_t", C.c_int32), ("str_h", C.c_int32), ("str_w", C.c_int32),
        ("low_t", C.c_int32), ("low_h", C.c_int32), ("low_w", C.c_int32),
        ("out_t", C.c_int32), ("out_h", C.c_int32), ("out_w", C.c_int32),
        ("out", C.c_void_p),
        ("os_n", C.c_int64), ("os_t", C.c_int64), ("os_h", C.c_int64), ("os_w", C.c_int64),
        ("accumulate", C.c_int32),
        ("stats", C.c_void_p),
        ("nsplit", C.c_int32),
    ]


class WgradDesc(C.Structure):
    """Mirror of ``sfb_wgrad_desc``."""

    _fields_ = [
        ("x_hi", C.c_void_p), ("x_lo", C.c_void_p),
        ("n", C.c_int32), ("d", C.c_int32), ("h", C.c_int32), ("w", C.c_int32), ("c", C.c_int32),
        ("c_pitch", C.c_int64),
        ("dy_hi", C.c_void_p), ("dy_lo", C.c_void_p),
        ("cout", C.c_int32), ("dy_pitch", C.c_int64),
        ("kt", C.c_int32), ("kh", C.c_int32), ("kw", C.c_int32),
        ("dil_t", C.c_int32), ("dil_h", C.c_int32), ("dil_w", C.c_int32),
        ("str_t", C.c_int32), ("str_h", C.c_int32), ("str_w", C.c_int32),
        ("low_t", C.c_int32), ("low_h", C.c_int32), ("low_w", C.c_int32),
        ("out_t", C.c_int32), ("out_h", C.c_int32), ("out_w", C.c_int32),
        ("dw", C.c_void_p),
        ("nsplit", C.c_int32),
    ]


class BnApplyDesc(C.Structure):
    _fields_ = [
        ("y", C.c_void_p), ("y_pitch", C.c_int64), ("scale", C.c_void_p), ("shift", C.c_void_p),
        ("y2", C.c_void_p), ("y2_pitch", C.c_int64), ("scale2", C.c_void_p), ("shift2", C.c_void_p),
        ("res_hi", C.c_void_p), ("res_lo", C.c_void_p), ("res_pitch", C.c_int64),
        ("out_hi", C.c_void_p), ("out_lo", C.c_void_p), ("out_pitch", C.c_int64),
        ("rows", C.c_int64), ("c", C.c_int32), ("relu", C.c_int32),
    ]


class BnBwdDesc(C.Structure):
    _fields_ = [
        ("dout", C.c_void_p), ("dout_pitch", C.c_int64),
        ("mask_hi", C.c_void_p), ("mask_pitch", C.c_int64),
        ("y", C.c_void_p), ("y_pitch", C.c_int64),
        ("mean", C.c_void_p), ("invstd", C.c_void_p), ("gamma", C.c_void_p),
        ("dgamma", C.c_void_p), ("dbeta", C.c_void_p), ("accumulate_param_grads", C.c_int32),
        ("training", C.c_int32),
        ("dy_hi", C.c_void_p), ("dy_lo", C.c_void_p), ("dy_pitch", C.c_int64),
        ("dres", C.c_void_p), ("dres_pitch", C.c_int64), ("dres_accumulate", C.c_int32),
        ("partials", C.c_void_p), ("coef", C.c_void_p),
        ("rows", C.c_int64), ("c", C.c_int32), ("c_valid", C.c_int32),
        ("mask_scale", C.c_void_p), ("mask_shift", C.c_void_p),
    ]


class AttnFwdDesc(C.Structure):
    """Mirror of ``sfb_attn_fwd_desc``."""

    _fields_ = [
        ("q_hi", C.c_void_p), ("q_lo", C.c_void_p), ("k_hi", C.c_void_p), ("k_lo", C.c_void_p), ("v_hi", C.c_void_p),
        ("v_lo", C.c_void_p), ("rq", C.c_void_p), ("rq_pitch", C.c_int64),
        ("bh", C.c_int32), ("nq", C.c_int32), ("nk", C.c_int32), ("hd", C.c_int32),
        ("qt", C.c_int32), ("qh", C.c_int32), ("qw", C.c_int32), ("kt", C.c_int32), ("kh", C.c_int32), ("kw", C.c_int32),
        ("scale", C.c_float), ("out", C.c_void_p), ("p_hi", C.c_void_p), ("p_lo", C.c_void_p), ("p_pitch", C.c_int64),
        ("lse", C.c_void_p), ("nsplit", C.c_int32),
    ]


class AttnBwdDesc(C.Structure):
    """Mirror of ``sfb_attn_bwd_desc``."""

    _fields_ = [
        ("do_hi", C.c_void_p), ("do_lo", C.c_void_p), ("v_hi", C.c_void_p), ("v_lo", C.c_void_p),
        ("p_hi", C.c_void_p), ("p_lo", C.c_void_p), ("p_pitch", C.c_int64),
        ("ds_hi", C.c_void_p), ("ds_lo", C.c_void_p), ("ds_pitch", C.c_int64),
        ("drq", C.c_void_p), ("rq_pitch", C.c_int64),
        ("bh", C.c_int32), ("nq", C.c_int32), ("nk", C.c_int32), ("hd", C.c_int32),
        ("qt", C.c_int32), ("qh", C.c_int32), ("qw", C.c_int32), ("kt", C.c_int32), ("kh", C.c_int32), ("kw", C.c_int32),
        ("nsplit", C.c_int32),
    ]


class OptChunk(C.Structure):
    """Mirror of ``sfb_opt_chunk``."""

    _fields_ = [("param", C.c_void_p), ("offset", C.c_int64), ("count", C.c_int32), ("group", C.c_int32)]


class PoolDesc(C.Structure):
    _fields_ = [
        ("y", C.c_void_p), ("scale", C.c_void_p), ("shift", C.c_void_p),
        ("n", C.c_int32), ("t", C.c_int32), ("h", C.c_int32), ("w", C.c_int32), ("c", C.c_int32),
        ("oh", C.c_int32), ("ow", C.c_int32), ("kh", C.c_int32), ("kw", C.c_int32),
        ("sh", C.c_int32), ("sw", C.c_int32), ("ph", C.c_int32), ("pw", C.c_int32),
        ("out_hi", C.c_void_p), ("out_lo", C.c_void_p), ("out_pitch", C.c_int64),
        ("argmax", C.c_void_p),
        ("dout", C.c_void_p), ("dout_pitch", C.c_int64),
        ("dz", C.c_void_p),
    ]


class DwPoolDesc(C.Structure):
    _fields_ = [
        ("src", C.c_void_p), ("src_pitch", C.c_int64), ("src_c0", C.c_int32), ("bias", C.c_void_p),
        ("w", C.c_void_p), ("out", C.c_void_p),
        ("b", C.c_int32), ("heads", C.c_int32), ("hd", C.c_int32), ("t", C.c_int32), ("h", C.c_int32),
        ("w_", C.c_int32), ("ot", C.c_int32), ("oh", C.c_int32), ("ow", C.c_int32),
        ("kt", C.c_int32), ("kh", C.c_int32), ("kw", C.c_int32), ("st", C.c_int32), ("sh", C.c_int32),
        ("sw", C.c_int32), ("has_pool", C.c_int32),
        ("dout", C.c_void_p), ("dsrc", C.c_void_p), ("wpartials", C.c_void_p),
    ]


class SoftmaxDesc(C.Structure):
    _fields_ = [
        ("s", C.c_void_p), ("s_pitch", C.c_int64), ("rq", C.c_void_p), ("rq_pitch", C.c_int64),
        ("p_hi", C.c_void_p), ("p_lo", C.c_void_p), ("p_pitch", C.c_int64),
        ("bh", C.c_int32), ("nq", C.c_int32), ("nk", C.c_int32),
        ("qt", C.c_int32), ("qh", C.c_int32), ("qw", C.c_int32), ("kt", C.c_int32), ("kh", C.c_int32),
        ("kw", C.c_int32),
        ("dp", C.c_void_p), ("dp_pitch", C.c_int64),
        ("ds_hi", C.c_void_p), ("ds_lo", C.c_void_p), ("ds_pitch", C.c_int64), ("drq", C.c_void_p),
    ]


class TokPoolDesc(C.Structure):
    _fields_ = [
        ("x", C.c_void_p), ("out", C.c_void_p), ("argmax", C.c_void_p),
        ("b", C.c_int32), ("c", C.c_int32), ("t", C.c_int32), ("h", C.c_int32), ("w", C.c_int32),
        ("ot", C.c_int32), ("oh", C.c_int32), ("ow", C.c_int32),
        ("kt", C.c_int32), ("kh", C.c_int32), ("kw", C.c_int32), ("st", C.c_int32), ("sh", C.c_int32),
        ("sw", C.c_int32),
        ("dout", C.c_void_p), ("dx", C.c_void_p), ("dx_accumulate", C.c_int32),
    ]


class Pool3dDesc(C.Structure):
    _fields_ = [
        ("in_hi", C.c_void_p), ("in_lo", C.c_void_p), ("in_pitch", C.c_int64),
        ("out_hi", C.c_void_p), ("out_lo", C.c_void_p), ("out_pitch", C.c_int64),
        ("argmax", C.c_void_p),
        ("n", C.c_int32), ("t", C.c_int32), ("h", C.c_int32), ("w", C.c_int32), ("c", C.c_int32),
        ("ot", C.c_int32), ("oh", C.c_int32), ("ow", C.c_int32),
        ("kt", C.c_int32), ("kh", C.c_int32), ("kw", C.c_int32), ("st", C.c_int32), ("sh", C.c_int32),
        ("sw", C.c_int32), ("pt", C.c_int32), ("ph", C.c_int32), ("pw", C.c_int32),
        ("dout", C.c_void_p), ("dout_pitch", C.c_int64),
        ("din", C.c_void_p), ("din_pitch", C.c_int64), ("din_accumulate", C.c_int32),
    ]


class StemDesc(C.Structure):
    _fields_ = [
        ("x_hi", C.c_void_p), ("x_lo", C.c_void_p),
        ("n", C.c_int32), ("t", C.c_int32), ("h", C.c_int32), ("wf", C.c_int32),
        ("f_hi", C.c_void_p), ("f_lo", C.c_void_p), ("dy_hi", C.c_void_p), ("dy_lo", C.c_void_p),
        ("cout", C.c_int32), ("kt", C.c_int32), ("kh", C.c_int32), ("kwf", C.c_int32),
        ("str_t", C.c_int32), ("str_h", C.c_int32), ("pad_t", C.c_int32), ("pad_h", C.c_int32),
        ("pad_wf", C.c_int32),
        ("out_t", C.c_int32), ("out_h", C.c_int32), ("out_w", C.c_int32),
        ("out", C.c_void_p), ("stats", C.c_void_p), ("dwm", C.c_void_p),
        ("nsplit", C.c_int32),
    ]


class BgemmDesc(C.Structure):
    _fields_ = [
        ("a_hi", C.c_void_p), ("a_lo", C.c_void_p), ("lda", C.c_int64), ("batch_stride_a", C.c_int64),
        ("a_mn_major", C.c_int32),
        ("b_hi", C.c_void_p), ("b_lo", C.c_void_p), ("ldb", C.c_int64), ("batch_stride_b", C.c_int64),
        ("b_mn_major", C.c_int32),
        ("m", C.c_int32), ("n", C.c_int32), ("k", C.c_int32), ("batch", C.c_int32),
        ("out", C.c_void_p), ("ldd", C.c_int64), ("batch_stride_d", C.c_int64),
        ("alpha", C.c_float), ("accumulate", C.c_int32), ("nsplit", C.c_int32),
    ]


_LIB = None

# every symbol include/slowfast_b200.h declares: (name, restype, argtypes)
class DwConvDesc(C.Structure):
    _fields_ = [
        ("x_hi", C.c_void_p), ("x_lo", C.c_void_p), ("x_f32", C.c_void_p), ("x_pitch", C.c_int64),
        ("w", C.c_void_p),
        ("y", C.c_void_p), ("y_pitch", C.c_int64), ("stats", C.c_void_p),
        ("n", C.c_int32), ("t", C.c_int32), ("h", C.c_int32), ("w_", C.c_int32), ("c", C.c_int32),
        ("c_valid", C.c_int32), ("ot", C.c_int32), ("oh", C.c_int32), ("ow", C.c_int32),
        ("kt", C.c_int32), ("kh", C.c_int32), ("kw", C.c_int32), ("st", C.c_int32), ("sh", C.c_int32),
        ("sw", C.c_int32), ("pt", C.c_int32), ("ph", C.c_int32), ("pw", C.c_int32),
        ("dy", C.c_void_p), ("dy_pitch", C.c_int64),
        ("dx", C.c_void_p), ("dx_hi", C.c_void_p), ("dx_lo", C.c_void_p), ("dx_pitch", C.c_int64),
        ("dx_accumulate", C.c_int32),
        ("wpartials", C.c_void_p),
        ("in_scale", C.c_void_p), ("in_shift", C.c_void_p), ("in_relu", C.c_int32),
    ]


class BnActDesc(C.Structure):
    _fields_ = [
        ("y", C.c_void_p), ("y_pitch", C.c_int64),
        ("scale", C.c_void_p), ("shift", C.c_void_p), ("mean", C.c_void_p), ("invstd", C.c_void_p),
        ("gate", C.c_void_p), ("act", C.c_int32),
        ("rows", C.c_int64), ("rows_per_sample", C.c_int64), ("c", C.c_int32),
        ("out_hi", C.c_void_p), ("out_lo", C.c_void_p), ("out_pitch", C.c_int64),
        ("dout", C.c_void_p), ("dout_pitch", C.c_int64),
        ("partials", C.c_void_p), ("davg", C.c_void_p), ("coef", C.c_void_p),
        ("dy", C.c_void_p), ("dy_pitch", C.c_int64),
    ]


class SeDesc(C.Structure):
    _fields_ = [
        ("n", C.c_int32), ("c", C.c_int32), ("c_pad", C.c_int32), ("f", C.c_int32),
        ("rows_per_sample", C.c_int64), ("tiles_per_sample", C.c_int32), ("m_tiles", C.c_int32),
        ("stats", C.c_void_p), ("scale", C.c_void_p), ("shift", C.c_void_p), ("mean", C.c_void_p),
        ("invstd", C.c_void_p),
        ("w1", C.c_void_p), ("b1", C.c_void_p), ("w2", C.c_void_p), ("b2", C.c_void_p),
        ("ymean", C.c_void_p), ("avg", C.c_void_p), ("hid", C.c_void_p), ("gate", C.c_void_p),
        ("partials", C.c_void_p), ("tiles2_per_sample", C.c_int32),
        ("a12", C.c_void_p), ("do2", C.c_void_p), ("dhid", C.c_void_p), ("davg", C.c_void_p),
        ("gamma", C.c_void_p), ("beta", C.c_void_p),
        ("dw1", C.c_void_p), ("db1", C.c_void_p), ("dw2", C.c_void_p), ("db2", C.c_void_p),
        ("dgamma", C.c_void_p), ("dbeta", C.c_void_p), ("coef", C.c_void_p),
        ("training", C.c_int32), ("has_se", C.c_int32),
    ]


class PackJob(C.Structure):
    _fields_ = [
        ("w", C.c_void_p), ("hi", C.c_void_p), ("lo", C.c_void_p),
        ("cout", C.c_int32), ("cin", C.c_int32), ("taps_total", C.c_int32), ("ntaps", C.c_int32),
        ("transpose", C.c_int32), ("cols_pad", C.c_int32),
        ("first_block", C.c_int32), ("n_blocks", C.c_int32),
        ("tapmap", C.c_int16 * 32),
    ]


_SIGNATURES = [
    ("sfb_last_error", C.c_char_p, []),
    ("sfb_abi_version", C.c_int, []),
    ("sfb_build_arch", C.c_char_p, []),
    ("sfb_conv_m_tiles", C.c_int64, [C.POINTER(ConvDesc)]),
    ("sfb_conv_igemm", C.c_int, [C.POINTER(ConvDesc), C.c_void_p]),
    ("sfb_conv_wgrad", C.c_int, [C.POINTER(WgradDesc), C.c_void_p]),
    ("sfb_zero_f32_2d", C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p]),
    ("sfb_add_f32_2d", C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int64, C.c_int64, C.c_void_p]),
    ("sfb_split_planes", C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64,
                                   C.c_void_p]),
    ("sfb_input_pack", C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                 C.c_void_p, C.c_void_p, C.c_void_p]),
    ("sfb_filter_pack", C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_int32), C.c_int32,
                                  C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("sfb_filter_unpack_grad", C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                         C.c_int32, C.c_void_p]),
    ("sfb_bn_finalize", C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_float, C.c_float, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_void_p]),
    ("sfb_bn_apply", C.c_int, [C.POINTER(BnApplyDesc), C.c_void_p]),
    ("sfb_bn_bwd_blocks", C.c_int32, [C.c_int64, C.c_int32]),
    ("sfb_bn_bwd", C.c_int, [C.POINTER(BnBwdDesc), C.c_void_p]),
    ("sfb_bn_relu_maxpool_fwd", C.c_int, [C.POINTER(PoolDesc), C.c_void_p]),
    ("sfb_bn_relu_maxpool_bwd", C.c_int, [C.POINTER(PoolDesc), C.c_void_p]),
    ("sfb_maxpool3d_fwd", C.c_int, [C.POINTER(Pool3dDesc), C.c_void_p]),
    ("sfb_maxpool3d_bwd", C.c_int, [C.POINTER(Pool3dDesc), C.c_void_p]),
    ("sfb_stem_input_fold", C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                      C.c_void_p, C.c_void_p]),
    ("sfb_stem_filter_fold", C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                       C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                       C.c_void_p]),
    ("sfb_stem_m_tiles", C.c_int64, [C.POINTER(StemDesc)]),
    ("sfb_stem_fprop", C.c_int, [C.POINTER(StemDesc), C.c_void_p]),
    ("sfb_stem_wgrad", C.c_int, [C.POINTER(StemDesc), C.c_void_p]),
    ("sfb_set_wgrad_direct", C.c_int, [C.c_int32]),
    ("sfb_stem8_supported", C.c_int, [C.POINTER(StemDesc)]),
    ("sfb_stem8_m_tiles", C.c_int64, [C.POINTER(StemDesc)]),
    ("sfb_stem8_input_fold", C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                       C.c_void_p, C.c_void_p]),
    ("sfb_stem8_filter_fold", C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("sfb_stem8_fprop", C.c_int, [C.POINTER(StemDesc), C.c_void_p]),
    ("sfb_stem8_wgrad", C.c_int, [C.POINTER(StemDesc), C.c_void_p]),
    ("sfb_gemm_batched", C.c_int, [C.POINTER(BgemmDesc), C.c_void_p]),
    ("sfb_layernorm_fwd", C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("sfb_rowslab_blocks", C.c_int32, [C.c_int64]),
    ("sfb_layernorm_bwd", C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    ("sfb_colsum", C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    ("sfb_tokens_assemble", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    ("sfb_tokens_split_grad", C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("sfb_dwpool_fwd", C.c_int, [C.POINTER(DwPoolDesc), C.c_void_p]),
    ("sfb_dwpool_wgrad_blocks", C.c_int32, [C.POINTER(DwPoolDesc)]),
    ("sfb_dwpool_bwd", C.c_int, [C.POINTER(DwPoolDesc), C.c_void_p, C.c_int32, C.c_void_p]),
    ("sfb_softmax_relpos_fwd", C.c_int, [C.POINTER(SoftmaxDesc), C.c_void_p]),
    ("sfb_softmax_relpos_bwd", C.c_int, [C.POINTER(SoftmaxDesc), C.c_void_p]),
    ("sfb_attn_merge", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("sfb_attn_split_grad", C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("sfb_residual_add", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p]),
    ("sfb_bias_gelu", C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("sfb_bias_gelu_bwd", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("sfb_scale_split", C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("sfb_token_maxpool_fwd", C.c_int, [C.POINTER(TokPoolDesc), C.c_void_p]),
    ("sfb_token_maxpool_bwd", C.c_int, [C.POINTER(TokPoolDesc), C.c_void_p]),
    ("sfb_global_avgpool_fwd", C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32,
                                         C.c_void_p, C.c_int64, C.c_void_p]),
    ("sfb_global_avgpool_bwd", C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                         C.c_int64, C.c_void_p]),
    ("sfb_window_avgpool_fwd", C.c_int, [C.c_void_p, C.c_void_p, C.c_int64] + [C.c_int32] * 8 +
     [C.c_void_p, C.c_int64, C.c_void_p]),
    ("sfb_rows_group_mean", C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    ("sfb_dropout_fwd", C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_float, C.c_uint64, C.c_void_p, C.c_void_p]),
    ("sfb_dropout_bwd", C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_float, C.c_void_p]),
    ("sfb_small_linear_fwd", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                       C.c_int32, C.c_void_p]),
    ("sfb_small_linear_bwd", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    ("sfb_row_softmax", C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]),
    ("sfb_droppath_scales", C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_uint64, C.c_void_p, C.c_void_p]),
    ("sfb_pack_job_size", C.c_int32, []),
    ("sfb_filter_pack_multi", C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]),
    ("sfb_stem_wgrad_direct", C.c_int, [C.c_void_p] + [C.c_int32] * 5 + [C.c_void_p, C.c_void_p] + [C.c_int32] * 10 +
     [C.c_void_p, C.c_void_p]),
    ("sfb_dwconv_m_tiles", C.c_int32, [C.POINTER(DwConvDesc)]),
    ("sfb_dwconv_tiles_per_sample", C.c_int32, [C.POINTER(DwConvDesc)]),
    ("sfb_dwconv_fwd", C.c_int, [C.POINTER(DwConvDesc), C.c_void_p]),
    ("sfb_dwconv_wgrad_blocks", C.c_int32, [C.POINTER(DwConvDesc)]),
    ("sfb_dwconv_bwd", C.c_int, [C.POINTER(DwConvDesc), C.c_void_p, C.c_void_p]),
    ("sfb_bnact_fwd", C.c_int, [C.POINTER(BnActDesc), C.c_void_p]),
    ("sfb_bnact_tiles_per_sample", C.c_int32, [C.c_int64, C.c_int64]),
    ("sfb_bnact_bwd_reduce", C.c_int, [C.POINTER(BnActDesc), C.c_void_p]),
    ("sfb_bnact_bwd_apply", C.c_int, [C.POINTER(BnActDesc), C.c_void_p]),
    ("sfb_se_fwd", C.c_int, [C.POINTER(SeDesc), C.c_void_p]),
    ("sfb_se_bwd", C.c_int, [C.POINTER(SeDesc), C.c_void_p]),
    ("sfb_relu_fwd", C.c_int, [C.c_void_p, C.c_int64, C.c_void_p]),
    ("sfb_relu_bwd", C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    ("sfb_mask_upsample", C.c_int, [C.c_void_p] + [C.c_int32] * 7 + [C.c_void_p, C.c_void_p]),
    ("sfb_tokens_assemble_masked", C.c_int, [C.c_void_p] * 5 + [C.c_int32] * 3 + [C.c_void_p, C.c_void_p]),
    ("sfb_tokens_split_grad_masked", C.c_int, [C.c_void_p] * 2 + [C.c_int32] * 3 + [C.c_void_p] * 5),
    ("sfb_rows_unpad_bias", C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                      C.c_void_p]),
    ("sfb_rows_pad_split", C.c_int, [C.c_void_p] + [C.c_int32] * 4 + [C.c_void_p] * 3),
    ("sfb_attn_fwd_supported", C.c_int32, [C.c_int32] * 5),
    ("sfb_attn_fwd", C.c_int, [C.POINTER(AttnFwdDesc), C.c_void_p]),
    ("sfb_attn_bwd_ds", C.c_int, [C.POINTER(AttnBwdDesc), C.c_void_p]),
    ("sfb_clip_normalize_pack", C.c_int, [C.c_void_p] + [C.c_int32] * 4 + [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                          C.c_int32, C.c_void_p, C.c_void_p]),
    ("sfb_allreduce_flat", C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_void_p]),
    ("sfb_set_simt_smallc", C.c_int, [C.c_int32, C.c_int32]),
    ("sfb_set_dw3", C.c_int, [C.c_int32]),
    ("sfb_opt_chunk_size", C.c_int32, []),
    ("sfb_flat_sumsq_blocks", C.c_int32, []),
    ("sfb_flat_sumsq", C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_float, C.c_float, C.c_void_p, C.c_void_p]),
    ("sfb_flat_sgd", C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                               C.c_float, C.c_float, C.c_int32, C.c_int32, C.c_void_p]),
    ("sfb_flat_adamw", C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_int64, C.c_void_p]),
    ("sfb_hog_targets", C.c_int, [C.c_void_p] + [C.c_int32] * 9 + [C.c_void_p, C.c_void_p]),
]


def exported_symbols():
    return [s[0] for s in _SIGNATURES]


def load() -> C.CDLL:
    """Load ``libsfb200.so`` (built in-tree by ``slowfast_b200.build.build_native``)."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = Path(lib_path())
    if not path.exists():
        raise NativeLibraryError(
            f"{path} is missing: build it with `python -m slowfast_b200.build` (nvcc, sm_90a). "
            "slowfast_b200 has no CPU fallback.")
    lib = C.CDLL(str(path))
    for name, res, args in _SIGNATURES:
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _LIB = lib
    return lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = load().sfb_last_error()
        raise NativeLibraryError(f"{what} failed (rc={rc}): {msg.decode() if msg else '?'}")
