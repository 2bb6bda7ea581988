"""ctypes binding of the C-ABI library (include/styletts2_b200.h).

The library is the product; this file is only the loader.  There is NO fallback: if the
shared object is missing or a CUDA device is absent, compute calls raise.
"""
from __future__ import annotations

import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libstyletts2_b200.so")

ACT_NONE, ACT_LRELU, ACT_SNAKE, ACT_TANH, ACT_GELU, ACT_GELU_TANH = 0, 1, 2, 3, 4, 5
TC_FAST, TC_ACCURATE, TC_F16X3 = 0, 1, 2      # precision recipes of the tensor-core conv (include/styletts2_b200.h)
TC_TMAJOR = 16                               # flag: time-major layout + kernel for narrow layers (FAST recipe, Cout <= 128)
ABI_VERSION = 2

_vp, _i, _f, _ll = C.c_void_p, C.c_int, C.c_float, C.c_longlong


class ConvArgs(C.Structure):
    _fields_ = [
        ("x", _vp), ("x_bstride", _ll), ("Cin", _i), ("Lin", _i),
        ("w", _vp), ("bias", _vp),
        ("y", _vp), ("y_bstride", _ll), ("Cout", _i), ("Lq", _i), ("y_len", _i),
        ("y_tstride", _i), ("y_toffset", _i),
        ("B", _i), ("K", _i), ("stride", _i), ("dil", _i), ("pad", _i),
        ("pre_a", _vp), ("pre_b", _vp), ("pre_act", _i), ("pre_slope", _f), ("pre_alpha", _vp),
        ("res", _vp), ("res_bstride", _ll), ("res_len", _i), ("res_shift", _i),
        ("out_div", _f), ("accum_mode", _i), ("accum_div", _f), ("out_act", _i),
        ("stats", _vp), ("stats_nparts", _i), ("stats_part_offset", _i), ("dup_q0_to", _i),
    ]


class Conv2dArgs(C.Structure):
    _fields_ = [
        ("x", _vp), ("wt", _vp), ("bias", _vp), ("res", _vp), ("out", _vp),
        ("B", _i), ("Cin", _i), ("H", _i), ("W", _i), ("Cout", _i), ("KH", _i), ("KW", _i), ("pad", _i),
        ("pre_act", _i), ("slope", _f), ("out_scale", _f),
    ]


class RowsArgs(C.Structure):
    _fields_ = [
        ("h_in", _vp), ("h_in_ld", _ll),
        ("x", _vp), ("Cx", _i), ("xs", _f), ("emb", _vp), ("emb_ld", _ll),
        ("add", _vp),
        ("h_out", _vp), ("h_out_ld", _ll),
        ("g1", _vp), ("b1", _vp), ("g2", _vp), ("b2", _vp), ("gb_bstride", _ll), ("ada", _i),
        ("out1", _vp), ("out1_ld", _ll), ("out2", _vp), ("out2_ld", _ll),
        ("B", _i), ("N", _i), ("C", _i), ("eps", _f),
        ("lengths", _vp),
    ]


# name -> argtypes (restype is int unless listed in _RESTYPES); mirrors include/styletts2_b200.h
SIGNATURES = {
    "st2_last_error": [],
    "st2_abi_version": [],
    "st2_launch_count": [],
    "st2_weight_norm_fold": [_vp, _vp, _vp, _i, _i, _vp],
    "st2_row_norm": [_vp, _vp, _i, _i, _vp],
    "st2_conv_weight_layout": [_vp, _vp, _i, _i, _i, _vp],
    "st2_convT_weight_layout": [_vp, _vp, _i, _i, _i, _i, _i, _vp],
    "st2_conv1d": [C.POINTER(ConvArgs), _vp],
    "st2_conv_stats_parts": [_i],
    "st2_conv_tc_weight_bytes": [_i, _i, _i],
    "st2_conv_tc_weight_layout": [_vp, _vp, _i, _i, _i, _i, _vp],
    "st2_conv_tc_supported": [_i, _i, _i, _i, _i],
    "st2_conv1d_tc": [C.POINTER(ConvArgs), _vp, _i, _i, _vp],
    "st2_debug_set_flags": [_i],
    "st2_convT_tc_weight_bytes": [_i, _i, _i, _i],
    "st2_convT_tc_weight_layout": [_vp, _vp, _i, _i, _i, _i, _i, _i, _vp],
    "st2_conv_transpose1d_tc2": [C.POINTER(ConvArgs), _vp, _i, _i, _i, _i, _i, _vp, _vp],
    "st2_conv_transpose1d": [C.POINTER(ConvArgs), _vp, _i, _i, _i, _i, _vp],
    "st2_instance_stats": [_vp, _ll, _i, _i, _i, _vp, _vp],
    "st2_adain_coef": [_vp, _i, _vp, _ll, _i, _i, _f, _vp, _vp, _vp],
    "st2_adain_lrelu_pool": [_vp, _ll, _vp, _vp, _vp, _vp, _f, _i, _i, _i, _vp, _ll, _vp],
    "st2_channel_layernorm_lrelu": [_vp, _vp, _vp, _vp, _f, _f, _vp, _i, _i, _i, _vp],
    "st2_rows_ln": [C.POINTER(RowsArgs), _vp],
    "st2_bcast_cols": [_vp, _ll, _i, _vp, _i, _i, _i, _vp, _vp],
    "st2_mean_rows": [_vp, _ll, _i, _i, _i, _vp, _vp],
    "st2_rows_ln_packed": [C.POINTER(RowsArgs), _vp, _i, _vp],
    "st2_mean_segments": [_vp, _ll, _vp, _i, _i, _vp, _vp],
    "st2_linear": [_vp, _ll, _ll, _ll, _i, _vp, _vp, _vp, _ll, _vp, _ll, _i, _i, _i, _i, _vp],
    "st2_linear_tc_weight_bytes": [_i, _i],
    "st2_linear_tc_weight_layout": [_vp, _vp, _i, _i, _vp],
    "st2_linear_tc": [_vp, _ll, _vp, _vp, _vp, _ll, _vp, _ll, _i, _i, _i, _i, _vp],
    "st2_linear_tc_pre": [_vp, _ll, _vp, _vp, _vp, _vp, _ll, _vp, _ll, _i, _i, _i, _i, _vp],
    "st2_linear_tc_split": [_vp, _ll, _i, _i, _vp, _vp],
    "st2_linear_tc_split_bytes": [_i, _i],
    "st2_range_flag_fetch": [_vp],
    "st2_attention": [_vp, _vp, _vp, _i, _i, _i, _i, _f, _vp],
    "st2_attention_ex": [_vp, _ll, _vp, _vp, _ll, _vp, _ll, _vp, _i, _i, _i, _i, _f, _vp],
    "st2_attention_tc_supported": [_ll, _ll, _ll, _i],
    "st2_attention_tc": [_vp, _ll, _vp, _vp, _ll, _vp, _ll, _vp, _i, _i, _i, _i, _f, _vp],
    "st2_attention_tc_packed": [_vp, _ll, _vp, _vp, _ll, _vp, _ll, _vp, _i, _i, _i, _i, _f, _vp],
    "st2_embedding_sum_rows": [_vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp],
    "st2_lstm_bidir": [_vp, _vp, _vp, _ll, _ll, _ll, _vp, _i, _i, _i, _vp, _vp],
    "st2_kdiff_step": [_vp, _vp, _vp, _f, _f, _f, _f, _vp, _f, _vp, _f, _vp, _i, _vp],
    "st2_scale": [_vp, _f, _vp, _i, _vp],
    "st2_time_embedding": [_vp, _vp, _i, _i, _vp, _ll, _vp],
    "st2_axpby": [_vp, _f, _vp, _f, _vp, _i, _vp],
    "st2_embedding_cl": [_vp, _vp, _vp, _i, _i, _i, _vp, _vp],
    "st2_durations": [_vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp],
    "st2_frame_tokens": [_vp, _i, _i, _i, _i, _vp, _vp, _vp],
    "st2_expand_rows": [_vp, _ll, _vp, _i, _i, _i, _i, _vp, _ll, _vp],
    "st2_expand_cl": [_vp, _vp, _i, _i, _i, _i, _vp, _ll, _vp],
    "st2_polyphase_gather": [_vp, _ll, _i, _i, _i, _i, _i, _i, _vp, _vp],
    "st2_sine_source": [_vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, C.c_ulonglong, C.c_ulonglong, _vp, _vp],
    "st2_randn": [_vp, _ll, C.c_ulonglong, C.c_ulonglong, _vp, _vp],
    "st2_rng_advance": [_vp, _vp],
    "st2_debug_lstm_cluster": [_i],
    "st2_debug_lstm_trace": [_vp],
    "st2_spectral_norm_fold": [_vp, _vp, _vp, _i, _i, _vp, _vp, _vp],
    "st2_conv2d": [C.POINTER(Conv2dArgs), _vp],
    "st2_dwconv3x3_s2": [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp],
    "st2_avgpool_half": [_vp, _vp, _i, _i, _i, _vp],
    "st2_mean_hw_lrelu": [_vp, _vp, _i, _i, _f, _vp],
    "st2_mel_frames": [_vp, _vp, _i, _i, _i, _i, _i, _vp, _vp],
    "st2_mel_power": [_vp, _i, _i, _vp, _vp],
    "st2_logmel": [_vp, _i, _i, _i, _f, _f, _f, _vp, _vp],
    "st2_stft20": [_vp, _i, _i, _vp, _vp],
    "st2_istft20_expsin": [_vp, _i, _i, _vp, _vp],
    "st2_pcm16": [_vp, _ll, _f, _vp, _vp],
}
_RESTYPES = {"st2_last_error": C.c_char_p, "st2_launch_count": C.c_longlong, "st2_conv_tc_weight_bytes": C.c_longlong,
             "st2_convT_tc_weight_bytes": C.c_longlong, "st2_linear_tc_weight_bytes": C.c_longlong,
             "st2_linear_tc_split_bytes": C.c_longlong}

_lib = None


def load():
    """dlopen the library (no CUDA call is made here)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -m styletts2_b200.build` "
            "(nvcc -gencode arch=compute_90a,code=sm_90a). There is no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, argtypes in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.argtypes = argtypes
        fn.restype = _RESTYPES.get(name, C.c_int)
    if lib.st2_abi_version() != ABI_VERSION:
        raise RuntimeError("styletts2_b200 ABI version mismatch")
    _lib = lib
    return lib


def last_error() -> str:
    return load().st2_last_error().decode()


def launch_count() -> int:
    return int(load().st2_launch_count())


def check(rc: int, what: str = ""):
    if rc != 0:
        raise RuntimeError(f"styletts2_b200 {what} failed (cudaError {rc}): {last_error()}")


def stream_ptr():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t):
    """Device pointer of a tensor (None -> NULL)."""
    if t is None:
        return None
    if not t.is_cuda:
        raise RuntimeError("styletts2_b200 kernels need CUDA tensors (no CPU fallback)")
    return C.c_void_p(t.data_ptr())


def call(name: str, *args):
    lib = load()
    rc = getattr(lib, name)(*args)
    check(rc, name)
