"""ctypes binding of libptq4vit_b200.so (the C ABI declared in include/ptq4vit_b200.h).

The product path has no CPU fallback: if the shared library is missing this module
raises at import of the first native call, loudly.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libptq4vit_b200.so")

OPERAND = {"auto": 0, "int8": 1, "bf16": 2}
KERNEL = {"tcgen05": 0, "simt": 1}


class LinearDesc(C.Structure):
    _fields_ = [("rows", C.c_int32), ("tokens", C.c_int32), ("in_features", C.c_int32), ("out_features", C.c_int32),
                ("n_V", C.c_int32), ("n_H", C.c_int32), ("n_a", C.c_int32), ("w_bit", C.c_int32), ("a_bit", C.c_int32),
                ("eq_n", C.c_int32), ("search_round", C.c_int32), ("eq_alpha", C.c_double), ("eq_beta", C.c_double),
                ("post_gelu", C.c_int32), ("has_bias", C.c_int32), ("operand", C.c_int32), ("kernel", C.c_int32),
                ("init_layerwise", C.c_int32), ("rows_per_chunk", C.c_int32)]


class MatMulDesc(C.Structure):
    _fields_ = [("batch", C.c_int32), ("heads", C.c_int32), ("S1", C.c_int32), ("S2", C.c_int32), ("S3", C.c_int32),
                ("A_bit", C.c_int32), ("B_bit", C.c_int32), ("eq_n", C.c_int32), ("search_round", C.c_int32),
                ("eq_alpha", C.c_double), ("eq_beta", C.c_double), ("sos", C.c_int32), ("operand", C.c_int32),
                ("kernel", C.c_int32), ("init_layerwise", C.c_int32), ("images_per_chunk", C.c_int32)]


class AttentionDesc(C.Structure):
    _fields_ = [("batch", C.c_int32), ("tokens", C.c_int32), ("heads", C.c_int32), ("head_dim", C.c_int32),
                ("scale_on_q", C.c_int32), ("n_windows", C.c_int32), ("scale", C.c_double)]


class ConvDesc(C.Structure):
    _fields_ = [("images", C.c_int32), ("out_channels", C.c_int32), ("K", C.c_int32), ("positions", C.c_int32),
                ("w_bit", C.c_int32), ("eq_n", C.c_int32), ("eq_alpha", C.c_double), ("eq_beta", C.c_double),
                ("has_bias", C.c_int32), ("kernel", C.c_int32), ("layerwise", C.c_int32)]


class ConvFrozenDesc(C.Structure):
    _fields_ = [("images", C.c_int32), ("in_channels", C.c_int32), ("height", C.c_int32), ("width", C.c_int32),
                ("out_channels", C.c_int32), ("kernel_h", C.c_int32), ("kernel_w", C.c_int32), ("w_bit", C.c_int32),
                ("layerwise", C.c_int32), ("has_bias", C.c_int32)]


class WindowLayout(C.Structure):
    _fields_ = [("images", C.c_int32), ("height", C.c_int32), ("width", C.c_int32), ("window", C.c_int32), ("shift", C.c_int32)]


GATHER = {"window": 1, "merge": 2}      # P4V_GATHER_WINDOW, P4V_GATHER_MERGE


class InputGather(C.Structure):
    _fields_ = [("mode", C.c_int32), ("layout", WindowLayout)]


_P = C.c_void_p
_SIGNATURES = {
    "p4v_linear_workspace_bytes": [C.POINTER(LinearDesc), C.POINTER(C.c_size_t)],
    "p4v_linear_score_log_floats": [C.POINTER(LinearDesc), C.POINTER(C.c_size_t)],
    "p4v_linear_calibrate": [C.POINTER(LinearDesc), _P, _P, _P, _P, _P, _P, C.c_size_t, _P, _P, _P, _P],
    "p4v_linear_begin": [C.POINTER(LinearDesc), _P, _P, _P, _P, _P, _P, C.c_size_t, _P],
    "p4v_linear_search_w": [C.POINTER(LinearDesc), _P, _P, _P, _P, C.c_int32, C.c_int32, _P, _P],
    "p4v_linear_search_a": [C.POINTER(LinearDesc), _P, _P, _P, _P, C.c_int32, C.c_int32, _P, _P],
    "p4v_linear_intervals": [C.POINTER(LinearDesc), _P, _P, _P, _P],
    "p4v_linear_quant_forward_workspace_bytes": [C.POINTER(LinearDesc), C.POINTER(C.c_size_t)],
    "p4v_linear_quant_forward": [C.POINTER(LinearDesc), _P, _P, _P, _P, _P, _P, C.c_size_t, _P, _P],
    "p4v_linear_pack_bytes": [C.POINTER(LinearDesc), C.POINTER(C.c_size_t)],
    "p4v_linear_pack": [C.POINTER(LinearDesc), _P, _P, _P, _P, C.c_size_t, _P],
    "p4v_linear_frozen_path": [C.POINTER(LinearDesc), C.POINTER(C.c_int)],
    "p4v_linear_frozen_workspace_bytes": [C.POINTER(LinearDesc), C.POINTER(C.c_size_t)],
    "p4v_linear_frozen_forward": [C.POINTER(LinearDesc), _P, _P, _P, _P, C.c_size_t, _P, _P],
    "p4v_matmul_workspace_bytes": [C.POINTER(MatMulDesc), C.POINTER(C.c_size_t)],
    "p4v_matmul_score_log_floats": [C.POINTER(MatMulDesc), C.POINTER(C.c_size_t)],
    "p4v_matmul_calibrate": [C.POINTER(MatMulDesc), _P, _P, _P, _P, _P, C.c_size_t, _P, _P, _P, _P, _P],
    "p4v_matmul_quant_forward_workspace_bytes": [C.POINTER(MatMulDesc), C.POINTER(C.c_size_t)],
    "p4v_matmul_quant_forward": [C.POINTER(MatMulDesc), _P, _P, _P, _P, _P, _P, C.c_size_t, _P, _P],
    "p4v_matmul_pack_bytes": [C.POINTER(MatMulDesc), C.POINTER(C.c_size_t)],
    "p4v_matmul_pack": [C.POINTER(MatMulDesc), _P, _P, _P, _P, C.c_size_t, _P],
    "p4v_matmul_frozen_forward": [C.POINTER(MatMulDesc), _P, C.POINTER(C.c_longlong), _P, C.POINTER(C.c_longlong), _P, _P, _P],
    "p4v_attention_fused_ok": [C.c_int32, C.c_int32, C.POINTER(C.c_int)],
    "p4v_attention_frozen_forward": [C.POINTER(AttentionDesc), _P, C.POINTER(C.c_longlong), C.POINTER(MatMulDesc), _P, C.c_size_t,
                                     C.POINTER(MatMulDesc), _P, C.c_size_t, _P, _P, _P, _P],
    "p4v_attention_long_ok": [C.c_int32, C.c_int32, C.POINTER(C.c_int)],
    "p4v_attention_frozen_forward_long": [C.POINTER(AttentionDesc), _P, C.POINTER(C.c_longlong), C.POINTER(MatMulDesc), _P,
                                          C.c_size_t, C.POINTER(MatMulDesc), _P, C.c_size_t, _P, _P, _P, _P],
    "p4v_mlp_fused_ok": [C.POINTER(LinearDesc), C.POINTER(LinearDesc), C.POINTER(C.c_int)],
    "p4v_mlp_frozen_workspace_bytes": [C.POINTER(LinearDesc), C.POINTER(LinearDesc), C.POINTER(C.c_size_t)],
    "p4v_mlp_frozen_forward": [C.POINTER(LinearDesc), _P, _P, _P, C.c_size_t, C.POINTER(LinearDesc), _P, _P, C.c_size_t, _P,
                               C.c_size_t, _P, _P],
    "p4v_gelu_probe": [_P, _P, C.c_longlong, _P],
    "p4v_linear_norm_ok": [C.POINTER(LinearDesc), C.POINTER(C.c_int)],
    "p4v_mlp_norm_ok": [C.POINTER(LinearDesc), C.POINTER(LinearDesc), C.POINTER(C.c_int)],
    "p4v_linear_frozen_forward_norm": [C.POINTER(LinearDesc), _P, _P, _P, C.c_float, _P, _P, _P, _P],
    "p4v_mlp_frozen_forward_norm": [C.POINTER(LinearDesc), _P, _P, _P, C.c_float, _P, _P, C.c_size_t, C.POINTER(LinearDesc), _P,
                                    _P, C.c_size_t, _P, C.c_size_t, _P, _P],
    "p4v_layer_norm_probe": [_P, _P, _P, C.c_float, C.c_longlong, C.c_int, _P, _P],
    "p4v_linear_frozen_forward_res": [C.POINTER(LinearDesc), _P, _P, _P, _P, C.c_size_t, _P, C.POINTER(WindowLayout), _P, _P],
    "p4v_mlp_frozen_forward_res": [C.POINTER(LinearDesc), _P, _P, _P, C.c_size_t, C.POINTER(LinearDesc), _P, _P, C.c_size_t, _P,
                                   C.c_size_t, _P, _P, _P],
    "p4v_mlp_frozen_forward_norm_res": [C.POINTER(LinearDesc), _P, _P, _P, C.c_float, _P, _P, C.c_size_t, C.POINTER(LinearDesc),
                                        _P, _P, C.c_size_t, _P, C.c_size_t, _P, _P, _P],
    "p4v_linear_gather_ok": [C.POINTER(LinearDesc), C.POINTER(InputGather), C.POINTER(C.c_int)],
    "p4v_linear_frozen_forward_norm_gather": [C.POINTER(LinearDesc), _P, _P, _P, C.c_float, _P, _P, C.POINTER(InputGather), _P, _P],
    "p4v_linear_qkv8_ok": [C.POINTER(LinearDesc), C.POINTER(AttentionDesc), C.c_int, C.POINTER(C.c_int)],
    "p4v_linear_frozen_forward_qkv8": [C.POINTER(LinearDesc), _P, _P, _P, C.POINTER(AttentionDesc), C.POINTER(MatMulDesc), _P,
                                       C.c_size_t, C.POINTER(MatMulDesc), _P, C.c_size_t, _P, _P, _P, C.c_float,
                                       C.POINTER(InputGather), _P],
    "p4v_attention_frozen_forward_i8": [C.POINTER(AttentionDesc), _P, C.POINTER(MatMulDesc), _P, C.c_size_t, C.POINTER(MatMulDesc),
                                        _P, C.c_size_t, _P, _P, _P, _P],
    "p4v_conv_workspace_bytes": [C.POINTER(ConvDesc), C.POINTER(C.c_size_t)],
    "p4v_conv_calibrate": [C.POINTER(ConvDesc), _P, _P, _P, _P, _P, _P, C.c_size_t, _P, _P, _P],
    "p4v_conv_frozen_ok": [C.POINTER(ConvFrozenDesc), C.POINTER(C.c_int)],
    "p4v_conv_pack_bytes": [C.POINTER(ConvFrozenDesc), C.POINTER(C.c_size_t)],
    "p4v_conv_pack": [C.POINTER(ConvFrozenDesc), _P, _P, _P, C.c_size_t, _P],
    "p4v_conv_frozen_forward": [C.POINTER(ConvFrozenDesc), _P, _P, _P, C.c_size_t, _P, _P],
    "p4v_conv_pos_ok": [C.POINTER(ConvFrozenDesc), C.POINTER(C.c_int)],
    "p4v_conv_norm_ok": [C.POINTER(ConvFrozenDesc), C.POINTER(C.c_int)],
    "p4v_conv_frozen_forward_pos": [C.POINTER(ConvFrozenDesc), _P, _P, _P, C.c_size_t, _P, C.c_size_t, _P, C.c_size_t, _P, _P],
    "p4v_conv_frozen_forward_norm": [C.POINTER(ConvFrozenDesc), _P, _P, _P, C.c_size_t, _P, _P, C.c_size_t, C.c_float, _P, _P],
    "p4v_export_quantized": [_P, C.c_longlong, C.c_longlong, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float,
                             _P, _P, _P],
}
EXPORTS = sorted(list(_SIGNATURES) + ["p4v_last_error", "p4v_version", "p4v_launch_count", "p4v_profile_enable", "p4v_profile_collect",
                                     "p4v_profile_collect_kinds", "p4v_profile_collect_launches",
                                     "p4v_selftest_rint_div"])

_lib = None


def lib():
    """Load the shared library once.  Raises (never falls back) when it is absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -m ptq4vit_b200.build` (or __graft_entry__.build()). "
                "ptq4vit_b200 has no CPU / PyTorch fallback for the search path.")
        l = C.CDLL(LIB_PATH)
        for name, args in _SIGNATURES.items():
            fn = getattr(l, name)
            fn.argtypes = args
            fn.restype = C.c_int
        l.p4v_last_error.restype = C.c_char_p
        l.p4v_version.restype = C.c_int
        l.p4v_launch_count.restype = C.c_longlong
        l.p4v_profile_enable.argtypes = [C.c_int]
        l.p4v_selftest_rint_div.argtypes = [C.c_ulonglong, C.c_ulonglong, C.POINTER(C.c_ulonglong), C.c_void_p]
        l.p4v_profile_collect.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_longlong), C.POINTER(C.c_double)]
        l.p4v_profile_collect_kinds.argtypes = [C.POINTER(C.c_double), C.c_int]
        l.p4v_profile_collect_launches.argtypes = [C.POINTER(C.c_double), C.c_int, C.POINTER(C.c_int)]
        _lib = l
    return _lib


class NativeError(RuntimeError):
    pass


def check(rc, what):
    if rc != 0:
        raise NativeError(f"{what} failed (rc={rc}): {lib().p4v_last_error().decode()}")


def launch_count():
    return int(lib().p4v_launch_count())


def ptr(t):
    """Device pointer of a torch tensor (or NULL)."""
    return None if t is None else C.c_void_p(t.data_ptr())


def default_operand():
    return OPERAND[os.environ.get("P4V_OPERAND", "auto")]


def default_kernel():
    return KERNEL[os.environ.get("P4V_KERNEL", "tcgen05")]
