"""ctypes binding of libmtadgat.so (C ABI declared in include/mtadgat.h).

The library is the product: if it is missing or fails to load, importing this module raises -- there is
no CPU or eager-PyTorch fallback anywhere in the package.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmtadgat.so")

_P = ctypes.c_void_p
_I = ctypes.c_int
_F = ctypes.c_float
_U = ctypes.c_uint
_LL = ctypes.c_longlong
_ULL = ctypes.c_ulonglong

# name -> (restype, argtypes); mirrors include/mtadgat.h one to one
SIGNATURES = {
    "mtadgat_last_error": (ctypes.c_char_p, []),
    "mtadgat_abi_version": (_I, []),
    "mtadgat_launch_count": (ctypes.c_ulonglong, []),
    "mtadgat_reset_launch_count": (None, []),
    "mtadgat_conv_relu_fwd": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "mtadgat_conv_relu_bwd": (_I, [_P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "mtadgat_conv_relu_bwd3": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "mtadgat_conv_relu_fwd_strided": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _LL, _P]),
    "mtadgat_gat_saved_floats": (_LL, [_I, _I, _I, _I, _I, _I, _I]),
    "mtadgat_gat_bwd_scratch_floats": (_LL, [_I, _I, _I, _I, _I, _I]),
    "mtadgat_gat_fwd": (_I, [_P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _F, _I, _F, _P, _P]),
    "mtadgat_set_gat_impl": (_I, [_I]),
    "mtadgat_get_gat_impl": (_I, []),
    "mtadgat_gat_bwd": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _F, _F, _P, _I, _P]),
    "mtadgat_gru_saved_floats": (_LL, [_I, _I, _I, _I]),
    "mtadgat_gru_fwd_scratch_floats": (_LL, [_I, _I, _I]),
    "mtadgat_gru_bwd_scratch_floats": (_LL, [_I, _I, _I]),
    "mtadgat_gru_fwd": (_I, [_P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "mtadgat_gru_bwd": (_I, [_P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I,
                             _P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "mtadgat_rep_J": (_I, [_I, _I]),
    "mtadgat_gru_rep_saved_floats": (_LL, [_I, _I, _I, _I, _I]),
    "mtadgat_gru_rep_bwd_scratch_floats": (_LL, [_I, _I, _I, _I]),
    "mtadgat_gru_rep_fwd": (_I, [_P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P]),
    "mtadgat_gru_rep_bwd": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _I, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P]),
    "mtadgat_gru_rep_last": (_I, [_P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "mtadgat_score_epilogue": (_I, [_P, _P, _P, _P, _I, _I, _I, _LL, _F, _P, _P, _P]),
    "mtadgat_find_epsilon_scratch_doubles": (_LL, [_LL]),
    "mtadgat_find_epsilon": (_I, [_P, _LL, _I, _P, _P, _P]),
    "mtadgat_adam_step": (_I, [_P, _I, _LL, _F, _F, _F, _F, _P, _P]),
    "mtadgat_linear_fwd": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _F, _P, _U, _P]),
    "mtadgat_linear_bwd": (_I, [_P, _P, _P, _P, _P, _I, _P, _P, _P, _I, _I, _I, _I, _F, _P, _U, _I, _P]),
    "mtadgat_rmse_pair_fwd": (_I, [_P, _P, _LL, _P, _P, _LL, _P, _P, _P]),
    "mtadgat_rmse_pair_bwd": (_I, [_P, _P, _LL, _P, _P, _LL, _P, _P, _P, _P, _P, _P]),
    "mtadgat_set_gemm_impl": (_I, [_I]),
    "mtadgat_get_gemm_impl": (_I, []),
    "mtadgat_workspace_reserve": (_I, [_P, _LL]),
    "mtadgat_workspace_release": (None, []),
    "mtadgat_set_gru_impl": (_I, [_I]),
    "mtadgat_get_gru_impl": (_I, []),
    "mtadgat_set_gru_split": (_I, [_I]),
    "mtadgat_set_gru_bptt": (_I, [_I]),
    "mtadgat_gru_recurrence_fwd": (_I, [_P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _P]),
    "mtadgat_gru_recurrence_bwd": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _P]),
    "mtadgat_tc_probe": (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _P]),
    "mtadgat_gru_debug_buffer": (None, [_P]),
    "mtadgat_cpu_conv_relu_fwd": (_I, [_P, _P, _P, _P, _I, _I, _I, _I]),
    "mtadgat_cpu_conv_relu_bwd": (_I, [_P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I]),
    "mtadgat_cpu_gat_fwd": (_I, [_P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _F, _F, _ULL]),
    "mtadgat_cpu_gat_bwd": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _F, _F, _ULL]),
    "mtadgat_cpu_gru_fwd": (_I, [_P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I]),
    "mtadgat_cpu_gru_bwd": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I]),
    "mtadgat_cpu_linear_fwd": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _F, _ULL, _U]),
    "mtadgat_cpu_linear_bwd": (_I, [_P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _F, _ULL, _U]),
    "mtadgat_dropout_mask": (_I, [_P, _LL, _F, _P, _U, _P]),
    "mtadgat_seed_advance": (_I, [_P, _P]),
}


class MtadGatLibraryError(RuntimeError):
    pass


def _load():
    if not os.path.exists(LIB_PATH):
        raise MtadGatLibraryError(
            f"{LIB_PATH} not found: build the sm_90a library first (python __graft_entry__.py build). "
            "mtad_gat_pytorch_b200 has no CPU / eager fallback.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)       # AttributeError here = header/library mismatch
        fn.restype = res
        fn.argtypes = args
    return lib


lib = _load()


def check(rc):
    if rc != 0:
        raise MtadGatLibraryError(lib.mtadgat_last_error().decode("utf-8", "replace"))
