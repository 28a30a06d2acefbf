"""ctypes binding of libmagvit2_b200.so (the C ABI declared in include/magvit2_b200.h).

There is no CPU fallback and no JIT: the shared library must have been built in-tree
(``python __graft_entry__.py`` / ``magvit2_pytorch_b200/csrc/build.sh``); a missing library
or a missing symbol raises immediately.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("MV2_LIB_PATH") or os.path.join(_HERE, "libmagvit2_b200.so")   # env override: A/B builds

MV2_F32, MV2_BF16, MV2_U8, MV2_F16, MV2_TF32 = 0, 1, 2, 3, 4
MV2_KWPACK_F32_DST = 0x100     # OR'd into mv2_ingest_kwpack's source dtype: fp32 destination (the TF32 conv_in)
ACT_NONE, ACT_ELU, ACT_SILU, ACT_LEAKY_RELU, ACT_RELU = 0, 1, 2, 3, 4
SHUFFLE_NONE, SHUFFLE_SPACE, SHUFFLE_TIME = 0, 1, 2


class Mv2Error(RuntimeError):
    pass


class ConvArgs(C.Structure):
    _fields_ = [
        ("x", C.c_void_p), ("w", C.c_void_p), ("bias", C.c_void_p), ("res", C.c_void_p), ("y", C.c_void_p),
        ("dtype", C.c_int32),
        ("B", C.c_int32), ("Ti", C.c_int32), ("Hi", C.c_int32), ("Wi", C.c_int32), ("Ci", C.c_int32),
        ("To", C.c_int32), ("Ho", C.c_int32), ("Wo", C.c_int32), ("Co", C.c_int32),
        ("kt", C.c_int32), ("kh", C.c_int32), ("kw", C.c_int32),
        ("st", C.c_int32), ("sh", C.c_int32), ("sw", C.c_int32),
        ("pt", C.c_int32), ("ph", C.c_int32), ("pw", C.c_int32),
        ("act", C.c_int32), ("shuffle", C.c_int32), ("x_token_shift", C.c_int32),
        ("oscale", C.c_void_p),
    ]


class AttnArgs(C.Structure):
    _fields_ = [
        ("qkv", C.c_void_p), ("out", C.c_void_p), ("mem_kv", C.c_void_p),
        ("dtype", C.c_int32), ("heads", C.c_int32), ("dim_head", C.c_int32), ("n_mem", C.c_int32),
        ("causal", C.c_int32),
        ("n_outer", C.c_int32), ("n_inner", C.c_int32), ("L", C.c_int32),
        ("outer_stride", C.c_int64), ("inner_stride", C.c_int64), ("tok_stride", C.c_int64),
    ]


class DropoutArgs(C.Structure):
    """mv2_dropout_args (attention dropout; see include/magvit2_b200.h)."""
    _fields_ = [("seed", C.c_uint64), ("call", C.c_uint32), ("p", C.c_float)]


class TcConvArgs(C.Structure):
    """mv2_tc_conv_args (wgmma implicit-GEMM path; see include/magvit2_b200.h)."""
    _fields_ = [
        ("x", C.c_void_p), ("w", C.c_void_p), ("bias", C.c_void_p), ("res", C.c_void_p), ("y", C.c_void_p),
        ("B", C.c_int32), ("Ti", C.c_int32), ("Hi", C.c_int32), ("Wi", C.c_int32), ("Ci", C.c_int32),
        ("To", C.c_int32), ("Ho", C.c_int32), ("Wo", C.c_int32), ("Co", C.c_int32),
        ("kt", C.c_int32), ("kh", C.c_int32), ("kw", C.c_int32),
        ("st", C.c_int32), ("sh", C.c_int32), ("sw", C.c_int32),
        ("pt", C.c_int32), ("ph", C.c_int32), ("pw", C.c_int32),
        ("act", C.c_int32), ("shuffle", C.c_int32), ("epi_mode", C.c_int32),
        ("oscale", C.c_void_p), ("out_layout", C.c_int32),
        ("dtype", C.c_int32),    # MV2_F16, MV2_TF32, or MV2_BF16 (also 0)
    ]


class TcRuArgs(C.Structure):
    """mv2_tc_ru_args (fused ResidualUnit front half; see include/magvit2_b200.h)."""
    _fields_ = [
        ("x", C.c_void_p), ("w3", C.c_void_p), ("b3", C.c_void_p), ("w1", C.c_void_p), ("b1", C.c_void_p),
        ("se_wk", C.c_void_p), ("se_bk", C.c_float), ("dtype", C.c_int32), ("y", C.c_void_p), ("se_ws", C.c_void_p),
        ("B", C.c_int32), ("T", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("C", C.c_int32),
        ("kt", C.c_int32), ("kh", C.c_int32), ("kw", C.c_int32),
    ]


class ConvHist(C.Structure):
    """mv2_conv_hist (frames in front of a streamed chunk; see include/magvit2_b200.h)."""
    _fields_ = [("h", C.c_void_p), ("T_h", C.c_int32), ("clip_stride", C.c_int64)]


# name -> (restype, argtypes); must list every symbol include/magvit2_b200.h declares
_VP, _I, _I64, _F, _SZ = C.c_void_p, C.c_int, C.c_int64, C.c_float, C.c_size_t
SIGNATURES = {
    "mv2_abi_version": (_I, []),
    "mv2_last_error": (C.c_char_p, []),
    "mv2_launch_count": (C.c_uint64, []),
    "mv2_device_arch": (_I, []),
    "mv2_set_pdl": (_I, [_I]),
    "mv2_to_channels_last": (_I, [_VP, _I, _VP, _I, _I, _I, _I, _I, _I, _I, _VP]),
    "mv2_to_channels_first": (_I, [_VP, _I, _VP, _I, _I, _I, _I, _I, _I, _I, _VP]),
    "mv2_ingest_kwpack": (_I, [_VP, _I, _VP, _I, _I, _I, _I, _I, _I, _I, _I, _I, _VP]),
    "mv2_copy_frames": (_I, [_VP, _VP, _I, _I, _I, _I, _I, _I, _SZ, _I, _VP]),
    "mv2_pad_cl": (_I, [_VP, _VP, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _VP]),
    "mv2_conv_forward": (_I, [C.POINTER(ConvArgs), C.POINTER(ConvHist), _VP]),
    "mv2_se_workspace_bytes": (_SZ, [_I, _I, _I]),
    "mv2_se_pool": (_I, [_VP, _I, _I, _I, _I, _VP, _F, _VP, _VP]),
    "mv2_se_gate": (_I, [_VP, _I, _I, _I, _I, _I, _VP, _VP, _VP, _VP, _VP, _VP]),
    "mv2_gate_residual": (_I, [_VP, _VP, _VP, _VP, _I, _I, _I, _I, _VP]),
    "mv2_rmsnorm": (_I, [_VP, _VP, _I, _VP, _I, _I, _I, _I, _I, _VP]),
    "mv2_attention": (_I, [C.POINTER(AttnArgs), _VP]),
    "mv2_attention_dropout": (_I, [C.POINTER(AttnArgs), C.POINTER(DropoutArgs), _VP]),
    "mv2_attention_dropout_mask": (_I, [_I, _I, _I, _I, C.POINTER(DropoutArgs), _VP, _VP]),
    "mv2_linattn_workspace_bytes": (_SZ, [_I, _I, _I]),
    "mv2_linear_attention": (_I, [_VP, _VP, _VP, _I, _I, _I, _I, _I, _VP, _VP]),
    "mv2_geglu": (_I, [_VP, _VP, _I, _I64, _I, _VP]),
    "mv2_lfq_forward": (_I, [_VP, _I, _I64, _I, _I, _I, _VP, _VP, _VP, _VP, _F, _I, _VP, _VP, _VP, _VP]),
    "mv2_lfq_decode": (_I, [_VP, _I, _I64, _I, _I, _I, _VP, _VP, _VP, _I, _VP]),
    "mv2_fsq_forward": (_I, [_VP, _I, _I64, _I, _I, _I, C.POINTER(C.c_int32), _VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP]),
    "mv2_fsq_decode": (_I, [_VP, _I, _I64, _I, _I, _I, C.POINTER(C.c_int32), _VP, _VP, _VP, _I, _VP]),
    "mv2_lfq_entropy_partials": (_I, [_VP, _I64, _I, _I, _F, _VP, _VP, _VP]),
    "mv2_lfq_aux_finalize": (_I, [_VP, _VP, _I, _I, _I64, _I64, _F, _F, _F, _VP, _VP]),
    "mv2_lfq_entropy_fact_workspace_bytes": (_SZ, [_I64, _I, _I]),
    "mv2_lfq_entropy_fact_partials": (_I, [_VP, _I64, _I, _I, _F, _VP, _VP, _VP, _VP]),
    "mv2_lfq_entropy_fact_backward": (_I, [_VP, _VP, _I64, _I, _I, _F, _F, _F, _VP, _VP, _VP]),
    "mv2_gateloop_scan": (_I, [_VP, _VP, _VP, _I, _I, _I, _I, _I, _VP]),
    "mv2_mse": (_I, [_VP, _I, _VP, _I, _I64, _VP, _VP, _VP]),
    "mv2_mse_workspace_bytes": (C.c_size_t, []),
    "mv2_maxpool2x2": (_I, [_VP, _VP, _I, _I, _I, _I, _I, _VP]),
    "mv2_maxpool2x2_backward": (_I, [_VP, _VP, _VP, _I, _I, _I, _I, _I, _VP]),
    "mv2_tc_conv_supported": (_I, [C.POINTER(TcConvArgs)]),
    "mv2_tc_conv_forward": (_I, [C.POINTER(TcConvArgs), C.POINTER(ConvHist), _VP]),
    "mv2_tc_slab_supported": (_I, [C.POINTER(TcConvArgs)]),
    "mv2_tc_slab_forward": (_I, [C.POINTER(TcConvArgs), C.POINTER(ConvHist), _VP]),
    "mv2_tc_down_space_supported": (_I, [C.POINTER(TcConvArgs)]),
    "mv2_tc_down_space_forward": (_I, [C.POINTER(TcConvArgs), _VP]),
    "mv2_tc_slab_plan": (_I, [C.POINTER(TcConvArgs), _I, C.POINTER(C.c_int32)]),
    "mv2_tc_slab_tile": (_I, [C.POINTER(TcConvArgs), _I, _I, _I, C.POINTER(C.c_int32)]),
    "mv2_dense_small": (_I, [_VP, _VP, _VP, _VP, _I, _I, _I, _I, _VP]),
    "mv2_mod_prepare": (_I, [_VP, _VP, _F, _VP, _VP, _I, _I, _I, _VP]),
    "mv2_scale_channels": (_I, [_VP, _VP, _VP, _I, _I, _I64, _I, _VP]),
    "mv2_tc_ru_supported": (_I, [C.POINTER(TcRuArgs)]),
    "mv2_tc_ru_records": (_I, [C.POINTER(TcRuArgs)]),
    "mv2_tc_ru_workspace_bytes": (_SZ, [C.POINTER(TcRuArgs)]),
    "mv2_tc_ru_forward": (_I, [C.POINTER(TcRuArgs), C.POINTER(ConvHist), _VP]),
    "mv2_se_gate_records": (_I, [_VP, _I, _I, _I, _I, _VP, _VP, _VP, _VP, _VP, _VP]),
    "mv2_rmsnorm_prev": (_I, [_VP, _VP, _I64, _VP, _I, _VP, _I, _I, _I, _I, _VP]),
    "mv2_attention_tail": (_I, [C.POINTER(AttnArgs), _VP, _I64, _I, _VP, _I64, _VP]),
    "mv2_tc_conv_hist_supported": (_I, [C.POINTER(TcConvArgs)]),
    "mv2_gateloop_scan_state": (_I, [_VP, _VP, _VP, _I, _I, _I, _I, _I, _VP, _VP]),
}

_lib = None


def load():
    """Load the library and bind every declared symbol; raises if anything is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise Mv2Error(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU / eager fallback)")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as e:
            raise Mv2Error(f"libmagvit2_b200.so does not export {name}") from e
        fn.restype = res
        fn.argtypes = args
    ver = lib.mv2_abi_version()
    if ver != 5:
        raise Mv2Error(f"ABI version mismatch: library {ver}, binding 5")
    _lib = lib
    return lib


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = load().mv2_last_error()
        raise Mv2Error(f"{what} failed with code {rc}: {msg.decode() if msg else ''}")
