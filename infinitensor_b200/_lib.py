"""ctypes loader for libit_b200.so (the C-ABI of include/it_b200.h).

The product has no CPU fallback: if the CUDA library is missing or does not load,
importing this module raises -- loudly -- instead of routing anywhere else.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_double, c_float, c_int, c_int64, c_longlong, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
# ITB_LIB_PATH: load another BUILD of the same library (instrumented / A-B variants made by tools/); never a fallback
LIB_PATH = os.environ.get("ITB_LIB_PATH") or os.path.join(_HERE, "libit_b200.so")


class B200BackendError(RuntimeError):
    """The C spelling of infini::Exception (reference include/core/common.h:44-55)."""


if not os.path.exists(LIB_PATH):
    raise ImportError(
        f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
        "(make -C infinitensor_b200/csrc). There is no CPU fallback.")

lib = ctypes.CDLL(LIB_PATH)  # RTLD_LOCAL: the infini:: C++ symbols must not leak into other loaded libraries

i64p = POINTER(c_int64)
i32p = POINTER(c_int)
vp = c_void_p

_SIGS = {
    "it_b200_last_error": (c_char_p, []),
    "it_b200_version": (c_int, []),
    "it_b200_tune_skinny": (None, [c_int, c_int]),
    "it_b200_launch_count": (c_longlong, []),
    "it_b200_unary": (c_int, [c_int, c_int, vp, vp, c_int64, vp]),
    "it_b200_unary_alpha": (c_int, [c_int, c_int, vp, vp, c_int64, c_float, vp]),
    "it_b200_binary": (c_int, [c_int, c_int, vp, vp, vp, c_int, i64p, i64p, i64p, vp]),
    "it_b200_cast": (c_int, [c_int, c_int, vp, vp, c_int64, vp]),
    "it_b200_where": (c_int, [c_int, vp, vp, vp, vp, c_int, i64p, i64p, i64p, i64p, vp]),
    "it_b200_expand": (c_int, [c_int, vp, vp, c_int, i64p, i64p, vp]),
    "it_b200_softmax": (c_int, [c_int, vp, vp, c_int64, c_int, c_int64, vp]),
    "it_b200_layernorm": (c_int, [c_int, vp, vp, vp, vp, c_int64, c_int, c_int64, c_int, c_int, c_float, vp]),
    "it_b200_rmsnorm": (c_int, [c_int, vp, vp, vp, c_int64, c_int, vp]),
    "it_b200_rmsnorm_constw": (c_int, [c_int, vp, vp, vp, c_int64, c_int, vp]),
    "it_b200_rope": (c_int, [c_int, vp, c_int, vp, vp, c_int, c_int, c_int, c_int, vp]),
    "it_b200_rope_freq": (c_int, [c_int, vp, c_int, vp, vp, c_int, c_int, c_int, c_int, vp, c_int, c_int64, vp]),
    "it_b200_transpose": (c_int, [c_int, vp, vp, c_int, i64p, i32p, vp]),
    "it_b200_concat": (c_int, [c_int, c_int, POINTER(vp), i64p, vp, c_int64, c_int64, vp]),
    "it_b200_split": (c_int, [c_int, c_int, POINTER(vp), i64p, vp, c_int64, c_int64, vp]),
    "it_b200_gather": (c_int, [c_int, c_int, vp, vp, vp, c_int64, c_int64, c_int64, c_int64, vp]),
    "it_b200_copy": (c_int, [vp, vp, c_int64, vp]),
    "it_b200_pad_slice": (c_int, [c_int, vp, vp, c_int, i64p, i64p, i64p, i64p, vp]),
    "it_b200_reduce": (c_int, [c_int, c_int, vp, vp, c_int, i64p, i32p, vp]),
    "it_b200_pool2d": (c_int, [c_int, c_int, vp, vp] + [c_int] * 14 + [vp]),
    "it_b200_pool2d_nhwc": (c_int, [c_int, c_int, vp, vp] + [c_int] * 14 + [vp]),
    "it_b200_batchnorm": (c_int, [c_int, vp, vp, vp, vp, vp, vp, c_int, c_int, c_int64, c_float, vp]),
    "it_b200_matmul_select": (None, [c_int, c_int]),
    "it_b200_matmul_workspace": (c_int64, [c_int, c_int64, c_int, c_int, c_int]),
    "it_b200_matmul": (c_int, [c_int, vp, vp, vp, vp, c_int64, c_int, c_int, c_int, c_int64, c_int64, c_int, c_int,
                               c_int64, c_int64, c_int64, c_int, vp, c_int64, vp]),
    "it_b200_matmul_fused": (c_int, [c_int, vp, vp, vp, vp, vp, c_int64, c_int, c_int, c_int, c_int64, c_int64, c_int, c_int, c_int64, c_int64, c_int64, c_int, vp]),
    "it_b200_matmul_grouped": (c_int, [c_int, vp, c_int, POINTER(vp), POINTER(vp), i32p, c_int, c_int, vp]),
    "it_b200_silu_mul": (c_int, [c_int, vp, vp, vp, c_int64, vp]),
    "it_b200_matmul_fp8w": (c_int, [c_int, vp, c_int, POINTER(vp), POINTER(vp), POINTER(vp), i32p, c_int, c_int, vp, vp]),
    "it_b200_dequantize_fp8": (c_int, [c_int, vp, vp, vp, c_int64, c_int64, vp]),
    "it_b200_matmul_nbits_workspace": (c_int64, [c_int, c_int, c_int, c_int, i32p]),
    "it_b200_matmul_nbits": (c_int, [c_int, vp, c_int, POINTER(vp), POINTER(vp), POINTER(vp), POINTER(vp), i32p, c_int, c_int, c_int,
                                     vp, vp, c_int64, vp]),
    "it_b200_dequantize_w4": (c_int, [c_int, vp, vp, vp, vp, c_int, c_int, c_int, vp]),
    "it_b200_allreduce_workspace_bytes": (c_int64, []),
    "it_b200_allreduce_fused": (c_int, [c_int, vp, vp, vp, vp, vp, c_int, c_int, POINTER(vp), c_int, c_int, vp, vp]),
    "it_b200_batchnorm_relu": (c_int, [c_int, vp, vp, vp, vp, vp, vp, c_int, c_int, c_int64, c_float, vp]),
    "it_b200_conv2d_fused": (c_int, [c_int, vp, vp, vp] + [c_int] * 14 + [vp, vp, vp, vp, c_float, vp, c_int, vp, c_int64, vp]),
    "it_b200_conv2d_workspace": (c_int64, [c_int] * 15),
    "it_b200_conv2d_nchw_to_nhwc_supported": (c_int, [c_int] * 15),
    "it_b200_conv2d_fused_nhwc_out": (c_int, [c_int, vp, vp, vp] + [c_int] * 14 + [vp, vp, vp, vp, c_float, vp, c_int, vp, c_int64, vp]),
    "it_b200_conv2d_stem_supported": (c_int, [c_int] * 12),
    "it_b200_conv2d_stem": (c_int, [c_int, vp, vp, vp] + [c_int] * 11 + [vp, vp, vp, vp, c_float, c_int, vp]),
    "it_b200_conv2d_nhwc_supported": (c_int, [c_int] * 12),
    "it_b200_conv_repack_filters": (c_int, [c_int, c_int, vp, vp, vp, vp, vp, vp, vp]),
    "it_b200_conv2d_nhwc_workspace": (c_int64, [c_int] * 5),
    "it_b200_conv2d_nhwc": (c_int, [c_int, vp, vp, vp] + [c_int] * 14 + [vp, vp, vp, vp, c_float, vp, c_int, vp, c_int64, vp]),
    "it_b200_conv2d": (c_int, [c_int, vp, vp, vp] + [c_int] * 14 + [vp, c_int64, vp]),
    "it_b200_attention_kvcache_workspace": (c_int64, [c_int] * 4),
    "it_b200_attention_kvcache_rope": (c_int, [c_int, vp, vp, vp, vp, vp, vp, c_int, vp, c_int, vp, c_int, c_int, c_int, c_int,
                                               vp, c_int64, vp]),
    "it_b200_attention_kvcache": (c_int, [c_int, vp, vp, vp, vp, vp, vp, c_int, vp, c_int, c_int, c_int, c_int,
                                          vp, c_int64, vp]),
    "it_b200_attention_kvcache_gqa": (c_int, [c_int, vp, vp, vp, vp, vp, vp, c_int, vp, c_int, vp, c_int, c_int, c_int, c_int,
                                              c_int, vp, c_int64, vp]),
    "it_b200_attention_kvcache_fp8": (c_int, [c_int, vp, vp, vp, vp, vp, vp, vp, vp, c_int, vp, c_int, vp, c_int, c_int, c_int,
                                              c_int, c_int, vp, c_int64, vp]),
    "it_b200_attention_kvcache_gqa_freq": (c_int, [c_int, vp, vp, vp, vp, vp, vp, c_int, vp, c_int, vp, c_int, c_int64, vp, c_int,
                                                   c_int, c_int, c_int, c_int, vp, c_int64, vp]),
    "it_b200_attention_kvcache_fp8_freq": (c_int, [c_int, vp, vp, vp, vp, vp, vp, vp, vp, c_int, vp, c_int, vp, c_int, c_int64, vp,
                                                   c_int, c_int, c_int, c_int, c_int, vp, c_int64, vp]),
    "it_b200_attention_kvcache_prompt": (c_int, [c_int, vp, vp, vp, vp, vp, vp, c_int, vp] + [c_int] * 6 + [vp]),
    "it_b200_attention_kvcache_window": (c_int, [c_int, vp, vp, vp, vp, vp, vp, vp, vp, c_int, vp, c_int, c_int64, c_int, vp, c_int,
                                                 vp, c_int, c_int, c_int, c_int, c_int, vp, c_int64, vp]),
    "it_b200_attention_kvcache_prompt_window": (c_int, [c_int, vp, vp, vp, vp, vp, vp, c_int, vp] + [c_int] * 7 + [vp]),
    "it_b200_attention_prefill": (c_int, [c_int, vp, vp, vp, vp, c_int, c_int, c_int, c_int, c_int, vp, c_int, vp, c_int64, c_int64,
                                          c_int64, c_int64, vp]),
    "it_b200_attention_prefill_strided": (c_int, [c_int, vp, vp, vp, vp] + [c_int] * 5 + [vp, vp, vp, vp, vp, c_int, vp, c_int64, c_int64, c_int64, c_int64, vp]),
}


for _name, (_res, _args) in _SIGS.items():
    _f = getattr(lib, _name)
    _f.restype = _res
    _f.argtypes = _args


def last_error() -> str:
    return lib.it_b200_last_error().decode()


def check(ret: int) -> None:
    if ret != 0:
        raise B200BackendError(last_error())


def i64arr(v):
    return (c_int64 * len(v))(*[int(x) for x in v])


def i32arr(v):
    return (c_int * len(v))(*[int(x) for x in v])


def exported_symbols():
    return sorted(_SIGS)
