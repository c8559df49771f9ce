"""ctypes binding of libmuse_b200.so (C ABI in include/muse_b200.h).

There is no CPU or PyTorch fallback: if the shared library is missing or a call fails, this module
raises.  The library is built in-tree by ``open_muse_b200.build`` / ``__graft_entry__.build()``.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_float, c_int, c_longlong, c_void_p, POINTER
from pathlib import Path

_PKG = Path(__file__).resolve().parent
LIB_PATH = _PKG / "libmuse_b200.so"

_lib = None

# name -> (restype, argtypes); mirrors include/muse_b200.h one to one
_P, _I, _L, _F = c_void_p, c_int, c_longlong, c_float
SIGNATURES = {
    "muse_abi_version": (c_int, []),
    "muse_last_error": (c_char_p, []),
    "muse_set_device": (c_int, [_I]),
    "muse_device_info": (c_int, [POINTER(c_int), POINTER(c_int), POINTER(c_int)]),
    "muse_reserve_sms": (c_int, [_I]),
    "muse_set_pdl": (c_int, [_I]),
    "muse_get_pdl": (c_int, []),
    "muse_gemm_bf16": (c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P]),
    "muse_gemm_fp8": (c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P]),
    "muse_gemm_fp8_res": (c_int, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P]),
    "muse_quantize_rows_e4m3": (c_int, [_P, _I, _P, _I, _P, _I, _I, _P]),
    "muse_gemm_splitk_workspace_bytes": (c_longlong, [_I, _I, _I]),
    "muse_gemm_bf16_splitk": (c_int, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _P, _L, _P]),
    "muse_pack_bf16": (c_int, [_P, _I, _L, _P]),
    "muse_adamw_ema_step": (c_int, [_P, _I, _P, _P, _P, _F, _F, _F, _F, _F, _I, _F, _F, _I, _I, _I, _F, _F, _P]),
    "muse_lion_ema_step": (c_int, [_P, _I, _P, _P, _P, _F, _F, _F, _F, _F, _F, _F, _I, _F, _F, _I, _I, _I, _F, _F, _P]),
    "muse_adamw8bit_ema_step": (c_int, [_P, _I, _P, _P, _P, _P, _F, _F, _F, _F, _F, _I, _F, _F, _I, _I, _I, _F, _F, _P]),
    "muse_cast_bf16": (c_int, [_P, _P, _L, _P]),
    "muse_embed_fwd": (c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "muse_embed_bwd": (c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "muse_embed_bwd_sorted_workspace_bytes": (c_longlong, [_I, _I, _I]),
    "muse_embed_bwd_sorted": (c_int, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "muse_norm_fwd": (c_int, [_P, _I, _P, _P, _P, _I, _P, _P, _P, _P, _I, _F, _I, _I, _F, _I, _I, _P]),
    "muse_norm_bwd": (c_int, [_P, _I, _P, _I, _P, _P, _P, _P, _P, _P, _F, _P, _I, _P, _P, _P, _I, _I, _I, _I, _P]),
    "muse_norm_bwd_workspace_floats": (c_longlong, [_I, _I, _I]),
    "muse_norm2_fwd": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _F, _I, _I, _P]),
    "muse_norm2_bwd": (c_int, [_P] * 15 + [_I, _I, _I, _I, _P]),
    "muse_norm_fwd_e4m3": (c_int, [_P, _I, _P, _P, _P, _P, _P, _P, _I, _I, _F, _I, _I, _P]),
    "muse_norm2_fwd_e4m3": (c_int, [_P] * 11 + [_I, _I, _F, _I, _I, _P]),
    "muse_glu_fwd": (c_int, [_P, _P, _I, _P, _P, _P, _I, _F, _L, _I, _P]),
    "muse_glu_bwd": (c_int, [_P, _P, _P, _F, _P, _L, _I, _P]),
    "muse_gelu_tanh_fwd": (c_int, [_P, _P, _I, _P, _L, _I, _P]),
    "muse_gelu_tanh_bwd": (c_int, [_P, _P, _P, _L, _I, _P]),
    "muse_attn_fwd": (c_int, [_P] * 7 + [_I, _F] + [_I] * 9 + [_F, _P]),
    "muse_attn_bwd": (c_int, [_P] * 6 + [_F] + [_P] * 4 + [_I] * 12 + [_F, _P]),
    "muse_dropout_fwd": (c_int, [_P, _P, _I, _P, _P, _I, _F, _L, _I, _P]),
    "muse_dropout_bwd": (c_int, [_P, _P, _I, _P, _F, _L, _I, _P]),
    "muse_ce_fwd": (c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _F, _P]),
    "muse_ce_bwd": (c_int, [_P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _F, _P]),
    "muse_add_norm_mod_fwd": (c_int, [_P, _I, _P, _P, _P, _L, _I, _P, _P, _I, _P, _I, _I, _F, _I, _P]),
    "muse_dwconv3x3_norm_fwd": (c_int, [_P, _P, _P, _P, _I, _P, _P, _I, _I, _I, _I, _F, _I, _P]),
    "muse_grn_fwd": (c_int, [_P] * 8 + [_I, _F, _I, _I, _I, _P]),
    "muse_add_norm_mod_bwd": (c_int, [_P, _I, _P, _P, _P, _P, _L, _I, _P, _I, _P, _P, _P, _I, _I, _F, _I, _P]),
    "muse_dwconv3x3_norm_bwd": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _F, _I, _P]),
    "muse_grn_bwd": (c_int, [_P] * 10 + [_F, _I, _I, _I, _P]),
    "muse_adaln_bwd": (c_int, [_P, _P, _P, _L, _P, _P, _I, _I, _I, _P]),
    "muse_silu_bwd": (c_int, [_P, _P, _I, _P, _I, _L, _I, _P]),
    "muse_adaln_apply": (c_int, [_P, _P, _L, _I, _I, _I, _P]),
    "muse_silu_bf16": (c_int, [_P, _I, _P, _L, _P]),
    "muse_vq_argmin": (c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _P]),
    "muse_vq_soft_code": (c_int, [_P, _P, _P, _P, _P, _P, _F, _I, _I, _I, _P]),
    "muse_vq_lookup_nchw": (c_int, [_P, _P, _P, _I, _I, _I, _I, _P]),
    "muse_sample_step": (c_int, [_P, _P, _L, _L, _F, _P, _P, _P, _P, _P, _P, _I, _I, _I, _L, _I, _F, _P]),
    "muse_conv2d_nhwc": (c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _P]),
    "muse_groupnorm_workspace_floats": (c_longlong, [_I, _I, _I]),
    "muse_groupnorm_silu_nhwc": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _F, _I, _I, _P]),
    "muse_spatial_groupnorm_silu_nhwc": (c_int, [_P] * 13 + [_I, _I, _I, _I, _I, _F, _I, _I, _I, _I, _I, _P]),
    "muse_split_s2d_bf16_nhwc": (c_int, [_P, _P, _P, _I, _I, _I, _I, _P]),
    "muse_softmax_split_rows": (c_int, [_P, _P, _P, _P, _L, _I, _F, _P]),
    "muse_conv2d_tc_tiles_per_image": (c_int, [_I, _I, _I, _I, _I, _I]),
    "muse_conv2d_tc_supported": (c_int, [_I, _I, _I, _I, _I]),
    "muse_conv2d_nhwc_tc": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _P]),
    "muse_conv2d_nhwc_tc_gelu_split": (c_int, [_P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _P]),
    "muse_im2col_split_nhwc": (c_int, [_P, _P, _P, _I, _I, _I, _I, _I, _P]),
    "muse_paella_resblock_spatial": (c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _F, _P]),
    "muse_split_bf16_nhwc": (c_int, [_P, _P, _P, _I, _I, _I, _I, _I, _P]),
    "muse_avgpool2_nhwc": (c_int, [_P, _P, _I, _I, _I, _I, _P]),
    "muse_image_to_uint8": (c_int, [_P, _P, _L, _P]),
    "muse_transpose_batched": (c_int, [_P, _P, _I, _I, _I, _P]),
}

ABI_VERSION = 11

# the mode argument of muse_conv2d_nhwc (enum muse_conv_mode): one geometry plus flags
CONV_SAME, CONV_UPSAMPLE2X, CONV_STRIDE2, CONV_S2P1, CONV_TRANSPOSE_S2 = 0, 1, 2, 3, 4
CONV_GEOMETRY, CONV_GELU, CONV_PIXEL_SHUFFLE = 7, 8, 16
# the mode argument of muse_conv2d_nhwc_tc / muse_conv2d_nhwc_tc_gelu_split (enum muse_conv_tc_mode)
CONV_TC_SAME, CONV_TC_UPSAMPLE2X, CONV_TC_FWD2X2, CONV_TC_GEOMETRY = 0, 1, 2, 3
CONV_TC_PER_IMAGE_WEIGHTS, CONV_TC_SINGLE_PASS, CONV_TC_PIXEL_SHUFFLE = 4, 8, 16


class MuseB200Error(RuntimeError):
    pass


def load():
    """Loads (once) and returns the ctypes handle; raises if the CUDA library is absent."""
    global _lib
    if _lib is not None:
        return _lib
    path = Path(os.environ.get("MUSE_B200_LIB", LIB_PATH))
    if not path.exists():
        raise MuseB200Error(
            f"{path} not found. Build it with `python -m open_muse_b200.build` (needs nvcc). "
            "open_muse_b200 has no CPU / PyTorch fallback for the hot path."
        )
    lib = ctypes.CDLL(str(path))
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as e:  # pragma: no cover
            raise MuseB200Error(f"{path} does not export {name}: stale build?") from e
        fn.restype = res
        fn.argtypes = args
    if lib.muse_abi_version() != ABI_VERSION:
        raise MuseB200Error(f"ABI mismatch: library {lib.muse_abi_version()} vs binding {ABI_VERSION}; rebuild")
    _lib = lib
    return lib


def check(status: int, what: str = ""):
    if status != 0:
        msg = load().muse_last_error()
        raise MuseB200Error(f"{what} failed (status {status}): {msg.decode() if msg else ''}")
