"""TEST-ONLY cross-check library binding (tests/xcheck/libmuse_b200_xcheck.so): first-generation mma.sync GEMM and
attention kernels with the product's argument conventions, used by the GPU tests as an independent on-device reference
for the wgmma kernels.  Not part of the product."""
import ctypes
from ctypes import c_char_p, c_float, c_int, c_void_p
from pathlib import Path

import torch

_LIB = None
_P, _I, _F = c_void_p, c_int, c_float


def load():
    global _LIB
    if _LIB is None:
        from open_muse_b200 import build

        lib = ctypes.CDLL(str(build.build_xcheck()))
        lib.xcheck_last_error.restype = c_char_p
        lib.xcheck_gemm_mma.argtypes = [_P, _P, _P, _P] + [_I] * 9 + [_P]
        lib.xcheck_attn_fwd.argtypes = [_P] * 5 + [_I] * 9 + [_F, _P]
        lib.xcheck_attn_bwd.argtypes = [_P] * 10 + [_I] * 13 + [_F, _P]
        _LIB = lib
    return _LIB


def _check(rc, what):
    if rc != 0:
        raise RuntimeError(f"{what}: {load().xcheck_last_error().decode()}")


def _st(t):
    return torch.cuda.current_stream(t.device.index).cuda_stream


def gemm(a, b, c, M, N, K, lda, ldb, ldc, a_mn=0, b_mn=0, epi=0, res=None):
    _check(load().xcheck_gemm_mma(a.data_ptr(), b.data_ptr(), c.data_ptr(), None if res is None else res.data_ptr(), M, N, K,
                                  lda, ldb, ldc, a_mn, b_mn, epi, _st(c)), "xcheck_gemm_mma")
    return c


def attn_fwd(q, k, v, B, nh, Sq, Skv, scale):
    o = torch.empty(B * Sq, nh * 64, dtype=torch.bfloat16, device=q.device)
    lse = torch.empty(B, nh, Sq, dtype=torch.float32, device=q.device)
    _check(load().xcheck_attn_fwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(), B, nh, Sq, Skv, 64,
                                  q.stride(0), k.stride(0), v.stride(0), o.stride(0), float(scale), _st(q)), "xcheck_attn_fwd")
    return o, lse


def attn_bwd(q, k, v, o, do, lse, dq, dk, dv, B, nh, Sq, Skv, scale):
    dvec = torch.empty(B, nh, Sq, dtype=torch.float32, device=q.device)
    _check(load().xcheck_attn_bwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), do.data_ptr(), lse.data_ptr(),
                                  dvec.data_ptr(), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), B, nh, Sq, Skv, 64, q.stride(0),
                                  k.stride(0), v.stride(0), o.stride(0), do.stride(0), dq.stride(0), dk.stride(0), dv.stride(0),
                                  float(scale), _st(q)), "xcheck_attn_bwd")
