"""Thin tensor-level wrappers over the C ABI (pointers, sizes, current CUDA stream).

PyTorch here is plumbing only: device memory (``torch.empty``), streams, autograd bookkeeping.
Every function launches hand-written sm_90a kernels from libmuse_b200.so and raises if the
library is missing or the tensors are not CUDA tensors -- there is no fallback path.
"""
from __future__ import annotations

import os
import weakref
from typing import NamedTuple

import torch

from . import _lib
from ._lib import (CONV_GELU, CONV_PIXEL_SHUFFLE, CONV_S2P1, CONV_SAME, CONV_STRIDE2, CONV_TC_FWD2X2,
                   CONV_TC_PER_IMAGE_WEIGHTS, CONV_TC_PIXEL_SHUFFLE, CONV_TC_SAME, CONV_TC_SINGLE_PASS, CONV_TC_UPSAMPLE2X,
                   CONV_TRANSPOSE_S2, CONV_UPSAMPLE2X)

F32, BF16, E4M3 = 0, 1, 2
FP8 = torch.float8_e4m3fn


class F8(NamedTuple):
    """An e4m3 GEMM operand with one fp32 scale per row: row r stands for q[r] * s[r] (the producers store
    e4m3_rn_satfinite(y / s) with s = amax(|y[r]|) / 448, or 1 for an all-zero row)."""
    q: torch.Tensor  # torch.float8_e4m3fn [rows, K]
    s: torch.Tensor  # fp32 [rows]

    @property
    def shape(self):
        return self.q.shape

EPI_BF16, EPI_F32, EPI_ATOMIC_F32, EPI_RESADD_F32 = 0, 1, 2, 3

_state = {"device": None, "launches": 0}


def reserve_sms(n: int):
    """Data-parallel training: leave n SMs to the NCCL all-reduce kernels that overlap backward (the persistent GEMMs then
    launch SM-count - n CTAs).  Pair it with NCCL_MAX_NCHANNELS=n (set before init_process_group)."""
    _lib.check(_lib.load().muse_reserve_sms(int(n)), "muse_reserve_sms")


def set_pdl(enabled: bool):
    """Programmatic dependent launch for every kernel of the library (include/muse_b200.h: muse_set_pdl).  Process-wide;
    call it before capturing CUDA graphs."""
    _lib.check(_lib.load().muse_set_pdl(1 if enabled else 0), "muse_set_pdl")


def get_pdl() -> bool:
    return bool(_lib.load().muse_get_pdl())


def launches() -> int:
    """Number of libmuse_b200 kernel-launching calls made so far (bench.py's gpu_launches)."""
    return _state["launches"]


def _prep(t: torch.Tensor):
    if not t.is_cuda:
        raise _lib.MuseB200Error("open_muse_b200 ops need CUDA tensors (no CPU fallback)")
    dev = t.device.index
    # the library's runtime must target the tensor's device; the user may have called torch.cuda.set_device since the
    # last op, so compare against torch's current device rather than a cached value
    if _state["device"] != dev or torch.cuda.current_device() != dev:
        _lib.check(_lib.load().muse_set_device(dev), "muse_set_device")
        _state["device"] = dev
    return torch.cuda.current_stream(dev).cuda_stream


def _dt(t: torch.Tensor) -> int:
    if t.dtype == torch.float32:
        return F32
    if t.dtype == torch.bfloat16:
        return BF16
    if t.dtype == FP8:
        return E4M3
    raise TypeError(f"unsupported dtype {t.dtype}")


def _new_out(rows, cols, dtype, device):
    """(output, its row scales or None): an F8 pair for dtype FP8, else a plain tensor"""
    y = torch.empty(rows, cols, dtype=dtype, device=device)
    if dtype != FP8:
        return y, None
    s = torch.empty(rows, dtype=torch.float32, device=device)
    return F8(y, s), s


def _data(y):
    return y.q if isinstance(y, F8) else y


def _p(t):
    return None if t is None else t.data_ptr()


_KERNELS_PER_CALL = {"muse_norm2_bwd": 3, "muse_sample_step": 2, "muse_gemm_bf16_splitk": 2, "muse_adamw_ema_step": 4, "muse_lion_ema_step": 4, "muse_ce_fwd": 2, "muse_attn_bwd": 2, "muse_embed_bwd": 2, "muse_embed_bwd_sorted": 4, "muse_vq_argmin": 2, "muse_vq_soft_code": 3,
                     "muse_groupnorm_silu_nhwc": 3, "muse_spatial_groupnorm_silu_nhwc": 3, "muse_grn_fwd": 3, "muse_grn_bwd": 3,
                     "muse_dwconv3x3_norm_bwd": 2}
_prof = {"on": False, "events": []}


def _call(name, *args):
    _state["launches"] += _KERNELS_PER_CALL.get(name, 1)
    _lib.check(getattr(_lib.load(), name)(*args), name)


def profile_gemms(enable: bool):
    """bench.py hook: while enabled every GEMM launch is bracketed by CUDA events on its stream.
    Disabling returns (total_ms, total_flops, n_launches)."""
    if enable:
        _prof["on"], _prof["events"] = True, []
        return None
    _prof["on"] = False
    torch.cuda.synchronize()
    ms = sum(a.elapsed_time(b) for a, b, _ in _prof["events"])
    fl = sum(f for _, _, f in _prof["events"])
    n = len(_prof["events"])
    _prof["events"] = []
    return ms, fl, n


# ------------------------------------------------------------------------------------------ GEMM
def gemm(a, b, c, M, N, K, lda, ldb, ldc, a_mn=0, b_mn=0, epi=EPI_BF16, res=None):
    st = _prep(c)
    if _prof["on"]:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    _call("muse_gemm_bf16", _p(a), _p(b), _p(c), _p(res), M, N, K, lda, ldb, ldc, a_mn, b_mn, epi, st)
    if _prof["on"]:
        e1.record()
        _prof["events"].append((e0, e1, 2.0 * M * N * K))
    return c


def gemm_fp8(a: F8, b: F8, c, M, N, K, lda, ldb, ldc):
    """c bf16 [M,N] = (a.q * a.s[:, None]) @ (b.q * b.s[:, None])^T with the e4m3 tensor cores (fp32 accumulation)."""
    st = _prep(c)
    if _prof["on"]:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    _call("muse_gemm_fp8", _p(a.q), _p(a.s), _p(b.q), _p(b.s), _p(c), M, N, K, lda, ldb, ldc, st)
    if _prof["on"]:
        e1.record()
        _prof["events"].append((e0, e1, 2.0 * M * N * K))
    return c


def gemm_fp8_res(a: F8, b: F8, res, c, M, N, K, lda, ldb, ldc):
    """c fp32 [M,N] = res + bf16((a.q * a.s[:, None]) @ (b.q * b.s[:, None])^T): gemm_fp8 with the residual add of
    EPI_RESADD_F32 fused into its epilogue (res and c fp32 with pitch ldc)."""
    st = _prep(c)
    if _prof["on"]:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    _call("muse_gemm_fp8_res", _p(a.q), _p(a.s), _p(b.q), _p(b.s), _p(res), _p(c), M, N, K, lda, ldb, ldc, st)
    if _prof["on"]:
        e1.record()
        _prof["events"].append((e0, e1, 2.0 * M * N * K))
    return c


def quantize_rows_e4m3(x, out: F8 | None = None) -> F8:
    """bf16 [rows, K] -> F8 with one scale per row (the FP8 weight operands); out: an F8 of the same shape to refresh in
    place (graph-capturable)."""
    st = _prep(x)
    rows, K = x.shape
    if out is None:
        out = F8(torch.empty(rows, K, dtype=FP8, device=x.device), torch.empty(rows, dtype=torch.float32, device=x.device))
    _call("muse_quantize_rows_e4m3", _p(x), x.stride(0), _p(out.q), out.q.stride(0), _p(out.s), rows, K, st)
    return out


def linear_fwd(x, w, out_dtype=torch.bfloat16, res=None, n_valid=None):
    """y[T,N] = x[T,K] @ w[N,K]^T.  res (fp32 [T,N]) selects the fused residual epilogue (fp32 output).  x and w both
    F8: the FP8 GEMM, with a bf16 output, or with res the fp32 output res + bf16(x @ w^T)."""
    if isinstance(x, F8):
        if not isinstance(w, F8) or (res is None and out_dtype != torch.bfloat16):
            raise TypeError("linear_fwd: an F8 activation needs an F8 weight, and a bf16 output without a residual")
        T, K = x.q.shape
        N = w.q.shape[0] if n_valid is None else n_valid
        if res is not None:
            y = torch.empty(T, N, dtype=torch.float32, device=x.q.device)
            return gemm_fp8_res(x, w, res, y, T, N, K, x.q.stride(0), w.q.stride(0), N)
        y = torch.empty(T, N, dtype=torch.bfloat16, device=x.q.device)
        return gemm_fp8(x, w, y, T, N, K, x.q.stride(0), w.q.stride(0), N)
    T, K = x.shape
    N = w.shape[0] if n_valid is None else n_valid
    if res is not None:
        y = torch.empty(T, N, dtype=torch.float32, device=x.device)
        return gemm(x, w, y, T, N, K, x.stride(0), w.stride(0), N, 0, 0, EPI_RESADD_F32, res)
    y = torch.empty(T, N, dtype=out_dtype, device=x.device)
    return gemm(x, w, y, T, N, K, x.stride(0), w.stride(0), N, 0, 0, EPI_BF16 if out_dtype == torch.bfloat16 else EPI_F32)


def linear_dgrad(dy, w, out_dtype=torch.bfloat16):
    """dx[T,K] = dy[T,N] @ w[N,K]  (w consumed as an MN-major B operand; no transpose copy)."""
    T, N = dy.shape
    K = w.shape[1]
    dx = torch.empty(T, K, dtype=out_dtype, device=dy.device)
    return gemm(dy, w, dx, T, K, N, dy.stride(0), w.stride(0), K, 0, 1, EPI_BF16 if out_dtype == torch.bfloat16 else EPI_F32)


def linear_dgrad_acc(dy, w, acc):
    """acc[T,K] (fp32) += dy[T,N] @ w[N,K]: gradients of a tensor consumed by many GEMMs (text states of U-ViT)."""
    T, N = dy.shape
    K = w.shape[1]
    return gemm(dy, w, acc, T, K, N, dy.stride(0), w.stride(0), acc.stride(0), 0, 1, EPI_ATOMIC_F32)


def linear_wgrad(dy, x, dw):
    """dw[N,K] += dy[T,N]^T @ x[T,K]  (both operands MN-major, split-K over tokens, fp32 atomics: accumulating but
    order-dependent; the MaskGiTUViT_v2 training path, whose gradients are summed across blocks)."""
    T, N = dy.shape
    K = x.shape[1]
    return gemm(dy, x, dw, N, K, T, dy.stride(0), x.stride(0), dw.stride(0), 1, 1, EPI_ATOMIC_F32)


def linear_wgrad_det(dy, x, out=None):
    """dw[N,K] = dy[T,N]^T @ x[T,K], run-to-run bit-identical: split-K partial tiles go to a workspace and an ordered
    reduction kernel sums them in split order and stores dw (no zero fill, no atomics on dw)."""
    st = _prep(dy)
    T, N = dy.shape
    K = x.shape[1]
    dev = dy.device
    dw = out if out is not None else torch.empty(N, K, dtype=torch.float32, device=dev)
    need = _lib.load().muse_gemm_splitk_workspace_bytes(N, K, T)
    ws = torch.empty(max(need, 16) // 4, dtype=torch.float32, device=dev)
    if _prof["on"]:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    _call("muse_gemm_bf16_splitk", _p(dy), _p(x), _p(dw), N, K, T, dy.stride(0), x.stride(0), dw.stride(0), 1, 1, _p(ws),
          need, st)
    if _prof["on"]:
        e1.record()
        _prof["events"].append((e0, e1, 2.0 * N * K * T))
    return dw


# ------------------------------------------------------------------------------------------ packing
def pack_bf16(table_dev, n_entries, total_blocks):
    st = _prep(table_dev)
    _call("muse_pack_bf16", _p(table_dev), n_entries, total_blocks, st)


def cast_bf16(src):
    st = _prep(src)
    dst = torch.empty(src.shape, dtype=torch.bfloat16, device=src.device)
    _call("muse_cast_bf16", _p(src), _p(dst), src.numel(), st)
    return dst


# ------------------------------------------------------------------------------------------ embedding
def embed_fwd(ids, word, pos):
    st = _prep(word)
    B, S = ids.shape
    H = word.shape[1]
    out = torch.empty(B * S, H, dtype=torch.float32, device=word.device)
    _call("muse_embed_fwd", _p(ids), _p(word), _p(pos), _p(out), B, S, H, word.shape[0], st)
    return out


def embed_bwd(ids, dx, dword, dpos):
    """dword[ids] += dx with atomics (dword zero-filled by the caller; order-dependent), dpos[:S] stored."""
    st = _prep(dx)
    B, S = ids.shape
    _call("muse_embed_bwd", _p(ids), _p(dx), _p(dword), _p(dpos), B, S, dword.shape[1], dword.shape[0], st)


_arange_cache = {}


def embed_bwd_det(ids, dx, vocab, n_pos):
    """Reproducible embedding backward: returns (dword [vocab, H], dpos [n_pos, H] or None when n_pos == 0), every row
    stored, token contributions summed in ascending token order.  The stable sort of the ids is index preparation (ATen);
    the data path is muse_embed_bwd_sorted."""
    st = _prep(dx)
    B, S = ids.shape
    H = dx.shape[1]
    dev = dx.device
    flat = ids.reshape(-1)
    # ids outside [0, vocab) are clamped to the sentinel `vocab`: they sort behind every real id and are ignored, like the
    # forward kernel ignores them.  16-bit keys when they fit (vocab < 32767): the radix sort then needs 2 passes, not 8.
    kdt = torch.int16 if vocab < 32767 else torch.int32
    keys = torch.where((flat < 0) | (flat >= vocab), vocab, flat).to(kdt)
    sorted_ids, order = torch.sort(keys, stable=True)
    key = (vocab, dev, kdt)
    probe = _arange_cache.get(key)
    if probe is None:
        probe = _arange_cache[key] = torch.arange(vocab + 1, device=dev, dtype=kdt)
    bounds = torch.searchsorted(sorted_ids, probe)
    dword = torch.empty(vocab, H, dtype=torch.float32, device=dev)
    dpos = None
    if n_pos:
        dpos = torch.empty(n_pos, H, dtype=torch.float32, device=dev) if n_pos == S else \
            torch.zeros(n_pos, H, dtype=torch.float32, device=dev)
    ws = torch.empty(_lib.load().muse_embed_bwd_sorted_workspace_bytes(B * S, H, vocab) // 4, dtype=torch.float32, device=dev)
    _call("muse_embed_bwd_sorted", _p(order), _p(bounds), _p(dx), _p(dword), _p(dpos), _p(ws), B, S, H, vocab, st)
    return dword, dpos


# ------------------------------------------------------------------------------------------ norms
def norm_fwd(x, w, eps, out_dtype, res=None, act=0, rms=0, save_stats=True, dropout=None):
    """act: 0 none, 1 GELU(x) first, 2 GLU (x is [rows, 2H] = [a | b], the normalised value is gelu(a) * b).
    dropout = (p, seed, site), act 2 with bf16 x and y only: FeedForward.dropout fused into the pass (the output is the
    dropped one); then returns (y, stats, bits) with bits int32 [rows, ceil(H / 32)] for norm_bwd (see dropout_fwd).
    out_dtype FP8: y is an F8, the A operand of the FP8 GEMMs (act 0 with H <= 1024, or act 2 with H <= 4096; no
    dropout)."""
    st = _prep(x)
    rows = x.shape[0]
    H = x.shape[1] // 2 if act == 2 else x.shape[1]
    if save_stats:
        stats = torch.empty(2, rows, dtype=torch.float32, device=x.device)
        mean, rstd = stats[0], stats[1]
    else:
        stats = mean = rstd = None
    if out_dtype == FP8:
        if dropout is not None:
            raise TypeError("norm_fwd: the e4m3 output takes no dropout")
        y, scale = _new_out(rows, H, FP8, x.device)
        _call("muse_norm_fwd_e4m3", _p(x), _dt(x), _p(w), _p(res), _p(y.q), _p(scale), _p(mean), _p(rstd), rows, H,
              float(eps), act, rms, st)
        return y, stats
    y = torch.empty(rows, H, dtype=out_dtype, device=x.device)
    if dropout is not None:
        assert act == 2 and x.dtype == torch.bfloat16 and out_dtype == torch.bfloat16 and res is None
    bits, seed, site, p = _drop_fwd_args(dropout, x.device, rows, cols=H)
    _call("muse_norm_fwd", _p(x), _dt(x), _p(w), _p(res), _p(y), _dt(y), _p(mean), _p(rstd), _p(bits), _p(seed), site, p,
          rows, H, float(eps), act, rms, st)
    return (y, stats) if bits is None else (y, stats, bits)


_bf16_copies = {}


def take_bf16_copy(t):
    """The bf16 copy norm_bwd(..., bf16_copy=True) produced alongside the fp32 tensor `t` (or None): consumed once."""
    hit = _bf16_copies.pop(t.data_ptr(), None)
    if hit is not None and hit[0] == (t._version, tuple(t.shape)):
        return hit[1]
    return None


def norm_bwd(dy, x, w, stats, dx_dtype, dw=None, dres=None, act=0, rms=0, y_fwd=None, want_dw=False, bf16_copy=False,
             dropout=None):
    """y_fwd: the saved forward output (act=2, bf16 only) -- lets the kernel skip one GELU pass over [a | b].
    dw: fp32 [H] buffer the weight gradient is ADDED to (atomics; caller zero-fills).  want_dw=True instead returns
    (dx, dw) with a freshly stored dw reduced in a fixed order (run-to-run bit-identical).
    dropout = (p, bits) from norm_fwd(..., dropout=...): dy (the gradient of the dropped output) is scaled by the bits as
    the kernel reads it; y_fwd is then ignored (the saved output is the dropped one, the GLU product is recomputed)."""
    st = _prep(x)
    rows = x.shape[0]
    H = x.shape[1] // 2 if act == 2 else x.shape[1]
    dx = torch.empty(x.shape, dtype=dx_dtype, device=x.device)
    p, bits = dropout if dropout is not None else (0.0, None)
    if dropout is not None:
        assert act == 2 and dy.dtype == x.dtype == dx_dtype == torch.bfloat16 and dres is None and not bf16_copy
        y_fwd = None
    if y_fwd is not None and not (act == 2 and y_fwd.dtype == torch.bfloat16 and y_fwd.is_contiguous()):
        y_fwd = None
    copy = None
    if bf16_copy and dx_dtype == torch.float32 and act != 2 and H <= 1024:
        copy = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
        if len(_bf16_copies) > 8:
            _bf16_copies.clear()
        _bf16_copies[dx.data_ptr()] = ((dx._version, tuple(dx.shape)), copy)
    ws = None
    if want_dw:
        dw = torch.empty(H, dtype=torch.float32, device=x.device)
        ws = torch.empty(max(1, _lib.load().muse_norm_bwd_workspace_floats(rows, H, act)), dtype=torch.float32, device=x.device)
        _state["launches"] += 1  # the ordered column sum
    _call("muse_norm_bwd", _p(dy), _dt(dy), _p(x), _dt(x), _p(w), _p(stats[0]), _p(stats[1]), _p(dres), _p(y_fwd), _p(bits),
          float(p), _p(dx), _dt(dx), _p(copy), _p(dw), _p(ws), rows, H, act, rms, st)
    return (dx, dw) if want_dw else dx


def norm2_fwd(a, res, w1, w2, eps, rms1=0, rms2=0, save_stats=True, h2_dtype=torch.bfloat16):
    """x2 = res + norm1(a) * w1 (fp32), h2 = norm2(x2) * w2 (bf16) in one pass; stats = [mean1, rstd1, mean2, rstd2].
    h2_dtype FP8: h2 is an F8, the A operand of the FP8 GEMM; x2 and stats are the same as the bf16 form's."""
    st = _prep(a)
    rows, H = a.shape
    x2 = torch.empty(rows, H, dtype=torch.float32, device=a.device)
    stats = torch.empty(4, rows, dtype=torch.float32, device=a.device) if save_stats else None
    sp = [None] * 4 if stats is None else [stats[i] for i in range(4)]
    if h2_dtype == FP8:
        h2, scale = _new_out(rows, H, FP8, a.device)
        _call("muse_norm2_fwd_e4m3", _p(a), _p(res), _p(w1), _p(w2), _p(x2), _p(h2.q), _p(scale), _p(sp[0]), _p(sp[1]),
              _p(sp[2]), _p(sp[3]), rows, H, float(eps), int(rms1), int(rms2), st)
        return x2, h2, stats
    h2 = torch.empty(rows, H, dtype=torch.bfloat16, device=a.device)
    _call("muse_norm2_fwd", _p(a), _p(res), _p(w1), _p(w2), _p(x2), _p(h2), _p(sp[0]), _p(sp[1]), _p(sp[2]), _p(sp[3]), rows, H,
          float(eps), int(rms1), int(rms2), st)
    return x2, h2, stats


def norm2_bwd(d_h2, x2, w2, dres, a, w1, stats, rms1=0, rms2=0):
    """joint backward of norm2_fwd: returns (dx2 fp32, d_a bf16, dw1, dw2), weight gradients stored in a fixed order."""
    st = _prep(a)
    rows, H = a.shape
    dev = a.device
    dx2 = torch.empty(rows, H, dtype=torch.float32, device=dev)
    d_a = torch.empty(rows, H, dtype=torch.bfloat16, device=dev)
    dw1 = torch.empty(H, dtype=torch.float32, device=dev)
    dw2 = torch.empty(H, dtype=torch.float32, device=dev)
    ws = torch.empty(2 * max(1, _lib.load().muse_norm_bwd_workspace_floats(rows, H, 0)), dtype=torch.float32, device=dev)
    _call("muse_norm2_bwd", _p(d_h2), _p(x2), _p(w2), _p(stats[2]), _p(stats[3]), _p(dres), _p(a), _p(w1), _p(stats[0]),
          _p(stats[1]), _p(dx2), _p(d_a), _p(dw2), _p(dw1), _p(ws), rows, H, int(rms1), int(rms2), st)
    return dx2, d_a, dw1, dw2


# ------------------------------------------------------------------------------------------ GLU / tanh-GELU
def glu_fwd(ab, dropout=None, out_dtype=torch.bfloat16):
    """dropout = (p, seed, site): FeedForward.dropout fused into the pass; then returns (out, bits) (see dropout_fwd).
    out_dtype FP8: out is an F8 (no dropout)."""
    st = _prep(ab)
    rows, two_i = ab.shape
    out, scale = _new_out(rows, two_i // 2, out_dtype, ab.device)
    bits, seed, site, p = _drop_fwd_args(dropout, ab.device, rows, cols=two_i // 2)
    _call("muse_glu_fwd", _p(ab), _p(_data(out)), _dt(_data(out)), _p(scale), _p(bits), _p(seed), site, p, rows, two_i // 2, st)
    return out if bits is None else (out, bits)


def glu_bwd(ab, dout, dropout=None):
    """dropout = (p, bits) from glu_fwd(..., dropout=...): dout is scaled by the bits as the kernel reads it."""
    st = _prep(ab)
    rows, two_i = ab.shape
    dab = torch.empty_like(ab)
    p, bits = dropout if dropout is not None else (0.0, None)
    _call("muse_glu_bwd", _p(ab), _p(dout), _p(bits), float(p), _p(dab), rows, two_i // 2, st)
    return dab


def gelu_tanh_fwd(pre, out_dtype=torch.bfloat16):
    """F.gelu(pre, approximate="tanh") of FusedGeLUFeedForward (use_fused_mlp): pre bf16 [rows, I] -> bf16 [rows, I].
    out_dtype FP8: out is an F8 (I <= 4096), the wo operand of the FP8 GEMM."""
    st = _prep(pre)
    rows, I = pre.shape
    out, scale = _new_out(rows, I, out_dtype, pre.device)
    _call("muse_gelu_tanh_fwd", _p(pre), _p(_data(out)), _dt(_data(out)), _p(scale), rows, I, st)
    return out


def gelu_tanh_bwd(pre, dout):
    """dpre bf16 [rows, I] = dout * gelu_tanh'(pre)"""
    st = _prep(pre)
    rows, I = pre.shape
    dpre = torch.empty_like(pre)
    _call("muse_gelu_tanh_bwd", _p(pre), _p(dout), _p(dpre), rows, I, st)
    return dpre


# ------------------------------------------------------------------------------------------ attention
def attn_fwd(q, k, v, B, nh, Sq, Skv, scale, head_dim=64, dropout=None):
    """q: [B*Sq, *] view with head h at columns h*head_dim; k, v: [B*Skv, *] views.  Returns ctx [B*Sq, nh*head_dim], lse.
    head_dim: 64 (default), 48 (configs/imagenet.yaml: hidden 768 / 16 heads), 96 or 128 (hidden 1024 / 8 heads).
    dropout = (p, seed, site): nn.Dropout(p) on the probabilities with the keep bits of (seed: int64 [1] device tensor,
    site) -- see dropout_fwd; then returns (ctx, lse, bits) with bits int32 [B, nh, Sq, ceil(Skv / 32)] for attn_bwd."""
    st = _prep(q)
    hd = int(head_dim)
    o = torch.empty(B * Sq, nh * hd, dtype=torch.bfloat16, device=q.device)
    lse = torch.empty(B, nh, Sq, dtype=torch.float32, device=q.device)
    bits, seed, site, p = _drop_fwd_args(dropout, q.device, B, nh, Sq, cols=Skv)
    _call("muse_attn_fwd", _p(q), _p(k), _p(v), _p(o), _p(lse), _p(bits), _p(seed), site, p, B, nh, Sq, Skv, hd,
          q.stride(0), k.stride(0), v.stride(0), o.stride(0), float(scale), st)
    return (o, lse) if bits is None else (o, lse, bits)


def attn_bwd(q, k, v, o, do, lse, dq, dk, dv, B, nh, Sq, Skv, scale, head_dim=64, dropout=None):
    """dropout = (p, bits): the rate and the keep bits attn_fwd(..., dropout=...) returned.  o is not read: the kernels
    recompute what they need from q, k, v and lse.  head_dim: 48, 64, 96 or 128, as for attn_fwd."""
    st = _prep(q)
    dvec = torch.empty(B, nh, Sq, dtype=torch.float32, device=q.device)
    p, bits = dropout if dropout is not None else (0.0, None)
    _call("muse_attn_bwd", _p(q), _p(k), _p(v), _p(do), _p(lse), _p(bits), float(p), _p(dvec), _p(dq), _p(dk), _p(dv), B,
          nh, Sq, Skv, int(head_dim), q.stride(0), k.stride(0), v.stride(0), do.stride(0), dq.stride(0), dk.stride(0),
          dv.stride(0), float(scale), st)


# ------------------------------------------------------------------------------------------ dropout
# nn.Dropout(p) in training mode.  The keep masks come from Philox4x32-10 keyed by a 64-bit seed that lives in device memory
# (an int64 [1] tensor drawn from torch's CUDA generator once per forward, so torch.manual_seed reproduces a run and a
# captured CUDA graph draws a fresh one per replay) and a site id unique within the forward; csrc/philox.cuh holds the
# mapping from (seed, site, coordinates) to bits and the rate actually applied, p_eff = round(p * 65536) / 65536.  The
# forward stores the bits (int32 words, rows padded to 32 bits, bit k % 32 of word k / 32 set = element k kept) and the
# backward reads them: no seed, no second draw.
_drop_state = {"log": None}


class dropout_record:
    """Test hook: ``with ops.dropout_record() as log:`` appends (site, bits) for every dropout op launched inside the block
    (attention and elementwise sites), so that tests can compare the masks with a restatement of the generator or hand
    them to another implementation.  Not a product switch."""

    def __enter__(self):
        self.prev = _drop_state["log"]
        _drop_state["log"] = []
        return _drop_state["log"]

    def __exit__(self, *exc):
        _drop_state["log"] = self.prev
        return False


def _drop_record(site, bits):
    if _drop_state["log"] is not None:
        _drop_state["log"].append((int(site), bits))


def _drop_fwd_args(dropout, device, *lead, cols):
    """(bits, seed, site, p) for a forward that takes dropout = (p, seed, site): fresh int32 keep-bit words
    [*lead, ceil(cols / 32)], recorded for dropout_record.  dropout None: (None, None, 0, 0.0), i.e. no dropout."""
    if dropout is None:
        return None, None, 0, 0.0
    p, seed, site = dropout
    bits = torch.empty(*lead, (cols + 31) // 32, dtype=torch.int32, device=device)
    _drop_record(site, bits)
    return bits, seed, int(site), float(p)


def dropout_fwd(x, p, seed, site):
    """x contiguous fp32 / bf16 [rows, cols] (cols % 8 == 0) is dropped IN PLACE: x * keep / (1 - p_eff).  Returns
    (x, bits) with bits int32 [rows, ceil(cols / 32)]."""
    st = _prep(x)
    rows, cols = x.shape
    assert x.is_contiguous()
    bits, seed, site, p = _drop_fwd_args((p, seed, site), x.device, rows, cols=cols)
    _call("muse_dropout_fwd", _p(x), _p(x), _dt(x), _p(bits), _p(seed), site, p, rows, cols, st)
    return x, bits


def dropout_bwd(dy, bits, p, out=None):
    """dx = dy * keep / (1 - p_eff) with the bits dropout_fwd stored; out (may be dy itself) receives dx."""
    st = _prep(dy)
    rows, cols = dy.shape
    assert dy.is_contiguous()
    dx = torch.empty_like(dy) if out is None else out
    _call("muse_dropout_bwd", _p(dy), _p(dx), _dt(dy), _p(bits), float(p), rows, cols, st)
    return dx


# ------------------------------------------------------------------------------------------ loss
def ce_fwd(logits_padded, labels, V, label_smoothing):
    st = _prep(logits_padded)
    rows, ld = logits_padded.shape
    ws = torch.empty(2, rows, dtype=torch.float32, device=logits_padded.device)  # lse, row_loss
    out = torch.empty(2, dtype=torch.float32, device=logits_padded.device)
    _call("muse_ce_fwd", _p(logits_padded), _p(labels), _p(ws[0]), _p(ws[1]), _p(out), rows, V, ld,
          float(label_smoothing), st)
    return out, ws


def ce_bwd(logits_padded, labels, ws, dloss, loss_out, V, label_smoothing, row_scale=None):
    st = _prep(logits_padded)
    rows, ld = logits_padded.shape
    dl = torch.empty_like(logits_padded)
    _call("muse_ce_bwd", _p(logits_padded), _p(labels), _p(ws[0]), _p(dloss), _p(loss_out), _p(row_scale), _p(dl), rows, V,
          ld, float(label_smoothing), st)
    return dl


# ------------------------------------------------------------------------------------------ U-ViT v2 forward ops
def add_norm_mod(a, w, eps, rms, out_dtype=torch.bfloat16, residual=None, mod=None, rows_per_sample=1, want_residual=True):
    """(r', y): r' = a + residual (fp32), y = norm(r') * w [* (1 + scale_b) + shift_b].  mod: fp32 [B, 2H] view (scale |
    shift per sample, row pitch mod.stride(0)) of the batched adaLN mapper output.  out_dtype FP8: y is an F8."""
    st = _prep(a)
    rows, H = a.shape
    y, scale = _new_out(rows, H, out_dtype, a.device)
    r_out = torch.empty(rows, H, dtype=torch.float32, device=a.device) if want_residual else None
    _call("muse_add_norm_mod_fwd", _p(a), _dt(a), _p(residual), _p(w), _p(mod), 0 if mod is None else mod.stride(0),
          int(rows_per_sample), _p(r_out), _p(_data(y)), _dt(_data(y)), _p(scale), rows, H, float(eps), int(rms), st)
    return r_out, y


def dwconv3x3_norm(x, wk, norm_w, B, hh, ww, eps, rms, save_conv=False, out_dtype=torch.bfloat16):
    """x fp32 [B*hh*ww, C] token-major, wk fp32 [9, C] -> bf16 [B*hh*ww, C] = Norm2D(depthwise3x3(x)).
    save_conv: also return the bf16 conv output (needed by dwconv3x3_norm_bwd).  out_dtype FP8: y is an F8."""
    st = _prep(x)
    C = x.shape[1]
    y, scale = _new_out(x.shape[0], C, out_dtype, x.device)
    conv = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device) if save_conv else None
    _call("muse_dwconv3x3_norm_fwd", _p(x), _p(wk), _p(norm_w), _p(_data(y)), _dt(_data(y)), _p(scale), _p(conv), B, hh,
          ww, C, float(eps), int(rms), st)
    return (y, conv) if save_conv else y


def grn(x, gamma, beta, B, HW, save_stats=False, dropout=None):
    """bf16 [B*HW, C] -> bf16: GELU + GlobalResponseNorm.  save_stats: also return (sumsq, nx) for grn_bwd.
    dropout = (p, seed, site): the ResBlock's dropout that follows GRN fused into the pass (the output is the dropped one);
    then returns (out, stats, bits) with bits int32 [B*HW, ceil(C / 32)] for grn_bwd (see dropout_fwd)."""
    st = _prep(x)
    C = x.shape[1]
    out = torch.empty_like(x)
    ws = torch.empty(2, B, C, dtype=torch.float32, device=x.device)
    bits, seed, site, p = _drop_fwd_args(dropout, x.device, B * HW, cols=C)
    _call("muse_grn_fwd", _p(x), _p(gamma), _p(beta), _p(out), _p(ws[0]), _p(ws[1]), _p(bits), _p(seed), site, p, B, HW, C,
          st)
    if bits is not None:
        return out, ws, bits
    return (out, ws) if save_stats else out


def add_norm_mod_bwd(dy, dr_out, x_saved, w, eps, rms, da_dtype, mod=None, rows_per_sample=1, dw=None, dmod=None,
                     want_dr=True):
    """Backward of add_norm_mod: returns (da, dr); dw [H] and dmod (view with the layout of mod) are accumulated."""
    st = _prep(x_saved)
    rows, H = x_saved.shape
    da = torch.empty(rows, H, dtype=da_dtype, device=x_saved.device)
    dr = torch.empty(rows, H, dtype=torch.float32, device=x_saved.device) if want_dr else None
    _call("muse_add_norm_mod_bwd", _p(dy), _dt(dy), _p(dr_out), _p(x_saved), _p(w), _p(mod),
          0 if mod is None else mod.stride(0), int(rows_per_sample), _p(da), _dt(da), _p(dr), _p(dw), _p(dmod), rows, H,
          float(eps), int(rms), st)
    return da, dr


def dwconv3x3_norm_bwd(dy, conv, x, wk, norm_w, dres, dwk, dnw, B, hh, ww, eps, rms):
    st = _prep(x)
    C = x.shape[1]
    ws = torch.empty(x.shape, dtype=torch.float32, device=x.device)
    dx = torch.empty(x.shape, dtype=torch.float32, device=x.device)
    _call("muse_dwconv3x3_norm_bwd", _p(dy), _p(conv), _p(x), _p(wk), _p(norm_w), _p(dres), _p(ws), _p(dx), _p(dwk), _p(dnw),
          B, hh, ww, C, float(eps), int(rms), st)
    return dx


def grn_bwd(x, dout, stats, gamma, dgamma, dbeta, B, HW, dropout=None):
    """dropout = (p, bits) from grn(..., dropout=...): dout is scaled by the bits as the kernels read it."""
    st = _prep(x)
    C = x.shape[1]
    dx = torch.empty_like(x)
    ws = torch.empty(B, C, dtype=torch.float32, device=x.device)
    p, bits = dropout if dropout is not None else (0.0, None)
    _call("muse_grn_bwd", _p(x), _p(dout), _p(stats[1]), _p(stats[0]), _p(gamma), _p(ws), _p(dx), _p(dgamma), _p(dbeta),
          _p(bits), float(p), B, HW, C, st)
    return dx


def adaln_bwd(dy, x, mod, dmod, B, rows_per_sample):
    st = _prep(x)
    dx = torch.empty_like(x)
    _call("muse_adaln_bwd", _p(dy), _p(x), _p(mod), mod.stride(0), _p(dx), _p(dmod), B, int(rows_per_sample), x.shape[1], st)
    return dx


def silu_bwd(dy, x, out=None, out_dtype=None):
    """dx = dy * silu'(x); out given: accumulate into it."""
    st = _prep(x)
    acc = out is not None
    if out is None:
        out = torch.empty(x.shape, dtype=out_dtype or x.dtype, device=x.device)
    _call("muse_silu_bwd", _p(dy), _p(x), _dt(x), _p(out), _dt(out), x.numel(), 1 if acc else 0, st)
    return out


def adaln_apply(x, mod, B, rows_per_sample):
    """out-of-place variant (training keeps the pre-modulation tensor for the backward pass)."""
    return adaln_apply_(x.clone(), mod, B, rows_per_sample)


def adaln_apply_(x, mod, B, rows_per_sample):
    st = _prep(x)
    _call("muse_adaln_apply", _p(x), _p(mod), mod.stride(0), B, int(rows_per_sample), x.shape[1], st)
    return x


def silu_bf16(x):
    st = _prep(x)
    y = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    _call("muse_silu_bf16", _p(x), _dt(x), _p(y), x.numel(), st)
    return y


# ------------------------------------------------------------------------------------------ VQ
def vq_argmin(z_flat, codebook, return_dmin=False):
    st = _prep(z_flat)
    n, D = z_flat.shape
    ncodes = codebook.shape[0]
    ids = torch.empty(n, dtype=torch.int64, device=z_flat.device)
    ws = torch.empty(ncodes, dtype=torch.float32, device=z_flat.device)
    dmin = torch.empty(n, dtype=torch.float32, device=z_flat.device) if return_dmin else None
    _call("muse_vq_argmin", _p(z_flat), _p(codebook), _p(ws), _p(ids), _p(dmin), n, ncodes, D, st)
    return (ids, dmin) if return_dmin else ids


def vq_soft_code(z_flat, codebook, temp=1.0, expo_noise=None):
    """softmax(-d/temp) over the codebook + ids (argmin, or argmax soft/q when Exp(1) noise q is given)."""
    st = _prep(z_flat)
    n, D = z_flat.shape
    ncodes = codebook.shape[0]
    soft = torch.empty(n, ncodes, dtype=torch.float32, device=z_flat.device)
    ids = torch.empty(n, dtype=torch.int64, device=z_flat.device)
    ws = torch.empty(ncodes, dtype=torch.float32, device=z_flat.device)
    _call("muse_vq_soft_code", _p(z_flat), _p(codebook), _p(ws), _p(soft), _p(ids), _p(expo_noise), float(temp), n,
          ncodes, D, st)
    return soft, ids


def vq_lookup_nchw(ids, codebook):
    st = _prep(codebook)
    B, P = ids.shape
    D = codebook.shape[1]
    out = torch.empty(B, D, P, dtype=torch.float32, device=codebook.device)
    _call("muse_vq_lookup_nchw", _p(ids), _p(codebook), _p(out), B, P, D, codebook.shape[0], st)
    return out


# ------------------------------------------------------------------------------------------ generate2 step
def sample_step(logits, input_ids, q_exp, u, K, mask_id, mask_len, temperature, logits_unc=None, guidance=0.0,
                skip_first_token=False, return_conf=False):
    """logits: bf16 [B, S, ld] view (S = L (+1 with a class token, skipped when skip_first_token)); see csrc/sample.cu."""
    st = _prep(logits)
    B, L = input_ids.shape
    off = 1 if skip_first_token else 0
    lg = logits[:, off:]
    lu = logits_unc[:, off:] if logits_unc is not None else None
    sampled = torch.empty(B, L, dtype=torch.int64, device=logits.device)
    nxt = torch.empty(B, L, dtype=torch.int64, device=logits.device)
    conf = torch.empty(B, L, dtype=torch.float32, device=logits.device)
    _call("muse_sample_step", _p(lg), _p(lu), lg.stride(1), lg.stride(0), float(guidance), _p(input_ids), _p(q_exp),
          _p(u), _p(sampled), _p(nxt), _p(conf), B, L, K, int(mask_id), int(mask_len), float(temperature), st)
    return (sampled, nxt, conf) if return_conf else (sampled, nxt)


# ------------------------------------------------------------------------------------------ VQGAN blocks (fp32 NHWC)
# Tensor-core convolution precision: "bf16x3" (default) carries every fp32 operand as bf16 hi + lo planes and accumulates
# hi*hi + lo*hi + hi*lo in fp32 -- fp32-faithful, what the bit-exact token-id contract needs.  "bf16" multiplies the hi
# planes only: one product instead of three and no lo planes written, at bf16-operand accuracy (the reference itself runs
# its tokenizer convolutions in TF32 on the GPU: cudnn.allow_tf32 defaults to True and training/train_maskgit_imagenet.py:
# 146-149 also enables it for matmuls, quirk Q19).  Token ids from the fast mode agree with the exact ones except near
# ties; bench.py reports the agreement rate.
_conv_state = {"single": False, "route": None}


class conv_precision:
    """``with ops.conv_precision("bf16"): ...`` -- scoped selection of the tokenizer convolution mode."""

    def __init__(self, mode):
        if mode not in ("bf16x3", "bf16"):
            raise ValueError("conv precision must be 'bf16x3' (fp32-faithful) or 'bf16' (single pass)")
        self.single = mode == "bf16"

    def __enter__(self):
        self.prev = _conv_state["single"]
        _conv_state["single"] = self.single

    def __exit__(self, *exc):
        _conv_state["single"] = self.prev
        return False


class conv_route:
    """Test hook: ``with ops.conv_route("simt")`` forces the fp32 FMA convolution kernels (the route geometries without a TMA
    tiling take anyway) so that tests can compare the tensor-core route against them.  Not a product switch."""

    def __init__(self, route):
        assert route in (None, "simt")
        self.route = route

    def __enter__(self):
        self.prev = _conv_state["route"]
        _conv_state["route"] = self.route

    def __exit__(self, *exc):
        _conv_state["route"] = self.prev
        return False


_wk_cache = {}
_WK_CACHE_ENTRIES = 4096


def _cached_pack(tag, w, pack):
    """pack(w as fp32), cached per live weight tensor w under `tag`.  The key holds w's weakref identity, storage pointer,
    version counter, shape and device, so a recycled id() or an in-place update never hits; the cache is emptied when it
    outgrows _WK_CACHE_ENTRIES."""
    key = (w.data_ptr(), w._version, tuple(w.shape), w.device)
    hit = _wk_cache.get((tag, id(w)))
    if hit is not None and hit[0]() is w and hit[1] == key:
        return hit[2]
    out = pack(w.detach().float())
    if len(_wk_cache) > _WK_CACHE_ENTRIES:
        _wk_cache.clear()
    _wk_cache[(tag, id(w))] = (weakref.ref(w), key, out)
    return out


def _planes(wk):
    """fp32 -> bf16 planes (hi, lo) with wk = hi + lo: hi = bf16(wk), lo = bf16(wk - hi)."""
    hi = wk.to(torch.bfloat16)
    return hi, (wk - hi.float()).to(torch.bfloat16)


def _pack_simt(wf):
    """[Cout, Cin, kh, kw] -> [kh*kw*Cin, Cout] (tap-major, then input channel), the weights of muse_conv2d_nhwc."""
    return wf.permute(2, 3, 1, 0).reshape(-1, wf.shape[0]).contiguous()


def _pack_tc(wf):
    """[Cout, Cin, kh, kw] -> bf16 planes of [Cout, kh*kw*Cin] (tap-major, then input channel)."""
    return _planes(wf.permute(0, 2, 3, 1).reshape(wf.shape[0], -1).contiguous())


def _pack_stem(wf):
    """Stem weight [Cout, Cin, k, k] with k*k*Cin <= 64 -> bf16 planes of [Cout, 64], columns tap-major, zero padded: the
    1x1 convolution over the rows of muse_im2col_split_nhwc."""
    wk = torch.zeros(wf.shape[0], 64, dtype=torch.float32, device=wf.device)
    flat = wf.permute(0, 2, 3, 1).reshape(wf.shape[0], -1)
    wk[:, : flat.shape[1]] = flat
    return _planes(wk)


def _tc_route(H, W, Cin, Cout, k, upsample2x=False):
    """Whether muse_conv2d_nhwc_tc runs this convolution, H, W the output dims; upsample2x: in the four-parity form of
    MUSE_CONV_TC_UPSAMPLE2X.  Never under the test hook ops.conv_route("simt")."""
    if _conv_state["route"] == "simt":
        return False
    if upsample2x:
        return _lib.load().muse_conv2d_tc_tiles_per_image(H, W, Cin, Cout, k, 1) > 0
    return bool(_lib.load().muse_conv2d_tc_supported(H, W, Cin, Cout, k))


def conv_uses_tensor_cores(H, W, Cin, Cout, k):
    """Whether conv2d() at output size H x W runs on the tensor cores (the wgmma implicit GEMM of csrc/conv_tc.cu) rather
    than the fp32 SIMT kernel: unless the geometry is unsupported or ops.conv_route("simt") is active.  Stems with
    k*k*Cin <= 64 go through an im2col to 64 columns and run as a 1x1 convolution."""
    if Cin % 64 != 0 and k * k * Cin <= 64:
        return _tc_route(H, W, 64, Cout, 1)
    return _tc_route(H, W, Cin, Cout, k)


def _new_planes(shape, device, exact=False):
    """Uninitialised bf16 operand planes (hi, lo); no lo plane in the single-pass precision unless exact."""
    hi = torch.empty(shape, dtype=torch.bfloat16, device=device)
    return hi, (torch.empty_like(hi) if exact or not _conv_state["single"] else None)


def _split(x, st, upsample2x=False, exact=False):
    """fp32 NHWC x -> its bf16 planes (hi, lo), those of its nearest x2 upsample with upsample2x.  An x of another rank is
    split as rows of its last dimension."""
    *lead, C = x.shape
    B, H, W = lead if len(lead) == 3 else (1, 1, x.numel() // C)
    if upsample2x:
        H, W = 2 * H, 2 * W
    hi, lo = _new_planes((B, H, W, C) if x.dim() == 4 else x.shape, x.device, exact)
    _call("muse_split_bf16_nhwc", _p(x), _p(hi), _p(lo), B, H, W, C, int(upsample2x), st)
    return hi, lo


def _split_s2d(x, st):
    """fp32 NHWC x [B, 2H, 2W, C] -> the bf16 planes of its space-to-depth [B, H, W, 4C]."""
    B, Hi, Wi, C = x.shape
    hi, lo = _new_planes((B, Hi // 2, Wi // 2, 4 * C), x.device)
    _call("muse_split_s2d_bf16_nhwc", _p(x), _p(hi), _p(lo), B, Hi // 2, Wi // 2, C, st)
    return hi, lo


def _im2col(x, H, W, k, st):
    """fp32 NHWC x -> bf16 planes [B, H, W, 64] of the k*k*Cin <= 64 taps per output pixel (k = 2: the PixelUnshuffle(2)
    block of x [B, 2H, 2W, Cin])."""
    B, Cin = x.shape[0], x.shape[3]
    hi, lo = _new_planes((B, H, W, 64), x.device)
    _call("muse_im2col_split_nhwc", _p(x), _p(hi), _p(lo), B, H, W, Cin, k, st)
    return hi, lo


def _conv_tc(x, w, bias, y, B, H, W, Cin, Cout, k, mode, st, res=None, stats=None, exact=False):
    """One tensor-core convolution of the activation planes x by the weight planes w, both (hi, lo) pairs.  y is the fp32
    output, or the (hi, lo) planes that receive GELU(conv + bias) (muse_conv2d_nhwc_tc_gelu_split).  The single-pass
    precision adds MUSE_CONV_TC_SINGLE_PASS to the mode unless exact."""
    if _conv_state["single"] and not exact:
        mode |= CONV_TC_SINGLE_PASS
    if isinstance(y, tuple):
        _call("muse_conv2d_nhwc_tc_gelu_split", _p(x[0]), _p(x[1]), _p(w[0]), _p(w[1]), _p(bias), _p(y[0]), _p(y[1]), B, H,
              W, Cin, Cout, k, mode, st)
    else:
        _call("muse_conv2d_nhwc_tc", _p(x[0]), _p(x[1]), _p(w[0]), _p(w[1]), _p(bias), _p(res), _p(y), _p(stats), B, H, W,
              Cin, Cout, k, mode, st)


def _gn_scratch(x):
    B, H, W, C = x.shape
    n_ws = _lib.load().muse_groupnorm_workspace_floats(B, H * W, C)
    if n_ws < 0:
        raise _lib.MuseB200Error(f"groupnorm: unsupported channel count {C}")
    return (torch.empty(n_ws, dtype=torch.float32, device=x.device),
            torch.empty(B * C * 3, dtype=torch.float32, device=x.device))


def _groupnorm(x, gn, spatial, st, planes=False):
    """GroupNorm (+ SiLU) of fp32 NHWC x, gn = (gamma, beta, groups, eps[, silu = 1]); MoVQ SpatialNorm with spatial (see
    groupnorm_silu).  Returns fp32 y, or with planes the bf16 operand planes of the next tensor-core convolution, which
    reuse the {sum, M2} tiles the convolution that produced x left on it."""
    B, H, W, C = x.shape
    gamma, beta = gn[0].detach().float(), gn[1].detach().float()
    groups, eps, silu = int(gn[2]), float(gn[3]), int(gn[4]) if len(gn) > 4 else 1
    pre = getattr(x, "_gn_stats", None) if planes else None
    if pre is not None and pre[2] == x._version:
        ws, tiles, _ = pre
        ss = torch.empty(B * C * 3, dtype=torch.float32, device=x.device)
    else:
        (ws, ss), tiles = _gn_scratch(x), 0
    if planes:
        y, (hi, lo) = None, _new_planes(x.shape, x.device)
    else:
        y, hi, lo = torch.empty_like(x), None, None
    if spatial is None:
        _call("muse_groupnorm_silu_nhwc", _p(x), _p(gamma), _p(beta), _p(y), _p(hi), _p(lo), _p(ws), _p(ss), B, H * W, C,
              groups, eps, tiles, silu, st)
    else:
        zq, mod, hz, wz, dq = _spatial_args(spatial)
        _call("muse_spatial_groupnorm_silu_nhwc", _p(x), _p(gamma), _p(beta), _p(zq), *mod, _p(y), _p(hi), _p(lo), _p(ws),
              _p(ss), B, H, W, C, groups, eps, hz, wz, dq, tiles, silu, st)
    return (hi, lo) if planes else y


def _spatial_args(spatial):
    """(zq, conv_y, conv_b) -> zq, the (wy, by, wb, bb) pointers, hz, wz, dq of muse_spatial_groupnorm_silu_nhwc; the 1x1
    weights are packed to [C, dq] once per parameter version"""
    zq, cy, cb = spatial
    zq = zq.float().contiguous()
    pack = lambda w: w.reshape(w.shape[0], -1).clone()  # noqa: E731  (a fresh, 16-byte aligned [C, dq] copy)
    wy, wb = _cached_pack("spatial_w", cy.weight, pack), _cached_pack("spatial_w", cb.weight, pack)
    by, bb = _cached_pack("spatial_b", cy.bias, torch.clone), _cached_pack("spatial_b", cb.bias, torch.clone)
    return zq, (_p(wy), _p(by), _p(wb), _p(bb)), zq.shape[1], zq.shape[2], zq.shape[3]


def _conv_stats_buffer(y, H, W, Cin, Cout, k, up=0):
    """The tensor-core convolution's epilogue leaves per-tile {sum, M2} of its output (M2: squared deviations from the tile
    mean): they ride along on the output tensor (``y._gn_stats``, with y's version counter) so that a following
    conv2d(gn=...) skips the GroupNorm statistics pass over y -- unless y was modified in place since."""
    if Cout <= 16 or Cout % 32 != 0:
        return None
    tiles = _lib.load().muse_conv2d_tc_tiles_per_image(H, W, Cin, Cout, k, up)
    stats = torch.empty(y.shape[0], tiles, Cout, 2, dtype=torch.float32, device=y.device)
    y._gn_stats = (stats, tiles, y._version)
    return stats


def _pack_upsample(wf):
    """3x3 weight of an UpsamplingBlock conv -> bf16 planes of the four stacked 2x2 parity matrices [4*Cout, 4*Cin].

    Output pixel (2y+py, 2x+px) of conv3x3(nearest_x2(v)) reads only v[y+a+py-1, x+b+px-1] for a, b in {0, 1}; the 3x3
    taps that land on the same low-resolution pixel are summed (fp32): rows R(0,0)={0}, R(0,1)={1,2}, R(1,0)={0,1},
    R(1,1)={2} (same for columns)."""
    sets = {(0, 0): [0], (0, 1): [1, 2], (1, 0): [0, 1], (1, 1): [2]}
    mats = []
    for py in (0, 1):
        for px in (0, 1):
            taps = []
            for a in (0, 1):
                for b in (0, 1):
                    acc = 0
                    for kh in sets[(py, a)]:
                        for kw in sets[(px, b)]:
                            acc = acc + wf[:, :, kh, kw]
                    taps.append(acc)  # [Cout, Cin]
            mats.append(torch.stack(taps, dim=1).reshape(wf.shape[0], -1))  # [Cout, 4*Cin], column = (a*2+b)*Cin + ci
    return _planes(torch.cat(mats, dim=0).contiguous())  # [4*Cout, 4*Cin], row = parity*Cout + co


def conv2d(x, w, bias=None, residual=None, upsample2x=False, gn=None, spatial=None):
    """Conv2dSame on fp32 NHWC x [B,Hi,Wi,Cin] with the nn.Conv2d weight w [Cout,Cin,k,k] -> fp32 NHWC [B,H,W,Cout].

    gn = (gamma, beta, groups, eps) applies GroupNorm+SiLU to x first (the ResnetBlock pattern); upsample2x applies the
    nearest x2 upsample first.  Heavy layers run on the tensor cores (csrc/conv_tc.cu) with operands carried as bf16
    hi/lo planes; the GroupNorm kernel emits the planes directly.  spatial = (zq, conv_y, conv_b) turns the GroupNorm
    into the MoVQ SpatialNorm (see groupnorm_silu)."""
    st = _prep(x)
    B, Hi, Wi, Cin = x.shape
    H, W = (Hi * 2, Wi * 2) if upsample2x else (Hi, Wi)
    Cout, k = w.shape[0], w.shape[2]
    y = torch.empty(B, H, W, Cout, dtype=torch.float32, device=x.device)
    b = None if bias is None else bias.detach().float()
    if upsample2x and gn is None and _tc_route(H, W, Cin, Cout, k, upsample2x=True):
        # nearest x2 + 3x3 conv as four 2x2 parity convolutions on the low-resolution planes (2.25x fewer FLOPs)
        _conv_tc(_split(x, st), _cached_pack("upsample", w, _pack_upsample), b, y, B, H, W, Cin, Cout, k,
                 CONV_TC_UPSAMPLE2X, st, res=residual, stats=_conv_stats_buffer(y, H, W, Cin, Cout, k, 1))
        return y
    if not conv_uses_tensor_cores(H, W, Cin, Cout, k):
        if gn is not None:
            x = _groupnorm(x, gn, spatial, st)
        _call("muse_conv2d_nhwc", _p(x), _p(_cached_pack("simt", w, _pack_simt)), _p(b), _p(residual), _p(y), B, H, W, Cin,
              Cout, k, CONV_UPSAMPLE2X if upsample2x else CONV_SAME, st)
        return y
    if Cin % 64 != 0:  # stem with k*k*Cin <= 64
        assert gn is None and not upsample2x
        _conv_tc(_im2col(x, H, W, k, st), _cached_pack("stem", w, _pack_stem), b, y, B, H, W, 64, Cout, 1, CONV_TC_SAME, st,
                 res=residual, stats=_conv_stats_buffer(y, H, W, 64, Cout, 1))
        return y
    if gn is None:
        planes = _split(x, st, upsample2x)
    else:
        assert not upsample2x
        planes = _groupnorm(x, gn, spatial, st, planes=True)
    _conv_tc(planes, _cached_pack("tc", w, _pack_tc), b, y, B, H, W, Cin, Cout, k, CONV_TC_SAME, st, res=residual,
             stats=_conv_stats_buffer(y, H, W, Cin, Cout, k))
    return y


def groupnorm_silu(x, gamma, beta, groups, eps, silu=1, spatial=None):
    """GroupNorm (+ SiLU unless silu=0), fp32 NHWC in and out.

    spatial = (zq, conv_y, conv_b): the MoVQ SpatialNorm (muse/modeling_movq.py:21-49) before the SiLU,
    GN(x) * conv_y(up(zq)) + conv_b(up(zq)), with zq the fp32 NHWC latent [B, hz, wz, dq] (H / hz and W / wz integers),
    conv_y / conv_b its 1x1 nn.Conv2d(dq, C) modules and `up` the nearest resize; computed per pixel inside the apply pass."""
    return _groupnorm(x, (gamma, beta, groups, eps, silu), spatial, _prep(x))


def _pack_s2d(wf):
    """3x3 stride-2 weight (pad (0,1,0,1)) -> bf16 planes [Cout, 4 taps * 4 * Cin] for the space-to-depth form:
    tap (a, b) in {0,1}^2 and plane (p, q) hold w[:, :, 2a + p, 2b + q] (zero where 2a + p or 2b + q exceeds 2)."""
    Cout, Cin = wf.shape[0], wf.shape[1]
    wk = torch.zeros(Cout, 2, 2, 2, 2, Cin, dtype=torch.float32, device=wf.device)  # [co, a, b, p, q, ci]
    for a in (0, 1):
        for b in (0, 1):
            for p_ in (0, 1):
                for q in (0, 1):
                    kh, kw = 2 * a + p_, 2 * b + q
                    if kh <= 2 and kw <= 2:
                        wk[:, a, b, p_, q] = wf[:, :, kh, kw]
    return _planes(wk.reshape(Cout, -1).contiguous())


def conv2d_down(x, w, bias=None):
    """taming Downsample (modeling_taming_vqgan.py:47-62): F.pad(x, (0,1,0,1)) then 3x3 conv with stride 2.
    x fp32 NHWC [B, 2H, 2W, Cin] -> fp32 [B, H, W, Cout].  Tensor-core route: space-to-depth + hi/lo split, then a
    stride-1 2x2 convolution over 4*Cin channels; other geometries use the fp32 SIMT kernel's stride-2 mode."""
    st = _prep(x)
    B, Hi, Wi, Cin = x.shape
    H, W = Hi // 2, Wi // 2
    Cout = w.shape[0]
    y = torch.empty(B, H, W, Cout, dtype=torch.float32, device=x.device)
    b = None if bias is None else bias.detach().float()
    if _tc_route(H, W, 4 * Cin, Cout, 2):
        _conv_tc(_split_s2d(x, st), _cached_pack("s2d", w, _pack_s2d), b, y, B, H, W, 4 * Cin, Cout, 2, CONV_TC_FWD2X2, st,
                 stats=_conv_stats_buffer(y, H, W, 4 * Cin, Cout, 2))
        return y
    _call("muse_conv2d_nhwc", _p(x), _p(_cached_pack("simt", w, _pack_simt)), _p(b), None, _p(y), B, H, W, Cin, Cout, 3,
          CONV_STRIDE2, st)
    return y


def attention_single_head(q, k, v, B, hh, ww):
    """softmax(q k^T / sqrt(C)) v per image with ONE head of width C (AttnBlock of the taming VQGAN, :148-174), fp32-faithful:
    q, k, v fp32 [B*hh*ww, C] -> fp32 [B*hh*ww, C].  Both products run as 1x1 tensor-core convolutions whose weights are
    the image's own keys / values (per-image weight mode of muse_conv2d_nhwc_tc); small geometries loop over the images
    with the SIMT kernel."""
    st = _prep(q)
    HW, C = hh * ww, q.shape[1]
    scale = float(C) ** -0.5
    out = torch.empty(B * HW, C, dtype=torch.float32, device=q.device)
    scores = torch.empty(B * HW, HW, dtype=torch.float32, device=q.device)
    vt = torch.empty(B, C, HW, dtype=torch.float32, device=q.device)
    _call("muse_transpose_batched", _p(v), _p(vt), B, HW, C, st)
    if _tc_route(hh, ww, C, HW, 1) and _tc_route(hh, ww, HW, C, 1):
        # exact: both products stay three-pass in the bf16 precision too, as the models' set_conv_precision promises
        queries, keys = _split(q, st, exact=True), _split(k, st, exact=True)  # keys: per-image weights [B][HW keys][C]
        _conv_tc(queries, keys, None, scores, B, hh, ww, C, HW, 1, CONV_TC_PER_IMAGE_WEIGHTS, st, exact=True)
        probs = _new_planes(scores.shape, q.device, exact=True)
        _call("muse_softmax_split_rows", _p(scores), _p(probs[0]), _p(probs[1]), None, B * HW, HW, scale, st)
        values = _split(vt, st, exact=True)  # per-image weights [B][C][HW keys]
        _conv_tc(probs, values, None, out, B, hh, ww, HW, C, 1, CONV_TC_PER_IMAGE_WEIGHTS, st, exact=True)
        return out
    kt = torch.empty(B, C, HW, dtype=torch.float32, device=q.device)
    _call("muse_transpose_batched", _p(k), _p(kt), B, HW, C, st)
    probs = torch.empty_like(scores)
    for b in range(B):  # SIMT weights are [K, Cout]: k_b^T for the scores, v_b for the output
        qb, sb = q[b * HW:(b + 1) * HW], scores[b * HW:(b + 1) * HW]
        _call("muse_conv2d_nhwc", _p(qb), _p(kt[b]), None, None, _p(sb), 1, hh, ww, C, HW, 1, CONV_SAME, st)
    _call("muse_softmax_split_rows", _p(scores), None, None, _p(probs), B * HW, HW, scale, st)
    for b in range(B):
        pb, ob = probs[b * HW:(b + 1) * HW], out[b * HW:(b + 1) * HW]
        _call("muse_conv2d_nhwc", _p(pb), _p(v[b * HW:(b + 1) * HW]), None, None, _p(ob), 1, hh, ww, HW, C, 1, CONV_SAME, st)
    return out


def avg_pool2x2(x):
    st = _prep(x)
    B, H, W, C = x.shape
    y = torch.empty(B, H // 2, W // 2, C, dtype=torch.float32, device=x.device)
    _call("muse_avgpool2_nhwc", _p(x), _p(y), B, H // 2, W // 2, C, st)
    return y


def to_nhwc(x_nchw):
    st = _prep(x_nchw)
    B, C, H, W = x_nchw.shape
    y = torch.empty(B, H, W, C, dtype=torch.float32, device=x_nchw.device)
    _call("muse_transpose_batched", _p(x_nchw), _p(y), B, C, H * W, st)
    return y


def to_nchw(x_nhwc):
    st = _prep(x_nhwc)
    B, H, W, C = x_nhwc.shape
    y = torch.empty(B, C, H, W, dtype=torch.float32, device=x_nhwc.device)
    _call("muse_transpose_batched", _p(x_nhwc), _p(y), B, H * W, C, st)
    return y


def image_to_uint8(x):
    """fp32 image tensor (any layout) -> uint8 with the reference's to_pil_image recipe, on the device."""
    st = _prep(x)
    x = x.contiguous()
    y = torch.empty(x.shape, dtype=torch.uint8, device=x.device)
    _call("muse_image_to_uint8", _p(x), _p(y), x.numel(), st)
    return y


# ------------------------------------------------------------------------------------------ Paella tokenizer (fp32 NHWC)
# muse/modeling_paella_vq.py.  Each op takes the nn weights (already gamma / BatchNorm-folded where the model folds them)
# and picks the tensor-core route when the geometry has a TMA tiling, else the fp32 SIMT kernels of conv.cu.
_KERNELS_PER_CALL["muse_paella_resblock_spatial"] = 2


def paella_resblock(x, wk, bias, w1, b1, w2, b2, eps=1e-6):
    """Paella ResBlock (modeling_paella_vq.py:112-145) on fp32 NHWC x [B,H,W,C] with its gammas folded into the weights:
    wk fp32 [9, C] and bias [C] of the depthwise 3x3 (tap-major), w1 [4C, C, 1, 1] / b1 and w2 [C, 4C, 1, 1] / b2 of the
    two Linears.  Four launches: LN1 statistics, the spatial pass (x1 = x + dw(LN1 x), LN2(x1)), Linear + GELU, Linear
    + residual x1."""
    st = _prep(x)
    B, H, W, C = x.shape
    Ch = w1.shape[0]
    x1 = torch.empty_like(x)
    stats = torch.empty(2 * B * H * W, dtype=torch.float32, device=x.device)
    y = torch.empty_like(x)
    if _tc_route(H, W, C, Ch, 1) and _tc_route(H, W, Ch, C, 1):
        n = _new_planes(x.shape, x.device)
        _call("muse_paella_resblock_spatial", _p(x), _p(wk), _p(bias), _p(stats), _p(x1), None, _p(n[0]), _p(n[1]), B, H, W,
              C, float(eps), st)
        g = _new_planes((B, H, W, Ch), x.device)
        _conv_tc(n, _cached_pack("tc", w1, _pack_tc), b1, g, B, H, W, C, Ch, 1, CONV_TC_SAME, st)
        _conv_tc(g, _cached_pack("tc", w2, _pack_tc), b2, y, B, H, W, Ch, C, 1, CONV_TC_SAME, st, res=x1)
        return y
    n2 = torch.empty_like(x)
    _call("muse_paella_resblock_spatial", _p(x), _p(wk), _p(bias), _p(stats), _p(x1), _p(n2), None, None, B, H, W, C,
          float(eps), st)
    g = torch.empty(B, H, W, Ch, dtype=torch.float32, device=x.device)
    _call("muse_conv2d_nhwc", _p(n2), _p(_cached_pack("simt", w1, _pack_simt)), _p(b1), None, _p(g), B, H, W, C, Ch, 1,
          CONV_GELU, st)
    _call("muse_conv2d_nhwc", _p(g), _p(_cached_pack("simt", w2, _pack_simt)), _p(b2), _p(x1), _p(y), B, H, W, Ch, C, 1,
          CONV_SAME, st)
    return y


def conv2d_unshuffle(x, w, bias=None):
    """nn.PixelUnshuffle(2) then the 1x1 conv w [Cout, 4*Cin, 1, 1] (Paella in_block): fp32 NHWC [B,2H,2W,Cin] ->
    [B,H,W,Cout].  Tensor cores: an im2col of the 2x2 blocks into 64 columns, then one 1x1 convolution; SIMT: the same
    weights as a 2x2 stride-2 convolution."""
    st = _prep(x)
    B, Hi, Wi, Cin = x.shape
    H, W, Cout = Hi // 2, Wi // 2, w.shape[0]
    y = torch.empty(B, H, W, Cout, dtype=torch.float32, device=x.device)
    b = None if bias is None else bias.detach().float()
    if 4 * Cin <= 64 and _tc_route(H, W, 64, Cout, 1):
        _conv_tc(_im2col(x, H, W, 2, st), _cached_pack("stem", w, _pack_stem), b, y, B, H, W, 64, Cout, 1, CONV_TC_SAME, st)
        return y
    wk = _cached_pack("unshuffle", w, lambda wf: _pack_simt(wf.view(Cout, Cin, 2, 2)))
    _call("muse_conv2d_nhwc", _p(x), _p(wk), _p(b), None, _p(y), B, H, W, Cin, Cout, 2, CONV_STRIDE2, st)
    return y


def _pack_s2p1(wf):
    """Conv2d(4, 2, 1) weight [Cout, Cin, 4, 4] -> bf16 planes [Cout, 9 taps * 4 * Cin] for a 3x3 pad-1 convolution over the
    space-to-depth grid: tap (a, b) and plane (p, q) hold w[:, :, 2a + p - 1, 2b + q - 1] (zero outside 0..3)."""
    Cout, Cin = wf.shape[0], wf.shape[1]
    wk = torch.zeros(Cout, 3, 3, 2, 2, Cin, dtype=torch.float32, device=wf.device)  # [co, a, b, p, q, ci]
    for a in range(3):
        for b in range(3):
            for p_ in (0, 1):
                for q in (0, 1):
                    kh, kw = 2 * a + p_ - 1, 2 * b + q - 1
                    if 0 <= kh <= 3 and 0 <= kw <= 3:
                        wk[:, a, b, p_, q] = wf[:, :, kh, kw]
    return _planes(wk.reshape(Cout, -1).contiguous())


def conv2d_s2p1(x, w, bias=None):
    """nn.Conv2d(k=4, s=2, p=1) on fp32 NHWC [B,2H,2W,Cin] -> [B,H,W,Cout].  Tensor cores: space-to-depth + hi/lo split,
    then a stride-1 3x3 convolution over the 4*Cin planes (16 of the 36 weight taps are non-zero); SIMT: stride-2 mode."""
    st = _prep(x)
    B, Hi, Wi, Cin = x.shape
    H, W, Cout = Hi // 2, Wi // 2, w.shape[0]
    y = torch.empty(B, H, W, Cout, dtype=torch.float32, device=x.device)
    b = None if bias is None else bias.detach().float()
    if _tc_route(H, W, 4 * Cin, Cout, 3):
        _conv_tc(_split_s2d(x, st), _cached_pack("s2p1", w, _pack_s2p1), b, y, B, H, W, 4 * Cin, Cout, 3, CONV_TC_SAME, st)
        return y
    _call("muse_conv2d_nhwc", _p(x), _p(_cached_pack("simt", w, _pack_simt)), _p(b), None, _p(y), B, H, W, Cin, Cout, 4,
          CONV_S2P1, st)
    return y


def _pack_transpose_parities(wf):
    """ConvTranspose2d(4, 2, 1) weight [Cin, Cout, 4, 4] -> [4 parities][Cout][4 taps * Cin]: output pixel (2i + py, 2j + px)
    reads input (i + a + py - 1, j + b + px - 1) with kernel tap (3 - 2a - py, 3 - 2b - px), a, b in {0, 1}."""
    mats = []
    for py in (0, 1):
        for px in (0, 1):
            taps = [wf[:, :, 3 - 2 * a - py, 3 - 2 * b - px].t() for a in (0, 1) for b in (0, 1)]  # [Cout, Cin] each
            mats.append(torch.stack(taps, dim=1).reshape(wf.shape[1], -1))  # [Cout, 4*Cin], column (a*2+b)*Cin + ci
    return torch.stack(mats)


def conv_transpose2d_s2(x, w, bias=None):
    """nn.ConvTranspose2d(k=4, s=2, p=1) on fp32 NHWC [B,H,W,Cin] with w [Cin, Cout, 4, 4] -> [B,2H,2W,Cout]: four 2x2
    parity convolutions of the input (MUSE_CONV_TC_UPSAMPLE2X, or MUSE_CONV_TRANSPOSE_S2 of the SIMT kernel)."""
    st = _prep(x)
    B, Hi, Wi, Cin = x.shape
    H, W, Cout = 2 * Hi, 2 * Wi, w.shape[1]
    y = torch.empty(B, H, W, Cout, dtype=torch.float32, device=x.device)
    b = None if bias is None else bias.detach().float()
    if _tc_route(H, W, Cin, Cout, 3, upsample2x=True):
        wk = _cached_pack("convT", w, lambda wf: _planes(_pack_transpose_parities(wf).reshape(4 * Cout, -1).contiguous()))
        _conv_tc(_split(x, st), wk, b, y, B, H, W, Cin, Cout, 3, CONV_TC_UPSAMPLE2X, st)
        return y
    wk = _cached_pack("convT_simt", w, lambda wf: _pack_transpose_parities(wf).transpose(1, 2).contiguous())
    _call("muse_conv2d_nhwc", _p(x), _p(wk), _p(b), None, _p(y), B, H, W, Cin, Cout, 4, CONV_TRANSPOSE_S2, st)
    return y


def conv1x1_pixel_shuffle(x, w, bias=None):
    """1x1 conv w [Cout, Cin, 1, 1] then nn.PixelShuffle(2) (Paella out_block), folded into the convolution's store:
    fp32 NHWC [B,H,W,Cin] -> [B,2H,2W,Cout/4]."""
    st = _prep(x)
    B, H, W, Cin = x.shape
    Cout = w.shape[0]
    y = torch.empty(B, 2 * H, 2 * W, Cout // 4, dtype=torch.float32, device=x.device)
    b = None if bias is None else bias.detach().float()
    if _tc_route(H, W, Cin, Cout, 1):
        _conv_tc(_split(x, st), _cached_pack("tc", w, _pack_tc), b, y, B, H, W, Cin, Cout, 1, CONV_TC_PIXEL_SHUFFLE, st)
        return y
    _call("muse_conv2d_nhwc", _p(x), _p(_cached_pack("simt", w, _pack_simt)), _p(b), None, _p(y), B, H, W, Cin, Cout, 1,
          CONV_PIXEL_SHUFFLE, st)
    return y
