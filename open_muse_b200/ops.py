"""Thin tensor-level wrappers over the C ABI (pointers, sizes, current CUDA stream).

PyTorch here is plumbing only: device memory (``torch.empty``), streams, autograd bookkeeping.
Every function launches hand-written sm_90a kernels from libmuse_b200.so and raises if the
library is missing or the tensors are not CUDA tensors -- there is no fallback path.
"""
from __future__ import annotations

import os

import torch

from . import _lib

F32, BF16 = 0, 1
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
    raise TypeError(f"unsupported dtype {t.dtype}")


def _p(t):
    return None if t is None else t.data_ptr()


_KERNELS_PER_CALL = {"muse_norm2_bwd": 3, "muse_sample_step": 2, "muse_gemm_bf16_splitk": 2, "muse_adamw_ema_step": 4, "muse_ce_fwd": 2, "muse_attn_bwd": 2, "muse_embed_bwd": 2, "muse_embed_bwd_sorted": 4, "muse_vq_argmin": 2, "muse_vq_soft_code": 3,
                     "muse_groupnorm_silu_nhwc": 3, "muse_grn_fwd": 3, "muse_grn_bwd": 3,
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


def linear_fwd(x, w, out_dtype=torch.bfloat16, res=None, n_valid=None):
    """y[T,N] = x[T,K] @ w[N,K]^T.  res (fp32 [T,N]) selects the fused residual epilogue."""
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
def norm_fwd(x, w, eps, out_dtype, res=None, act=0, rms=0, save_stats=True):
    """act: 0 none, 1 GELU(x) first, 2 GLU (x is [rows, 2H] = [a | b], the normalised value is gelu(a) * b)."""
    st = _prep(x)
    rows = x.shape[0]
    H = x.shape[1] // 2 if act == 2 else x.shape[1]
    y = torch.empty(rows, H, dtype=out_dtype, device=x.device)
    if save_stats:
        stats = torch.empty(2, rows, dtype=torch.float32, device=x.device)
        mean, rstd = stats[0], stats[1]
    else:
        stats = mean = rstd = None
    _call("muse_norm_fwd", _p(x), _dt(x), _p(w), _p(res), _p(y), _dt(y), _p(mean), _p(rstd), rows, H, float(eps),
          act, rms, st)
    return y, stats


_bf16_copies = {}


def take_bf16_copy(t):
    """The bf16 copy norm_bwd(..., bf16_copy=True) produced alongside the fp32 tensor `t` (or None): consumed once."""
    hit = _bf16_copies.pop(t.data_ptr(), None)
    if hit is not None and hit[0] == (t._version, tuple(t.shape)):
        return hit[1]
    return None


def norm_bwd(dy, x, w, stats, dx_dtype, dw=None, dres=None, act=0, rms=0, y_fwd=None, want_dw=False, bf16_copy=False):
    """y_fwd: the saved forward output (act=2, bf16 only) -- lets the kernel skip one GELU pass over [a | b].
    dw: fp32 [H] buffer the weight gradient is ADDED to (atomics; caller zero-fills).  want_dw=True instead returns
    (dx, dw) with a freshly stored dw reduced in a fixed order (run-to-run bit-identical)."""
    st = _prep(x)
    rows = x.shape[0]
    H = x.shape[1] // 2 if act == 2 else x.shape[1]
    dx = torch.empty(x.shape, dtype=dx_dtype, device=x.device)
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
    _call("muse_norm_bwd", _p(dy), _dt(dy), _p(x), _dt(x), _p(w), _p(stats[0]), _p(stats[1]), _p(dres), _p(y_fwd), _p(dx),
          _dt(dx), _p(copy), _p(dw), _p(ws), rows, H, act, rms, st)
    return (dx, dw) if want_dw else dx


def norm2_fwd(a, res, w1, w2, eps, rms1=0, rms2=0, save_stats=True):
    """x2 = res + norm1(a) * w1 (fp32), h2 = norm2(x2) * w2 (bf16) in one pass; stats = [mean1, rstd1, mean2, rstd2]."""
    st = _prep(a)
    rows, H = a.shape
    x2 = torch.empty(rows, H, dtype=torch.float32, device=a.device)
    h2 = torch.empty(rows, H, dtype=torch.bfloat16, device=a.device)
    stats = torch.empty(4, rows, dtype=torch.float32, device=a.device) if save_stats else None
    sp = [None] * 4 if stats is None else [stats[i] for i in range(4)]
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


# ------------------------------------------------------------------------------------------ GLU
def glu_fwd(ab):
    st = _prep(ab)
    rows, two_i = ab.shape
    out = torch.empty(rows, two_i // 2, dtype=torch.bfloat16, device=ab.device)
    _call("muse_glu_fwd", _p(ab), _p(out), rows, two_i // 2, st)
    return out


def glu_bwd(ab, dout):
    st = _prep(ab)
    rows, two_i = ab.shape
    dab = torch.empty_like(ab)
    _call("muse_glu_bwd", _p(ab), _p(dout), _p(dab), rows, two_i // 2, st)
    return dab


# ------------------------------------------------------------------------------------------ attention
def attn_fwd(q, k, v, B, nh, Sq, Skv, scale, head_dim=64):
    """q: [B*Sq, *] view with head h at columns h*head_dim; k, v: [B*Skv, *] views.  Returns ctx [B*Sq, nh*head_dim], lse.
    head_dim: 64 (default) or 48 (configs/imagenet.yaml: hidden 768 / 16 heads)."""
    st = _prep(q)
    hd = int(head_dim)
    o = torch.empty(B * Sq, nh * hd, dtype=torch.bfloat16, device=q.device)
    lse = torch.empty(B, nh, Sq, dtype=torch.float32, device=q.device)
    _call("muse_attn_fwd", _p(q), _p(k), _p(v), _p(o), _p(lse), B, nh, Sq, Skv, hd, q.stride(0), k.stride(0),
          v.stride(0), o.stride(0), float(scale), st)
    return o, lse


def attn_bwd(q, k, v, o, do, lse, dq, dk, dv, B, nh, Sq, Skv, scale, head_dim=64):
    st = _prep(q)
    dvec = torch.empty(B, nh, Sq, dtype=torch.float32, device=q.device)
    _call("muse_attn_bwd", _p(q), _p(k), _p(v), _p(o), _p(do), _p(lse), _p(dvec), _p(dq), _p(dk), _p(dv), B, nh, Sq,
          Skv, int(head_dim), q.stride(0), k.stride(0), v.stride(0), o.stride(0), do.stride(0), dq.stride(0), dk.stride(0),
          dv.stride(0), float(scale), st)


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
    shift per sample, row pitch mod.stride(0)) of the batched adaLN mapper output."""
    st = _prep(a)
    rows, H = a.shape
    y = torch.empty(rows, H, dtype=out_dtype, device=a.device)
    r_out = torch.empty(rows, H, dtype=torch.float32, device=a.device) if want_residual else None
    _call("muse_add_norm_mod_fwd", _p(a), _dt(a), _p(residual), _p(w), _p(mod), 0 if mod is None else mod.stride(0),
          int(rows_per_sample), _p(r_out), _p(y), _dt(y), rows, H, float(eps), int(rms), st)
    return r_out, y


def dwconv3x3_norm(x, wk, norm_w, B, hh, ww, eps, rms, save_conv=False):
    """x fp32 [B*hh*ww, C] token-major, wk fp32 [9, C] -> bf16 [B*hh*ww, C] = Norm2D(depthwise3x3(x)).
    save_conv: also return the bf16 conv output (needed by dwconv3x3_norm_bwd)."""
    st = _prep(x)
    C = x.shape[1]
    y = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    conv = torch.empty_like(y) if save_conv else None
    _call("muse_dwconv3x3_norm_fwd", _p(x), _p(wk), _p(norm_w), _p(y), _p(conv), B, hh, ww, C, float(eps), int(rms), st)
    return (y, conv) if save_conv else y


def grn(x, gamma, beta, B, HW, save_stats=False):
    """bf16 [B*HW, C] -> bf16: GELU + GlobalResponseNorm.  save_stats: also return (sumsq, nx) for grn_bwd."""
    st = _prep(x)
    C = x.shape[1]
    out = torch.empty_like(x)
    ws = torch.empty(2, B, C, dtype=torch.float32, device=x.device)
    _call("muse_grn_fwd", _p(x), _p(gamma), _p(beta), _p(out), _p(ws[0]), _p(ws[1]), B, HW, C, st)
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


def grn_bwd(x, dout, stats, gamma, dgamma, dbeta, B, HW):
    st = _prep(x)
    C = x.shape[1]
    dx = torch.empty_like(x)
    ws = torch.empty(B, C, dtype=torch.float32, device=x.device)
    _call("muse_grn_bwd", _p(x), _p(dout), _p(stats[1]), _p(stats[0]), _p(gamma), _p(ws), _p(dx), _p(dgamma), _p(dbeta), B, HW,
          C, st)
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
_wk_cache = {}

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


def _lo_like(hi):
    return None if _conv_state["single"] else torch.empty_like(hi)


def _tc_mode(mode):
    return mode | 8 if _conv_state["single"] else mode


def _packed_conv_weight(w):
    """[Cout, Cin, kh, kw] -> [kh*kw*Cin, Cout] (tap-major, then input channel); cached per live weight tensor
    (weakref identity + storage pointer + version counter, so a recycled id() or an in-place update never hits)."""
    import weakref

    key = (w.data_ptr(), w._version, tuple(w.shape), w.device)
    hit = _wk_cache.get(id(w))
    if hit is not None and hit[0]() is w and hit[1] == key:
        return hit[2]
    wk = w.detach().float().permute(2, 3, 1, 0).reshape(-1, w.shape[0]).contiguous()
    if len(_wk_cache) > 4096:
        _wk_cache.clear()
    _wk_cache[id(w)] = (weakref.ref(w), key, wk)
    return wk


def _packed_conv_weight_split(w):
    """[Cout, Cin, kh, kw] -> bf16 planes (hi, lo) of [Cout, kh*kw*Cin] (tap-major, then input channel), w = hi + lo."""
    import weakref

    key = (w.data_ptr(), w._version, tuple(w.shape), w.device)
    hit = _wk_cache.get(("split", id(w)))
    if hit is not None and hit[0]() is w and hit[1] == key:
        return hit[2]
    wk = w.detach().float().permute(0, 2, 3, 1).reshape(w.shape[0], -1).contiguous()
    hi = wk.to(torch.bfloat16)
    lo = (wk - hi.float()).to(torch.bfloat16)
    if len(_wk_cache) > 4096:
        _wk_cache.clear()
    _wk_cache[("split", id(w))] = (weakref.ref(w), key, (hi, lo))
    return hi, lo


def conv_uses_tensor_cores(H, W, Cin, Cout, k):
    """Route of conv2d(): wgmma bf16x3 implicit GEMM unless the geometry is unsupported or MUSE_B200_CONV=simt.
    Stems with k*k*Cin <= 64 go through an im2col to 64 columns and run as a 1x1 convolution."""
    if _conv_state["route"] == "simt":  # private test hook (ops.conv_route): cross-check against the fp32 FMA kernels
        return False
    if Cin % 64 != 0 and k * k * Cin <= 64:
        return bool(_lib.load().muse_conv2d_tc_supported(H, W, 64, Cout, 1))
    return bool(_lib.load().muse_conv2d_tc_supported(H, W, Cin, Cout, k))


def _packed_conv_weight_split_stem(w):
    """Stem weight [Cout, Cin, k, k] with k*k*Cin <= 64 -> bf16 (hi, lo) of [Cout, 64], columns tap-major, zero padded."""
    import weakref

    key = (w.data_ptr(), w._version, tuple(w.shape), w.device)
    hit = _wk_cache.get(("stem", id(w)))
    if hit is not None and hit[0]() is w and hit[1] == key:
        return hit[2]
    wk = torch.zeros(w.shape[0], 64, dtype=torch.float32, device=w.device)
    flat = w.detach().float().permute(0, 2, 3, 1).reshape(w.shape[0], -1)
    wk[:, : flat.shape[1]] = flat
    hi = wk.to(torch.bfloat16)
    lo = (wk - hi.float()).to(torch.bfloat16)
    _wk_cache[("stem", id(w))] = (weakref.ref(w), key, (hi, lo))
    return hi, lo


def _gn_scratch(x):
    B, H, W, C = x.shape
    n_ws = _lib.load().muse_groupnorm_workspace_floats(B, H * W, C)
    if n_ws < 0:
        raise _lib.MuseB200Error(f"groupnorm: unsupported channel count {C}")
    return (torch.empty(n_ws, dtype=torch.float32, device=x.device),
            torch.empty(B * C * 2, dtype=torch.float32, device=x.device))


def _packed_conv_weight_upsample(w):
    """3x3 weight of an UpsamplingBlock conv -> bf16 (hi, lo) of the four stacked 2x2 parity matrices [4*Cout, 4*Cin].

    Output pixel (2y+py, 2x+px) of conv3x3(nearest_x2(v)) reads only v[y+a+py-1, x+b+px-1] for a, b in {0, 1}; the 3x3
    taps that land on the same low-resolution pixel are summed (fp32): rows R(0,0)={0}, R(0,1)={1,2}, R(1,0)={0,1},
    R(1,1)={2} (same for columns)."""
    import weakref

    key = (w.data_ptr(), w._version, tuple(w.shape), w.device)
    hit = _wk_cache.get(("up", id(w)))
    if hit is not None and hit[0]() is w and hit[1] == key:
        return hit[2]
    wf = w.detach().float()  # [Cout, Cin, 3, 3]
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
    wk = torch.cat(mats, dim=0).contiguous()  # [4*Cout, 4*Cin], row = parity*Cout + co
    hi = wk.to(torch.bfloat16)
    lo = (wk - hi.float()).to(torch.bfloat16)
    _wk_cache[("up", id(w))] = (weakref.ref(w), key, (hi, lo))
    return hi, lo


def _conv_stats_buffer(y, H, W, Cin, Cout, k, up=0):
    """The tensor-core convolution's epilogue leaves per-tile {sum, sumsq} of its output: they ride along on the output
    tensor (``y._gn_stats``) so that a following conv2d(gn=...) skips the GroupNorm statistics pass over y."""
    if Cout <= 16 or Cout % 32 != 0:
        return None, 0
    tiles = _lib.load().muse_conv2d_tc_tiles_per_image(H, W, Cin, Cout, k, up)
    stats = torch.empty(y.shape[0], tiles, Cout, 2, dtype=torch.float32, device=y.device)
    y._gn_stats = (stats, tiles)
    return stats, tiles


def conv2d(x, w, bias=None, residual=None, upsample2x=False, gn=None):
    """Conv2dSame on fp32 NHWC x [B,Hi,Wi,Cin] with the nn.Conv2d weight w [Cout,Cin,k,k] -> fp32 NHWC [B,H,W,Cout].

    gn = (gamma, beta, groups, eps) applies GroupNorm+SiLU to x first (the ResnetBlock pattern); upsample2x applies the
    nearest x2 upsample first.  Heavy layers run on the tensor cores (csrc/conv_tc.cu) with operands carried as bf16
    hi/lo planes; the GroupNorm kernel emits the planes directly."""
    st = _prep(x)
    B, Hi, Wi, Cin = x.shape
    H, W = (Hi * 2, Wi * 2) if upsample2x else (Hi, Wi)
    Cout, k = w.shape[0], w.shape[2]
    y = torch.empty(B, H, W, Cout, dtype=torch.float32, device=x.device)
    b = None if bias is None else bias.detach().float()
    if conv_uses_tensor_cores(H, W, Cin, Cout, k) and Cin % 64 != 0:
        assert gn is None and not upsample2x
        hi = torch.empty(B, H, W, 64, dtype=torch.bfloat16, device=x.device)
        lo = _lo_like(hi)
        _call("muse_im2col_split_nhwc", _p(x), _p(hi), _p(lo), B, H, W, Cin, k, st)
        w_hi, w_lo = _packed_conv_weight_split_stem(w)
        stats, tiles = _conv_stats_buffer(y, H, W, 64, Cout, 1)
        _call("muse_conv2d_nhwc_tc", _p(hi), _p(lo), _p(w_hi), _p(w_lo), _p(b), _p(residual), _p(y), _p(stats), B, H, W, 64,
              Cout, 1, _tc_mode(0), st)
        return y
    if upsample2x and gn is None and conv_uses_tensor_cores(H, W, Cin, Cout, k) and \
            _lib.load().muse_conv2d_tc_tiles_per_image(H, W, Cin, Cout, k, 1) > 0:
        # nearest x2 + 3x3 conv as four 2x2 parity convolutions on the low-resolution planes (2.25x fewer FLOPs)
        hi = torch.empty(B, Hi, Wi, Cin, dtype=torch.bfloat16, device=x.device)
        lo = _lo_like(hi)
        _call("muse_split_bf16_nhwc", _p(x), _p(hi), _p(lo), B, Hi, Wi, Cin, 0, st)
        w_hi, w_lo = _packed_conv_weight_upsample(w)
        stats, tiles = _conv_stats_buffer(y, H, W, Cin, Cout, k, 1)
        _call("muse_conv2d_nhwc_tc", _p(hi), _p(lo), _p(w_hi), _p(w_lo), _p(b), _p(residual), _p(y), _p(stats), B, H, W, Cin,
              Cout, k, _tc_mode(1), st)
        return y
    if conv_uses_tensor_cores(H, W, Cin, Cout, k):
        hi = torch.empty(B, H, W, Cin, dtype=torch.bfloat16, device=x.device)
        lo = _lo_like(hi)
        if gn is not None:
            assert not upsample2x
            pre = getattr(x, "_gn_stats", None)  # {sum, sumsq} tiles left by the convolution that produced x
            if pre is not None:
                ws, tiles = pre
                ss = torch.empty(B * Cin * 2, dtype=torch.float32, device=x.device)
            else:
                (ws, ss), tiles = _gn_scratch(x), 0
            _call("muse_groupnorm_silu_nhwc", _p(x), _p(gn[0].detach().float()), _p(gn[1].detach().float()), None, _p(hi),
                  _p(lo), _p(ws), _p(ss), B, H * W, Cin, int(gn[2]), float(gn[3]), tiles, int(gn[4]) if len(gn) > 4 else 1, st)
        else:
            _call("muse_split_bf16_nhwc", _p(x), _p(hi), _p(lo), B, H, W, Cin, 1 if upsample2x else 0, st)
        w_hi, w_lo = _packed_conv_weight_split(w)
        stats, tiles = _conv_stats_buffer(y, H, W, Cin, Cout, k)
        _call("muse_conv2d_nhwc_tc", _p(hi), _p(lo), _p(w_hi), _p(w_lo), _p(b), _p(residual), _p(y), _p(stats), B, H, W, Cin,
              Cout, k, _tc_mode(0), st)
        return y
    if gn is not None:
        x = groupnorm_silu(x, *gn)
    _call("muse_conv2d_nhwc", _p(x), _p(_packed_conv_weight(w)), _p(b), _p(residual), _p(y), B, H, W, Cin, Cout, k,
          1 if upsample2x else 0, st)
    return y


def groupnorm_silu(x, gamma, beta, groups, eps, silu=1):
    """GroupNorm (+ SiLU unless silu=0), fp32 NHWC in and out."""
    st = _prep(x)
    B, H, W, C = x.shape
    y = torch.empty_like(x)
    ws, ss = _gn_scratch(x)
    _call("muse_groupnorm_silu_nhwc", _p(x), _p(gamma.detach().float()), _p(beta.detach().float()), _p(y), None, None,
          _p(ws), _p(ss), B, H * W, C, groups, float(eps), 0, int(silu), st)
    return y


def _packed_conv_weight_down(w):
    """3x3 stride-2 weight (pad (0,1,0,1)) -> bf16 (hi, lo) [Cout, 4 taps * 4 * Cin] for the space-to-depth form:
    tap (a, b) in {0,1}^2 and plane (p, q) hold w[:, :, 2a + p, 2b + q] (zero where 2a + p or 2b + q exceeds 2)."""
    import weakref

    key = (w.data_ptr(), w._version, tuple(w.shape), w.device)
    hit = _wk_cache.get(("down", id(w)))
    if hit is not None and hit[0]() is w and hit[1] == key:
        return hit[2]
    wf = w.detach().float()
    Cout, Cin = wf.shape[0], wf.shape[1]
    wk = torch.zeros(Cout, 2, 2, 2, 2, Cin, dtype=torch.float32, device=w.device)  # [co, a, b, p, q, ci]
    for a in (0, 1):
        for b in (0, 1):
            for p_ in (0, 1):
                for q in (0, 1):
                    kh, kw = 2 * a + p_, 2 * b + q
                    if kh <= 2 and kw <= 2:
                        wk[:, a, b, p_, q] = wf[:, :, kh, kw]
    wk = wk.reshape(Cout, -1).contiguous()
    hi = wk.to(torch.bfloat16)
    lo = (wk - hi.float()).to(torch.bfloat16)
    _wk_cache[("down", id(w))] = (weakref.ref(w), key, (hi, lo))
    return hi, lo


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
    if _conv_state["route"] != "simt" and (4 * Cin) % 64 == 0 and \
            _lib.load().muse_conv2d_tc_supported(H, W, 4 * Cin, Cout, 2):
        hi = torch.empty(B, H, W, 4 * Cin, dtype=torch.bfloat16, device=x.device)
        lo = _lo_like(hi)
        _call("muse_split_s2d_bf16_nhwc", _p(x), _p(hi), _p(lo), B, H, W, Cin, st)
        w_hi, w_lo = _packed_conv_weight_down(w)
        stats, tiles = _conv_stats_buffer(y, H, W, 4 * Cin, Cout, 2)
        _call("muse_conv2d_nhwc_tc", _p(hi), _p(lo), _p(w_hi), _p(w_lo), _p(b), None, _p(y), _p(stats), B, H, W, 4 * Cin, Cout,
              2, _tc_mode(2), st)
        return y
    _call("muse_conv2d_nhwc", _p(x), _p(_packed_conv_weight(w)), _p(b), None, _p(y), B, H, W, Cin, Cout, 3, 2, st)
    return y


def attention_single_head(q, k, v, B, hh, ww):
    """softmax(q k^T / sqrt(C)) v per image with ONE head of width C (AttnBlock of the taming VQGAN, :148-174), fp32-faithful:
    q, k, v fp32 [B*hh*ww, C] -> fp32 [B*hh*ww, C].  Both products run as 1x1 tensor-core convolutions whose weights are
    the image's own keys / values (per-image weight mode of muse_conv2d_nhwc_tc); small geometries loop over the images
    with the SIMT kernel."""
    import os

    st = _prep(q)
    HW, C = hh * ww, q.shape[1]
    lib = _lib.load()
    scale = float(C) ** -0.5
    out = torch.empty(B * HW, C, dtype=torch.float32, device=q.device)
    scores = torch.empty(B * HW, HW, dtype=torch.float32, device=q.device)
    vt = torch.empty(B, C, HW, dtype=torch.float32, device=q.device)
    _call("muse_transpose_batched", _p(v), _p(vt), B, HW, C, st)
    tc = _conv_state["route"] != "simt" and lib.muse_conv2d_tc_supported(hh, ww, C, HW, 1) and \
        lib.muse_conv2d_tc_supported(hh, ww, HW, C, 1) and HW % 64 == 0 and C % 64 == 0

    def planes(t):
        hi = torch.empty(t.shape, dtype=torch.bfloat16, device=t.device)
        lo = torch.empty_like(hi)
        _call("muse_split_bf16_nhwc", _p(t), _p(hi), _p(lo), 1, 1, t.numel() // t.shape[-1], t.shape[-1], 0, st)
        return hi, lo

    if tc:
        qh, ql = planes(q)
        kh, kl = planes(k)        # per-image weights [B][HW keys][C]
        _call("muse_conv2d_nhwc_tc", _p(qh), _p(ql), _p(kh), _p(kl), None, None, _p(scores), None, B, hh, ww, C, HW, 1, 4, st)
        ph = torch.empty(B * HW, HW, dtype=torch.bfloat16, device=q.device)
        pl = torch.empty_like(ph)
        _call("muse_softmax_split_rows", _p(scores), _p(ph), _p(pl), None, B * HW, HW, scale, st)
        vh, vl = planes(vt)       # per-image weights [B][C][HW keys]
        _call("muse_conv2d_nhwc_tc", _p(ph), _p(pl), _p(vh), _p(vl), None, None, _p(out), None, B, hh, ww, HW, C, 1, 4, st)
        return out
    kt = torch.empty(B, C, HW, dtype=torch.float32, device=q.device)
    _call("muse_transpose_batched", _p(k), _p(kt), B, HW, C, st)
    probs = torch.empty_like(scores)
    for b in range(B):  # SIMT weights are [K, Cout]: k_b^T for the scores, v_b for the output
        qb, sb = q[b * HW:(b + 1) * HW], scores[b * HW:(b + 1) * HW]
        _call("muse_conv2d_nhwc", _p(qb), _p(kt[b]), None, None, _p(sb), 1, hh, ww, C, HW, 1, 0, st)
    _call("muse_softmax_split_rows", _p(scores), None, None, _p(probs), B * HW, HW, scale, st)
    for b in range(B):
        pb, ob = probs[b * HW:(b + 1) * HW], out[b * HW:(b + 1) * HW]
        _call("muse_conv2d_nhwc", _p(pb), _p(v[b * HW:(b + 1) * HW]), None, None, _p(ob), 1, hh, ww, HW, C, 1, 0, st)
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
