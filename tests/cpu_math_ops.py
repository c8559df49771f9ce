"""NUMERIC CPU stand-ins for the libmuse_b200 entry points the host code calls (test infrastructure; the product never
imports this).  Each function restates the documented contract of one ``open_muse_b200.ops`` wrapper (or, for the fused
optimizer, of the C entry point itself) in plain torch, so everything ABOVE the C ABI -- the autograd Functions of
MaskGitTransformer and MaskGiTUViT_v2, the packed-operand pointer table, the order in which gradients are handed back, the
generate2 loops, the tokenizers' module wiring, PipelineMuse, FusedAdamW's launch table -- can be run end to end WITHOUT a GPU
and compared with what the unmodified reference computed (tests/golden/*.pt).  The kernels themselves are checked on the
GPU (tests/test_kernels_gpu.py, tests/test_model_gpu.py, ...).

Two modes:
  exact=True   ``torch.bfloat16`` is aliased to ``torch.float32`` while the stand-ins are installed, so every tensor the host
               code allocates "in bf16" carries full fp32 values: the host wiring must then reproduce the reference's fp32
               outputs and gradients to ~1e-5 -- a mis-routed or mis-scaled gradient cannot hide under bf16 noise.
  exact=False  outputs are rounded to the dtype the kernel writes (bf16 activations, fp32 residual stream / statistics /
               weight gradients): the precision RECIPE of the hot path, emulated on the CPU.

Backward stand-ins use the saved statistics (mean, rstd) exactly as the kernels do -- norm_bwd / norm2_bwd receive no eps --
so a wrong statistics row handed over by the host shows up as a wrong gradient; pointer tables (muse_pack_bf16,
muse_adamw_ema_step) are dereferenced with ctypes like the library dereferences them.
"""
import ctypes

import torch
import torch.nn.functional as F

F32 = torch.float32


def _bf():  # looked up at call time: aliased to float32 in exact mode
    return torch.bfloat16


def _act(x, act):
    x = x.float()
    if act == 1:
        return F.gelu(x)
    if act == 2:
        h = x.shape[1] // 2
        return F.gelu(x[:, :h]) * x[:, h:]
    return x


def _stats(x, eps, rms):
    if rms:
        mean = torch.zeros(x.shape[0])
        rstd = torch.rsqrt(x.pow(2).mean(-1) + eps)
    else:
        mean = x.mean(-1)
        rstd = torch.rsqrt(x.var(-1, unbiased=False) + eps)
    return mean, rstd


def _norm_apply(x, w, mean, rstd):
    y = (x - mean[:, None]) * rstd[:, None]
    return y if w is None else y * w.float()


def _norm_grad(dy, x, w, mean, rstd, rms):
    """gradient of y = ((x - mean) * rstd) * w w.r.t. x and w from the SAVED statistics (layer norm: mean / rstd depend on
    x; RMS norm: mean is 0 and only rstd depends on x)."""
    dy = dy.float()
    xhat = (x - mean[:, None]) * rstd[:, None]
    g = dy if w is None else dy * w.float()
    c2 = (g * xhat).mean(-1, keepdim=True)
    dx = rstd[:, None] * (g - xhat * c2 - (0.0 if rms else g.mean(-1, keepdim=True)))
    return dx, (dy * xhat).sum(0)


# ------------------------------------------------------------------------------------------------------------- GEMMs
def linear_fwd(x, w, out_dtype=None, res=None, n_valid=None):
    n = w.shape[0] if n_valid is None else n_valid
    assert x.dtype == _bf() and w.dtype == _bf() and x.shape[1] == w.shape[1], (x.dtype, w.dtype, x.shape, w.shape)
    y = x.float() @ w[:n].float().t()
    if res is not None:
        assert res.dtype == F32 and res.shape == y.shape
        return y + res
    return y.to(_bf() if out_dtype is None else out_dtype)


def linear_dgrad(dy, w, out_dtype=None):
    assert dy.dtype == _bf() and w.dtype == _bf() and dy.shape[1] == w.shape[0]
    return (dy.float() @ w.float()).to(_bf() if out_dtype is None else out_dtype)


def linear_wgrad_det(dy, x, out=None):
    assert dy.dtype == _bf() and x.dtype == _bf() and dy.shape[0] == x.shape[0]
    dw = dy.float().t() @ x.float()
    if out is not None:
        out.copy_(dw)
        return out
    return dw


def gemm(a, b, c, M, N, K, lda, ldb, ldc, a_mn=0, b_mn=0, epi=0, res=None):
    """only the K-major x K-major form the head uses: c[:M, :N] = a[:M, :K] @ b[:N, :K]^T"""
    assert a_mn == 0 and b_mn == 0 and res is None and a.stride(0) == lda and b.stride(0) == ldb and c.stride(0) == ldc
    c[:M, :N] = (a[:M, :K].float() @ b[:N, :K].float().t()).to(c.dtype)
    return c


def pack_bf16(table, n_entries, total_blocks):
    """the pointer table of _PackedWeights: rows (src fp32 pointer, dst bf16 pointer, numel, first block)"""
    two_byte = torch.bfloat16 != torch.float32
    for src, dst, numel, _ in table[:n_entries].tolist():
        s = torch.frombuffer((ctypes.c_float * numel).from_address(src), dtype=F32)
        if two_byte:
            d = torch.frombuffer((ctypes.c_uint16 * numel).from_address(dst), dtype=torch.bfloat16)
        else:
            d = torch.frombuffer((ctypes.c_float * numel).from_address(dst), dtype=F32)
        d.copy_(s)


def cast_bf16(x):
    return x.to(_bf())


def take_bf16_copy(t):
    return None


# --------------------------------------------------------------------------------------------------------- embedding
def embed_fwd(ids, word, pos):
    B, S = ids.shape
    out = word.float()[ids.reshape(-1)]
    if pos is not None:
        out = out + pos.float()[:S].repeat(B, 1)
    return out


def embed_bwd_det(ids, dx, vocab, n_pos):
    B, S = ids.shape
    assert dx.dtype == F32 and dx.shape[0] == B * S
    dword = torch.zeros(vocab, dx.shape[1]).index_add_(0, ids.reshape(-1), dx)
    dpos = None
    if n_pos:
        dpos = torch.zeros(n_pos, dx.shape[1])
        dpos[:S] = dx.view(B, S, -1).sum(0)
    return dword, dpos


# ------------------------------------------------------------------------------------------------------------- norms
def norm_fwd(x, w, eps, out_dtype, res=None, act=0, rms=0, save_stats=True):
    xa = _act(x, act)
    assert w is None or (w.dtype == F32 and w.shape == (xa.shape[1],))
    mean, rstd = _stats(xa, eps, rms)
    y = _norm_apply(xa, w, mean, rstd)
    if res is not None:
        assert res.dtype == F32 and res.shape == y.shape
        y = y + res
    return y.to(out_dtype), (torch.stack([mean, rstd]) if save_stats else None)


def norm_bwd(dy, x, w, stats, dx_dtype, dw=None, dres=None, act=0, rms=0, y_fwd=None, want_dw=False, bf16_copy=False):
    assert stats is not None and stats.shape == (2, x.shape[0])
    xin = x.detach().float().requires_grad_(act != 0)
    with torch.enable_grad():
        xa = _act(xin, act)
    assert dy.shape == xa.shape
    dxa, gw = _norm_grad(dy, xa.detach(), w, stats[0], stats[1], rms)
    dx = torch.autograd.grad(xa, xin, dxa)[0] if act else dxa
    if dres is not None:
        assert dres.dtype == F32 and dres.shape == dx.shape
        dx = dx + dres
    if dw is not None:
        dw += gw
    return (dx.to(dx_dtype), gw) if want_dw else dx.to(dx_dtype)


def norm2_fwd(a, res, w1, w2, eps, rms1=0, rms2=0, save_stats=True):
    assert a.dtype == _bf() and res.dtype == F32 and a.shape == res.shape
    m1, r1 = _stats(a.float(), eps, rms1)
    x2 = res + _norm_apply(a.float(), w1, m1, r1)
    m2, r2 = _stats(x2, eps, rms2)
    h2 = _norm_apply(x2, w2, m2, r2)
    return x2, h2.to(_bf()), (torch.stack([m1, r1, m2, r2]) if save_stats else None)


def norm2_bwd(d_h2, x2, w2, dres, a, w1, stats, rms1=0, rms2=0):
    assert stats.shape == (4, a.shape[0]) and x2.dtype == F32 and dres.dtype == F32
    d2, dw2 = _norm_grad(d_h2, x2, w2, stats[2], stats[3], rms2)
    dx2 = d2 + dres
    d_a, dw1 = _norm_grad(dx2, a.float(), w1, stats[0], stats[1], rms1)
    return dx2, d_a.to(_bf()), dw1, dw2


def glu_fwd(ab):
    return _act(ab, 2).to(_bf())


def glu_bwd(ab, dout):
    x = ab.detach().float().requires_grad_(True)
    with torch.enable_grad():
        y = _act(x, 2)
    return torch.autograd.grad(y, x, dout.float())[0].to(ab.dtype)


# --------------------------------------------------------------------------------------------------------- attention
def _heads(t, B, S, nh, hd):
    assert t.shape[0] == B * S and t.shape[1] == nh * hd
    return t.float().reshape(B, S, nh, hd).permute(0, 2, 1, 3)


def _attn(q, k, v, B, nh, Sq, Skv, scale, hd):
    s = (_heads(q, B, Sq, nh, hd) @ _heads(k, B, Skv, nh, hd).transpose(-1, -2)) * scale
    o = s.softmax(-1) @ _heads(v, B, Skv, nh, hd)
    return o.permute(0, 2, 1, 3).reshape(B * Sq, nh * hd), torch.logsumexp(s, -1)


def attn_fwd(q, k, v, B, nh, Sq, Skv, scale, head_dim=64):
    o, lse = _attn(q, k, v, B, nh, Sq, Skv, scale, int(head_dim))
    return o.to(_bf()), lse


def attn_bwd(q, k, v, o, do, lse, dq, dk, dv, B, nh, Sq, Skv, scale, head_dim=64):
    assert do.shape == o.shape and dq.shape == q.shape and dk.shape == k.shape and dv.shape == v.shape
    qq, kk, vv = (t.detach().float().clone().requires_grad_(True) for t in (q, k, v))
    with torch.enable_grad():
        out, lse2 = _attn(qq, kk, vv, B, nh, Sq, Skv, scale, int(head_dim))
    assert torch.allclose(lse2.detach(), lse, atol=1e-3, rtol=1e-3)  # the host handed over this call's own log-sum-exp
    gq, gk, gv = torch.autograd.grad(out, (qq, kk, vv), do.float())
    dq.copy_(gq), dk.copy_(gk), dv.copy_(gv)


# -------------------------------------------------------------------------------------------------------------- loss
def ce_fwd(logits_padded, labels, V, label_smoothing):
    lg = logits_padded[:, :V].float()
    loss = F.cross_entropy(lg, labels, ignore_index=-100, label_smoothing=label_smoothing)
    n = (labels != -100).sum().float()
    row = F.cross_entropy(lg, labels, ignore_index=-100, label_smoothing=label_smoothing, reduction="none")
    return torch.stack([loss, n]), torch.stack([torch.logsumexp(lg, -1), row])


def ce_bwd(logits_padded, labels, ws, dloss, loss_out, V, label_smoothing, row_scale=None):
    assert row_scale is None and dloss.shape == (1,)
    x = logits_padded[:, :V].detach().float().requires_grad_(True)
    with torch.enable_grad():
        loss = F.cross_entropy(x, labels, ignore_index=-100, label_smoothing=label_smoothing)
    dl = torch.zeros(logits_padded.shape, dtype=logits_padded.dtype)
    dl[:, :V] = (torch.autograd.grad(loss, x)[0] * dloss).to(dl.dtype)
    return dl


# ---------------------------------------------------------------------------------------------------------- sampling
def sample_step(logits, input_ids, q_exp, u, K, mask_id, mask_len, temperature, logits_unc=None, guidance=0.0,
                skip_first_token=False, return_conf=False):
    """csrc/sample.cu's contract (its header comment), written with torch ops"""
    B, L = input_ids.shape
    off = 1 if skip_first_token else 0
    x = logits[:, off:, :K].float()
    if logits_unc is not None:
        xu = logits_unc[:, off:, :K].float()
        x = xu + guidance * (x - xu)
    e = torch.exp(x - x.max(-1, keepdim=True).values)
    sampled = (e / q_exp.view(B, L, K)).argmax(-1)
    unknown = input_ids == mask_id
    sampled = torch.where(unknown, sampled, input_ids)
    p_sel = e.gather(-1, sampled.clamp(max=K - 1)[..., None]).squeeze(-1) / e.sum(-1)
    p_sel = torch.where(unknown, p_sel, torch.finfo(torch.float32).max)
    gumbel = -torch.log((-torch.log(u.view(B, L).clamp(min=1e-20))).clamp(min=1e-20))
    conf = torch.log(p_sel.clamp(min=1e-20)) + temperature * gumbel
    k = torch.clamp(torch.minimum(unknown.sum(-1, keepdim=True) - 1, torch.tensor(int(mask_len))), min=1)
    cut = conf.sort(-1).values.gather(1, k)
    nxt = torch.where(conf < cut, mask_id, sampled)
    return (sampled, nxt, conf) if return_conf else (sampled, nxt)


# ------------------------------------------------------------------------------------------- U-ViT v2 (csrc/uvit*.cu)
def _mod_rows(mod, rows_per_sample, H):
    """mod: fp32 [B, 2H] view (scale | shift) of the stacked adaLN mapper output -> per-row scale, shift"""
    assert mod.dtype == F32 and mod.shape[1] == 2 * H
    return mod[:, :H].repeat_interleave(rows_per_sample, 0), mod[:, H:].repeat_interleave(rows_per_sample, 0)


def _mod_grad(dmod, dy, n, rows_per_sample, H):
    B = dmod.shape[0]
    dmod[:, :H] += (dy * n).view(B, rows_per_sample, H).sum(1)
    dmod[:, H:] += dy.view(B, rows_per_sample, H).sum(1)


def add_norm_mod(a, w, eps, rms, out_dtype=None, residual=None, mod=None, rows_per_sample=1, want_residual=True):
    r = a.float() if residual is None else a.float() + residual
    assert residual is None or residual.dtype == F32
    mean, rstd = _stats(r, eps, rms)
    y = _norm_apply(r, w, mean, rstd)
    if mod is not None:
        sc, sh = _mod_rows(mod, rows_per_sample, r.shape[1])
        y = y * (1 + sc) + sh
    return (r if want_residual else None), y.to(_bf() if out_dtype is None else out_dtype)


def add_norm_mod_bwd(dy, dr_out, x_saved, w, eps, rms, da_dtype, mod=None, rows_per_sample=1, dw=None, dmod=None,
                     want_dr=True):
    assert x_saved.dtype == F32 and dy.shape == x_saved.shape and (dr_out is None or dr_out.dtype == F32)
    x = x_saved
    mean, rstd = _stats(x, eps, rms)
    g = dy.float()
    if mod is not None:
        sc, _ = _mod_rows(mod, rows_per_sample, x.shape[1])
        _mod_grad(dmod, g, _norm_apply(x, w, mean, rstd), rows_per_sample, x.shape[1])
        g = g * (1 + sc)
    dx, gw = _norm_grad(g, x, w, mean, rstd, rms)
    if dw is not None:
        dw += gw
    tot = dx if dr_out is None else dx + dr_out
    return tot.to(da_dtype), (tot if want_dr else None)


def _dwconv_norm(x, wk, norm_w, B, hh, ww, eps, rms):
    C = x.shape[1]
    img = x.float().view(B, hh, ww, C).permute(0, 3, 1, 2)
    conv = F.conv2d(img, wk.t().reshape(C, 1, 3, 3), padding=1, groups=C).permute(0, 2, 3, 1).reshape(B * hh * ww, C)
    mean, rstd = _stats(conv, eps, rms)
    return conv, _norm_apply(conv, norm_w, mean, rstd)


def dwconv3x3_norm(x, wk, norm_w, B, hh, ww, eps, rms, save_conv=False):
    assert x.dtype == F32 and wk.shape == (9, x.shape[1])
    conv, y = _dwconv_norm(x, wk, norm_w, B, hh, ww, eps, rms)
    return (y.to(_bf()), conv.to(_bf())) if save_conv else y.to(_bf())


def dwconv3x3_norm_bwd(dy, conv, x, wk, norm_w, dres, dwk, dnw, B, hh, ww, eps, rms):
    xx, kk = x.detach().clone().requires_grad_(True), wk.detach().clone().requires_grad_(True)
    nn_ = None if norm_w is None else norm_w.detach().clone().requires_grad_(True)
    with torch.enable_grad():
        _, y = _dwconv_norm(xx, kk, nn_, B, hh, ww, eps, rms)
    gs = torch.autograd.grad(y, [xx, kk] + ([] if nn_ is None else [nn_]), dy.float())
    dwk += gs[1]
    if nn_ is not None:
        dnw += gs[2]
    return gs[0] + dres


def _grn(x, gamma, beta, B, HW):
    g = F.gelu(x.float()).view(B, HW, -1)
    sumsq = g.pow(2).sum(1)
    nx = sumsq.sqrt() / (sumsq.sqrt().mean(-1, keepdim=True) + 1e-6)
    out = gamma.float() * (g * nx[:, None]) + beta.float() + g
    return out.reshape(B * HW, -1), sumsq, nx


def grn(x, gamma, beta, B, HW, save_stats=False):
    out, sumsq, nx = _grn(x, gamma, beta, B, HW)
    return (out.to(x.dtype), torch.stack([sumsq, nx])) if save_stats else out.to(x.dtype)


def grn_bwd(x, dout, stats, gamma, dgamma, dbeta, B, HW):
    xx = x.detach().float().requires_grad_(True)
    gg, bb = gamma.detach().clone().requires_grad_(True), torch.zeros_like(gamma).requires_grad_(True)  # d out / d beta = 1
    with torch.enable_grad():
        out, _, nx = _grn(xx, gg, bb, B, HW)
    assert torch.allclose(nx.detach(), stats[1], rtol=2e-2, atol=1e-3)  # the host handed over this block's statistics
    gx, g_g, g_b = torch.autograd.grad(out, (xx, gg, bb), dout.float())
    dgamma += g_g
    dbeta += g_b
    return gx.to(x.dtype)


def adaln_apply(x, mod, B, rows_per_sample):
    sc, sh = _mod_rows(mod, rows_per_sample, x.shape[1])
    return x * (1 + sc) + sh


def adaln_apply_(x, mod, B, rows_per_sample):
    x.copy_(adaln_apply(x, mod, B, rows_per_sample))
    return x


def adaln_bwd(dy, x, mod, dmod, B, rows_per_sample):
    assert dy.dtype == F32 and x.dtype == F32
    sc, _ = _mod_rows(mod, rows_per_sample, x.shape[1])
    _mod_grad(dmod, dy, x, rows_per_sample, x.shape[1])
    return dy * (1 + sc)


def silu_bf16(x):
    return F.silu(x.float()).to(_bf())


def silu_bwd(dy, x, out=None, out_dtype=None):
    xf = x.float()
    sg = torch.sigmoid(xf)
    d = dy.float() * (sg * (1 + xf * (1 - sg)))
    if out is not None:
        out += d.to(out.dtype)
        return out
    return d.to(out_dtype or x.dtype)


def linear_wgrad(dy, x, dw):
    assert dw.dtype == F32 and dw.shape == (dy.shape[1], x.shape[1]) and dy.dtype == _bf() and x.dtype == _bf()
    dw += dy.float().t() @ x.float()
    return dw


def linear_dgrad_acc(dy, w, acc):
    assert acc.dtype == F32 and acc.shape == (dy.shape[0], w.shape[1])
    acc += dy.float() @ w.float()
    return acc


def embed_bwd(ids, dx, dword, dpos):
    B, S = ids.shape
    dword.index_add_(0, ids.reshape(-1), dx)
    if dpos is not None:
        dpos[:S] = dx.view(B, S, -1).sum(0)


def ce_bwd_rows(logits_padded, labels, ws, dloss, loss_out, V, label_smoothing, row_scale=None):
    """ce_bwd with the optional per-row weights of the loss_weight path (loss = sum_r row_scale_r * loss_r)"""
    if row_scale is None:
        return ce_bwd(logits_padded, labels, ws, dloss, loss_out, V, label_smoothing)
    x = logits_padded[:, :V].detach().float().requires_grad_(True)
    with torch.enable_grad():
        rows = F.cross_entropy(x, labels, ignore_index=-100, label_smoothing=label_smoothing, reduction="none")
        loss = (rows * row_scale).sum()
    dl = torch.zeros(logits_padded.shape, dtype=logits_padded.dtype)
    dl[:, :V] = (torch.autograd.grad(loss, x)[0] * dloss).to(dl.dtype)
    return dl


V2_STAND_INS = dict(
    add_norm_mod=add_norm_mod, add_norm_mod_bwd=add_norm_mod_bwd, dwconv3x3_norm=dwconv3x3_norm,
    dwconv3x3_norm_bwd=dwconv3x3_norm_bwd, grn=grn, grn_bwd=grn_bwd, adaln_apply=adaln_apply, adaln_apply_=adaln_apply_,
    adaln_bwd=adaln_bwd, silu_bf16=silu_bf16, silu_bwd=silu_bwd, linear_wgrad=linear_wgrad, linear_dgrad_acc=linear_dgrad_acc,
    embed_bwd=embed_bwd, ce_bwd=ce_bwd_rows)


# --------------------------------------------------------------------------------- VQGAN ops (csrc/conv*.cu, vq.cu)
def _nchw(x):
    return x.permute(0, 3, 1, 2)


def _gn_silu(x_nhwc, gamma, beta, groups, eps, silu=1):
    y = F.group_norm(_nchw(x_nhwc.float()), int(groups), gamma.float(), beta.float(), float(eps))
    return (F.silu(y) if silu else y).permute(0, 2, 3, 1)


def conv2d(x, w, bias=None, residual=None, upsample2x=False, gn=None):
    """Conv2dSame (odd kernels, stride 1) on fp32 NHWC, optional GroupNorm+SiLU prologue, nearest x2 upsample first, fp32
    residual added to the output"""
    assert x.dtype == F32 and x.dim() == 4 and w.shape[1] == x.shape[3] and w.shape[2] % 2 == 1
    if gn is not None:
        x = _gn_silu(x, *gn)
    t = _nchw(x)
    if upsample2x:
        t = F.interpolate(t, scale_factor=2.0, mode="nearest")
    y = F.conv2d(t, w.float(), None if bias is None else bias.float(), padding=w.shape[2] // 2).permute(0, 2, 3, 1)
    if residual is not None:
        assert residual.shape == y.shape and residual.dtype == F32
        y = y + residual
    return y.contiguous()


def groupnorm_silu(x, gamma, beta, groups, eps, silu=1):
    return _gn_silu(x, gamma, beta, groups, eps, silu).contiguous()


def conv2d_down(x, w, bias=None):
    t = F.pad(_nchw(x), (0, 1, 0, 1))
    return F.conv2d(t, w.float(), None if bias is None else bias.float(), stride=2).permute(0, 2, 3, 1).contiguous()


def attention_single_head(q, k, v, B, hh, ww):
    C = q.shape[1]
    qq, kk, vv = (t.float().view(B, hh * ww, C) for t in (q, k, v))
    p = torch.softmax(qq @ kk.transpose(1, 2) * (float(C) ** -0.5), dim=-1)
    return (p @ vv).reshape(B * hh * ww, C)


def avg_pool2x2(x):
    return F.avg_pool2d(_nchw(x), 2).permute(0, 2, 3, 1).contiguous()


def to_nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def to_nchw(x):
    return x.permute(0, 3, 1, 2).contiguous()


def image_to_uint8(x):
    t = (torch.clamp(2.0 * x - 1.0, -1.0, 1.0) + 1.0) / 2.0
    return (255.0 * t).to(torch.uint8)  # truncation (pipeline_muse.py:245-252)


def _vq_dist(z, cb):
    """muse/modeling_maskgit_vqgan.py:303-312: |z|^2 + |e|^2 - 2 z e^T"""
    z, cb = z.float(), cb.float()
    return z.pow(2).sum(1, keepdim=True) + cb.pow(2).sum(1)[None] - 2.0 * z @ cb.t()


def vq_argmin(z_flat, codebook, return_dmin=False):
    d = _vq_dist(z_flat, codebook)
    ids = d.argmin(1)
    return (ids, d.min(1).values) if return_dmin else ids


def vq_soft_code(z_flat, codebook, temp=1.0, expo_noise=None):
    soft = torch.softmax(-_vq_dist(z_flat, codebook) / temp, dim=-1)
    ids = soft.argmax(1) if expo_noise is None else (soft / expo_noise).argmax(1)
    return soft, ids


def vq_lookup_nchw(ids, codebook):
    return codebook.float()[ids].permute(0, 2, 1).contiguous()  # [B, P, D] -> [B, D, P]


VQGAN_STAND_INS = dict(
    conv2d=conv2d, groupnorm_silu=groupnorm_silu, conv2d_down=conv2d_down, attention_single_head=attention_single_head,
    avg_pool2x2=avg_pool2x2, to_nhwc=to_nhwc, to_nchw=to_nchw, image_to_uint8=image_to_uint8, vq_argmin=vq_argmin,
    vq_soft_code=vq_soft_code, vq_lookup_nchw=vq_lookup_nchw)


STAND_INS = dict(
    linear_fwd=linear_fwd, linear_dgrad=linear_dgrad, linear_wgrad_det=linear_wgrad_det, gemm=gemm, pack_bf16=pack_bf16,
    cast_bf16=cast_bf16, take_bf16_copy=take_bf16_copy, embed_fwd=embed_fwd, embed_bwd_det=embed_bwd_det, norm_fwd=norm_fwd,
    norm_bwd=norm_bwd, norm2_fwd=norm2_fwd, norm2_bwd=norm2_bwd, glu_fwd=glu_fwd, glu_bwd=glu_bwd, attn_fwd=attn_fwd,
    attn_bwd=attn_bwd, ce_fwd=ce_fwd, ce_bwd=ce_bwd, sample_step=sample_step)


# ------------------------------------------------------------------------------------------ fused optimizer (optim.cu)
def _view(ptr, numel, ctype, dtype):
    return torch.frombuffer((ctype * numel).from_address(ptr), dtype=dtype)


def adamw_ema_step(entries_host, n_entries, scal_ptr, step_ptr, lr_dev_ptr, lr_host, beta1, beta2, eps, weight_decay,
                   ema_enabled, ema_decay, ema_min_decay, ema_update_after_step, ema_update_every, ema_use_warmup,
                   ema_inv_gamma, ema_power, stream):
    """csrc/optim.cu restated: the HOST table of {p, g, m, v, ema, packed, numel, -} pointer rows, the device-resident step
    counter, the per-step scalars (bias corrections in double, EMA decay schedule of muse/modeling_ema.py:89-106), then ONE
    pass: decoupled weight decay, Adam moments, update, EMA of the updated weight, bf16 copy into the packed operand."""
    step = _view(step_ptr, 1, ctypes.c_int64, torch.int64)
    s = int(step[0]) + 1
    step[0] = s
    inv_bc1 = float(torch.tensor(1.0 / (1.0 - beta1 ** s), dtype=F32))
    inv_sqrt_bc2 = float(torch.tensor(1.0 / (1.0 - beta2 ** s) ** 0.5, dtype=F32))
    lr = float(_view(lr_dev_ptr, 1, ctypes.c_float, F32)[0]) if lr_dev_ptr else lr_host
    omd = None
    if ema_enabled:
        decay, st = 0.0, max(0, s - ema_update_after_step - 1)
        if st > 0:
            value = 1.0 - (1.0 + st / ema_inv_gamma) ** (-ema_power) if ema_use_warmup else (1.0 + st) / (10.0 + st)
            decay = max(min(value, ema_decay), ema_min_decay)
        if (s - 1) % max(1, ema_update_every) == 0:
            omd = float(torch.tensor(1.0 - decay, dtype=F32))
    table = torch.frombuffer((ctypes.c_int64 * (8 * n_entries)).from_address(entries_host), dtype=torch.int64).view(-1, 8)
    two_byte = torch.bfloat16 != torch.float32
    for p_, g_, m_, v_, e_, k_, numel, _ in table.tolist():
        assert numel > 0 and numel % 4 == 0
        p, g, m, v = (_view(x, numel, ctypes.c_float, F32) for x in (p_, g_, m_, v_))
        p -= lr * weight_decay * p
        m += (1.0 - beta1) * (g - m)
        v.mul_(beta2).add_((1.0 - beta2) * g * g)
        p -= (lr * inv_bc1) * m / (v.sqrt() * inv_sqrt_bc2 + eps)
        if e_ and omd is not None:
            e = _view(e_, numel, ctypes.c_float, F32)
            e -= omd * (e - p)
        if k_:
            dst = _view(k_, numel, ctypes.c_uint16, torch.bfloat16) if two_byte else _view(k_, numel, ctypes.c_float, F32)
            dst.copy_(p)


def install_optimizer(mp):
    """route ops._call("muse_adamw_ema_step", ...) to the restatement (FusedAdamW calls the C ABI through ops._call)"""
    from open_muse_b200 import ops

    def call(name, *args):
        if name != "muse_adamw_ema_step":
            raise AssertionError(f"unexpected library call on the CPU: {name}")
        adamw_ema_step(*args)

    mp.setattr(ops, "_call", call)
    mp.setattr(ops, "_prep", lambda t: 0)


class PlainSetter:
    """stands in for pytest's monkeypatch in a spawned worker process (nothing to restore: the process ends)"""

    @staticmethod
    def setattr(obj, name, value, raising=True):
        setattr(obj, name, value)


def install(mp, exact=True):
    """monkeypatch ``open_muse_b200.ops`` with the stand-ins (restored by pytest's monkeypatch at the end of the test)"""
    from open_muse_b200 import ops, uvit_v2_train

    if exact:
        mp.setattr(torch, "bfloat16", torch.float32)
        # module-level dtype constants / default arguments bound at import time
        mp.setattr(uvit_v2_train, "BF16", torch.float32)
        mp.setattr(uvit_v2_train._lin_bwd, "__defaults__", (torch.float32, True))
    for name, fn in {**STAND_INS, **V2_STAND_INS, **VQGAN_STAND_INS}.items():
        mp.setattr(ops, name, fn)
    mp.setattr(torch.Tensor, "is_cuda", property(lambda self: True))  # the model refuses CPU tensors (no fallback)
