"""``MaskGitTransformer`` with the reference's Python surface and a hand-written sm_90a hot path.

Boundary (reference: muse/modeling_transformer.py:1083-1456): same constructor arguments, ``config``
keys, parameter names / shapes / construction order (so ``torch.manual_seed(s); Model(**cfg)`` gives
the reference's initial weights and ``pytorch_model.bin`` files are interchangeable), same
``forward`` / ``generate2`` signatures and return values.

Underneath, nothing is torch-eager: the module tree only *holds* the fp32 master parameters.
``forward`` runs three kinds of ``torch.autograd.Function`` -- embedding, one per transformer layer
(so DDP's gradient buckets fire layer by layer during backward), and head+loss -- whose bodies are
sequences of libmuse_b200 kernels (wgmma GEMMs, fused attention, fused norm/GELU/residual, masked
cross-entropy).  Compute precision is the reference's bf16-autocast recipe: bf16 GEMM operands with
fp32 accumulation, fp32 residual stream, fp32 norm / softmax / loss statistics.
"""
from __future__ import annotations

import math
from typing import Optional

import torch
from torch import nn

from . import ops
from .modeling_utils import ConfigMixin, ModelMixin, register_to_config
from .sampling import cosine_schedule, mask_by_random_topk

import os as _os

_CHECK_IDS = _os.environ.get("MUSE_B200_CHECK_IDS", "0") == "1"


# --------------------------------------------------------------------------------------------
# Parameter containers (names/shapes/order == reference modules; they carry no compute)
# --------------------------------------------------------------------------------------------
class LayerNorm(nn.Module):
    """Weight-only LayerNorm parameters (reference :124-137)."""

    def __init__(self, dim, eps=1e-5, use_bias=False, elementwise_affine=True):
        super().__init__()
        self.dim, self.eps = dim, eps
        self.weight = nn.Parameter(torch.ones(dim)) if elementwise_affine else None
        self.bias = nn.Parameter(torch.zeros(dim)) if (elementwise_affine and use_bias) else None


class RMSNorm(nn.Module):
    """RMSNorm parameters (reference :79-100)."""

    def __init__(self, normalized_shape, eps=1e-6, elementwise_affine=True):
        super().__init__()
        self.elementwise_affine = elementwise_affine
        if elementwise_affine:
            self.weight = nn.Parameter(torch.ones(normalized_shape))
        self.variance_epsilon = eps


def _norm(norm_type, dim, eps, use_bias=False):
    return LayerNorm(dim, eps=eps, use_bias=use_bias) if norm_type == "layernorm" else RMSNorm(dim, eps=eps)


class Attention(nn.Module):
    def __init__(self, hidden_size, num_heads, encoder_hidden_size=None, attention_dropout=0.0, use_bias=False):
        super().__init__()
        self.hidden_size, self.num_heads = hidden_size, num_heads
        self.head_dim = hidden_size // num_heads
        self.attention_dropout = attention_dropout
        if self.head_dim * num_heads != hidden_size:
            raise ValueError(
                f"embed_dim must be divisible by num_heads (got `embed_dim`: {hidden_size} and `num_heads`: {num_heads})."
            )
        kv_in = hidden_size if encoder_hidden_size is None else encoder_hidden_size
        self.query = nn.Linear(hidden_size, hidden_size, bias=use_bias)
        self.key = nn.Linear(kv_in, hidden_size, bias=use_bias)
        self.value = nn.Linear(kv_in, hidden_size, bias=use_bias)
        self.out = nn.Linear(hidden_size, hidden_size, bias=use_bias)
        self.dropout = nn.Dropout(attention_dropout)


class FeedForward(nn.Module):
    def __init__(self, hidden_size, intermediate_size, hidden_dropout, norm_type, eps, use_normformer, use_bias):
        super().__init__()
        self.use_normformer = use_normformer
        self.pre_mlp_layer_norm = LayerNorm(hidden_size, eps=eps, use_bias=use_bias)  # always LayerNorm (:767)
        self.wi_0 = nn.Linear(hidden_size, intermediate_size, bias=use_bias)
        self.wi_1 = nn.Linear(hidden_size, intermediate_size, bias=use_bias)
        if use_normformer:
            self.mid_mlp_layer_norm = _norm(norm_type, intermediate_size, eps, use_bias)
        self.wo = nn.Linear(intermediate_size, hidden_size, bias=use_bias)
        self.dropout = nn.Dropout(hidden_dropout)


class TransformerLayer(nn.Module):
    def __init__(self, hidden_size, intermediate_size, num_attention_heads, encoder_hidden_size, add_cross_attention,
                 hidden_dropout, attention_dropout, norm_type, eps, use_normformer, use_bias):
        super().__init__()
        self.use_normformer = use_normformer
        self.attn_layer_norm = _norm(norm_type, hidden_size, eps, use_bias)
        self.attention = Attention(hidden_size, num_attention_heads, attention_dropout=attention_dropout, use_bias=use_bias)
        if use_normformer:
            self.post_attn_layer_norm = _norm(norm_type, hidden_size, eps, use_bias)
        self.ffn = FeedForward(hidden_size, intermediate_size, hidden_dropout, norm_type, eps, use_normformer, use_bias)
        if add_cross_attention:
            self.crossattn_layer_norm = _norm(norm_type, hidden_size, eps, use_bias)
            self.crossattention = Attention(hidden_size, num_attention_heads, encoder_hidden_size, attention_dropout, use_bias)
            if use_normformer:
                self.post_crossattn_layer_norm = _norm(norm_type, hidden_size, eps, use_bias)


class Embed(nn.Module):
    def __init__(self, vocab_size, embedding_size, hidden_dropout, max_position_embeddings):
        super().__init__()
        self.word_embeddings = nn.Embedding(vocab_size, embedding_size)
        self.position_embeddings = nn.Embedding(max_position_embeddings, embedding_size)
        self.dropout = nn.Dropout(hidden_dropout)


class MlmLayer(nn.Module):
    def __init__(self, hidden_size, vocab_size, norm_type, eps, use_mlm_layernorm, use_bias):
        super().__init__()
        self.use_mlm_layernorm = use_mlm_layernorm
        self.mlm_dense = nn.Linear(hidden_size, hidden_size, bias=use_bias)
        if use_mlm_layernorm:
            self.mlm_ln = _norm(norm_type, hidden_size, eps, use_bias)
        self.to_logits = nn.Linear(hidden_size, vocab_size, bias=use_bias)


class Norm2D(nn.Module):
    """Per-pixel channel norm container (reference :302-311): parameter name ``norm.weight``."""

    def __init__(self, dim, eps=1e-5, use_bias=False, norm_type="layernorm"):
        super().__init__()
        self.norm = _norm(norm_type, dim, eps, use_bias)


class ConvEmbed(nn.Module):
    """``use_conv_in_out`` input side (reference :988-1041): token embedding -> norm -> PixelUnshuffle(patch) -> 1x1 conv
    -> + position embedding.  ``max_position_embeddings`` is the class default 256 whatever the model config says (the
    reference does not forward it, :1133-1141)."""

    def __init__(self, vocab_size, embedding_size, hidden_size, patch_size=2, max_position_embeddings=256,
                 norm_type="layernorm", layer_norm_eps=1e-5, use_bias=False):
        super().__init__()
        self.hidden_size, self.patch_size, self.max_position_embeddings = hidden_size, patch_size, max_position_embeddings
        self.embeddings = nn.Embedding(vocab_size, embedding_size)
        self.layer_norm = _norm(norm_type, embedding_size, layer_norm_eps, use_bias)
        self.conv = nn.Conv2d(embedding_size * (patch_size ** 2), hidden_size, kernel_size=1, bias=use_bias)
        self.position_embeddings = nn.Embedding(max_position_embeddings, hidden_size)


class ConvMlmLayer(nn.Module):
    """``use_conv_in_out`` output side (reference :1043-1080): 1x1 conv -> PixelShuffle(patch) -> Norm2D -> 1x1 conv."""

    def __init__(self, vocab_size, embedding_size, hidden_size, patch_size=2, norm_type="layernorm", layer_norm_eps=1e-5,
                 use_bias=False):
        super().__init__()
        self.vocab_size, self.patch_size = vocab_size, patch_size
        self.conv1 = nn.Conv2d(hidden_size, embedding_size * (patch_size ** 2), kernel_size=1, bias=use_bias)
        self.layer_norm = Norm2D(embedding_size, eps=layer_norm_eps, use_bias=use_bias, norm_type=norm_type)
        self.conv2 = nn.Conv2d(embedding_size, vocab_size, kernel_size=1, bias=use_bias)


# --------------------------------------------------------------------------------------------
# bf16 operand cache: every Linear weight packed (fused per GEMM) in ONE kernel launch per update
# --------------------------------------------------------------------------------------------
class _PackedWeights:
    """Fused bf16 copies of the Linear weights: [q;k;v] -> [3H,H], [wi_0;wi_1] -> [2I,H], padded
    to_logits -> [Vpad,H] ...  Re-packed (one ``muse_pack_bf16`` launch) whenever a parameter's
    version counter or storage changes, i.e. once per optimizer step and never during ``generate2``.

    In FP8 GEMM precision (``MaskGitTransformer.set_gemm_precision``) the layer entries of the FP8 sites (``FP8_SITES``)
    are ``ops.F8`` copies: the per-output-row e4m3 quantization of the bf16 copies, which stay, as the fused optimizers'
    destinations (``quantized``: (bf16 copy, F8 copy) while in FP8 precision).  The buffers depend on the parameters'
    storage only, never on the precision: the bf16 copies are allocated once per storage layout, the F8 copies the first
    time FP8 precision runs on that layout, and both keep their addresses across precision switches (the F8 copies then
    stay allocated in bf16 precision too).  Every refresh re-packs and, in FP8 precision, re-quantizes in place, so a
    captured ``generate2`` graph of either precision stays valid.  A new layout drops the model's captured graphs."""

    FP8_SITES = ("qkv", "cq", "wi", "wo")

    def __init__(self, model: "MaskGitTransformer"):
        self.model = model
        self.key = None
        self.layers = []
        self.head = {}
        self.quantized = []
        self.buffers_key = None
        self.bf16_layers, self.fp8_layers, self.f8_pairs = [], None, []

    def _plan(self):
        m = self.model
        groups = []  # (name, [params], rows_padded)
        for i, layer in enumerate(m.transformer_layers):
            a, f = layer.attention, layer.ffn
            groups.append((i, "qkv", [a.query.weight, a.key.weight, a.value.weight], None))
            groups.append((i, "ao", [a.out.weight], None))
            groups.append((i, "wi", [f.wi_0.weight, f.wi_1.weight], None))
            groups.append((i, "wo", [f.wo.weight], None))
            if m.config.add_cross_attention:
                c = layer.crossattention
                groups.append((i, "cq", [c.query.weight], None))
                groups.append((i, "ckv", [c.key.weight, c.value.weight], None))
                groups.append((i, "co", [c.out.weight], None))
        if m.config.add_cross_attention and m.config.project_encoder_hidden_states:
            groups.append((-1, "eproj", [m.encoder_proj.weight], None))
        if m.config.use_conv_in_out:  # 1x1 convolutions are GEMMs over the channel dimension: [out, in, 1, 1] packs as [out, in]
            groups.append((-1, "cin", [m.embed.conv.weight], None))
        if m.config.use_mlm_layer and m.config.use_conv_in_out:
            groups.append((-1, "c1", [m.mlm_layer.conv1.weight], None))
            groups.append((-1, "logits", [m.mlm_layer.conv2.weight], m.padded_output_size))
        elif m.config.use_mlm_layer:
            groups.append((-1, "dense", [m.mlm_layer.mlm_dense.weight], None))
            groups.append((-1, "logits", [m.mlm_layer.to_logits.weight], m.padded_output_size))
        else:
            groups.append((-1, "logits", [m.to_logits.weight], m.padded_output_size))
        return groups

    def _key(self, groups):
        return (self.model._gemm_precision,) + tuple((p.data_ptr(), p._version, p.dtype) for _, _, ps, _ in groups for p in ps)

    def _quantize(self):
        for src, dst in self.quantized:
            ops.quantize_rows_e4m3(src, out=dst)

    def sync(self):
        """after a fused optimizer step that wrote every packed copy through ``dst_of``: the cache is current once the F8
        copies are re-quantized from the new bf16 copies, so its key follows the parameters' new version counters (no
        re-pack on the next forward)"""
        if self.key is not None:
            self._quantize()
            self.key = self._key(self._plan())

    def refresh(self):
        m = self.model
        groups = self._plan()
        params = [p for _, _, ps, _ in groups for p in ps]
        key = self._key(groups)
        if key == self.key:
            return self
        dev = params[0].device
        fp8 = self.model._gemm_precision == "fp8"
        buffers_key = tuple(p.data_ptr() for p in params)
        if self.buffers_key != buffers_key:
            total = 0
            offs = []
            for _, _, ps, rows_pad in groups:
                cols = ps[0].shape[1]
                rows = sum(p.shape[0] for p in ps)
                rows_alloc = rows_pad if rows_pad is not None else rows
                offs.append((total, rows_alloc, cols))
                total += ((rows_alloc * cols + 127) // 128) * 128  # keep every group 256B aligned
            self.flat = torch.zeros(total, dtype=torch.bfloat16, device=dev)
            self.bf16_layers = [dict() for _ in m.transformer_layers]
            self.fp8_layers, self.f8_pairs = None, []
            self.head = {}
            entries = []
            block = 0
            self.slow = []  # non-fp32 parameters are copied by torch (inference-only convenience)
            for (li, name, ps, _), (off, rows_alloc, cols) in zip(groups, offs):
                view = self.flat[off: off + rows_alloc * cols].view(rows_alloc, cols)
                (self.head if li < 0 else self.bf16_layers[li])[name] = view
                r = 0
                for p in ps:
                    dst = view[r: r + p.shape[0]]
                    if p.dtype == torch.float32 and p.numel() % 4 == 0:
                        entries.append((p.data_ptr(), dst.data_ptr(), p.numel(), block))
                        block += (p.numel() + 1023) // 1024
                    else:
                        self.slow.append((p, dst))
                    r += p.shape[0]
            self.n_entries, self.n_blocks = len(entries), block
            self.dst_of = {e[0]: e[1] for e in entries}  # parameter pointer -> bf16 copy (used by the fused optimizers)
            self.table = torch.tensor(entries, dtype=torch.int64).to(dev) if entries else None
            self.buffers_key = buffers_key
            m.__dict__.pop("_gen_graphs", None)  # graphs captured on the old buffers must never replay
        if fp8 and self.fp8_layers is None:
            self.fp8_layers = [dict(d) for d in self.bf16_layers]
            for d in self.fp8_layers:
                for name in self.FP8_SITES:
                    if name in d:
                        src = d[name]
                        d[name] = ops.F8(torch.empty(src.shape, dtype=ops.FP8, device=dev),
                                         torch.empty(src.shape[0], dtype=torch.float32, device=dev))
                        self.f8_pairs.append((src, d[name]))
        self.layers = self.fp8_layers if fp8 else self.bf16_layers
        self.quantized = self.f8_pairs if fp8 else []
        self.layout_key = (self.model._gemm_precision,) + buffers_key
        if self.table is not None:
            ops.pack_bf16(self.table, self.n_entries, self.n_blocks)
        for p, dst in self.slow:
            dst.copy_(p.detach())
        self._quantize()
        self.key = key
        return self


# --------------------------------------------------------------------------------------------
# autograd Functions (bodies are libmuse_b200 kernel sequences)
# --------------------------------------------------------------------------------------------
def _f32(p):
    return p if p.dtype == torch.float32 else p.float()


class _EmbedFn(torch.autograd.Function):
    """word[ids] + pos (reference Embed.forward :942-957); drop = (p, seed, site) applies its dropout (:956)."""

    @staticmethod
    def forward(ctx, ids, word, pos, drop=None):
        ctx.save_for_backward(ids)
        ctx.shapes = (word.shape, pos.shape)
        x = ops.embed_fwd(ids, _f32(word), _f32(pos))
        ctx.drop = None
        if drop is not None:
            x, bits = ops.dropout_fwd(x, *drop)
            ctx.drop = (drop[0], bits)
        return x

    @staticmethod
    def backward(ctx, dx):
        (ids,) = ctx.saved_tensors
        wshape, pshape = ctx.shapes
        dx = dx.contiguous()
        if ctx.drop is not None:
            dx = ops.dropout_bwd(dx, ctx.drop[1], ctx.drop[0])
        dword, dpos = ops.embed_bwd_det(ids, dx, wshape[0], pshape[0])
        return None, dword, dpos, None


class _ConvSpec:
    """Static description of the ``use_conv_in_out`` embedding / head (reference :988-1080): ``n`` x ``n`` tokens outside the
    transformer, ``n / p`` x ``n / p`` inside."""

    def __init__(self, B, n, p, E, H, eps, rms, w, V=0, Vpad=0, use_enc_ln=True, label_smoothing=0.0, n_cols=None):
        self.B, self.n, self.p, self.E, self.H, self.eps, self.rms, self.w = B, n, p, E, H, eps, rms, w
        self.V, self.Vpad, self.use_enc_ln, self.ls, self.n_cols = V, Vpad, use_enc_ln, label_smoothing, n_cols
        self.train = torch.is_grad_enabled()


def _to_patches(t, B, n, p, C):
    """tokens [B*n*n, C] -> [B*(n/p)^2, C*p*p] with the channel order of nn.PixelUnshuffle (c, dy, dx), i.e. the input
    channel order of the reference's 1x1 convolution weight"""
    m = n // p
    return t.view(B, m, p, m, p, C).permute(0, 1, 3, 5, 2, 4).reshape(B * m * m, C * p * p)


def _from_patches(t, B, n, p, C):
    """inverse of _to_patches = nn.PixelShuffle on the token-major layout: [B*(n/p)^2, C*p*p] -> tokens [B*n*n, C]"""
    m = n // p
    return t.view(B, m, m, C, p, p).permute(0, 1, 4, 2, 5, 3).reshape(B * n * n, C)


class _ConvEmbedFn(torch.autograd.Function):
    """ConvEmbed.forward (reference :1023-1041): gather -> norm -> PixelUnshuffle -> 1x1 conv as ONE GEMM over
    ``[B*S/p^2, (c, dy, dx)]`` patches whose fp32 residual epilogue adds the position rows."""

    @staticmethod
    def forward(ctx, ids, spec, w_word, w_ln, w_conv, w_pos):
        s = spec
        grad = s.train and any(ctx.needs_input_grad)
        B, n, p, E = s.B, s.n, s.p, s.E
        e = ops.embed_fwd(ids, _f32(w_word), None)
        y, st = ops.norm_fwd(e, _f32(w_ln), s.eps, torch.bfloat16, rms=s.rms, save_stats=grad)
        a = _to_patches(y, B, n, p, E)
        pos_ids = torch.arange((n // p) ** 2, device=ids.device, dtype=torch.int64).repeat(B, 1)
        pos_rows = ops.embed_fwd(pos_ids, _f32(w_pos), None)
        x = ops.linear_fwd(a, s.w["cin"], res=pos_rows)
        if grad:
            ctx.sv = (ids, pos_ids, e, st, a, w_ln)
            ctx.spec, ctx.shapes = s, (w_word.shape, w_conv.shape, w_pos.shape)
        return x

    @staticmethod
    def backward(ctx, dx):
        s = ctx.spec
        ids, pos_ids, e, st, a, w_ln = ctx.sv
        wshape, cshape, pshape = ctx.shapes
        dx = dx.contiguous()
        dxb = ops.take_bf16_copy(dx)
        if dxb is None:
            dxb = ops.cast_bf16(dx)
        d_a = ops.linear_dgrad(dxb, s.w["cin"])
        g_conv = ops.linear_wgrad_det(dxb, a).view(cshape)
        d_y = _from_patches(d_a, s.B, s.n, s.p, s.E)
        d_e, g_ln = ops.norm_bwd(d_y, e, _f32(w_ln), st, torch.float32, rms=s.rms, want_dw=True)
        g_word, _ = ops.embed_bwd_det(ids, d_e, wshape[0], 0)
        g_pos, _ = ops.embed_bwd_det(pos_ids, dx, pshape[0], 0)  # rows beyond the used positions are stored as zeros
        ctx.sv = None
        return None, None, g_word, g_ln, g_conv, g_pos


class _ConvHeadFn(torch.autograd.Function):
    """encoder_layer_norm -> ConvMlmLayer (1x1 conv, PixelShuffle, Norm2D, 1x1 conv; reference :1070-1080) -> masked CE."""

    @staticmethod
    def forward(ctx, x, labels, spec, *params):
        s = spec
        grad = s.train and any(ctx.needs_input_grad)
        it = iter(params)
        w_enc = next(it) if s.use_enc_ln else None
        w_c1, w_ln, w_c2 = next(it), next(it), next(it)
        B, n, p, E = s.B, s.n, s.p, s.E
        T = B * n * n
        if s.use_enc_ln:
            hN, st0 = ops.norm_fwd(x, _f32(w_enc), s.eps, torch.bfloat16, rms=s.rms, save_stats=grad)
        else:
            hN, st0 = ops.cast_bf16(x), None
        c1 = ops.linear_fwd(hN, s.w["c1"])
        t = _from_patches(c1, B, n, p, E)
        e, st1 = ops.norm_fwd(t, _f32(w_ln), s.eps, torch.bfloat16, rms=s.rms, save_stats=grad)
        if s.n_cols is not None:
            if grad or labels is not None:
                raise RuntimeError("column-restricted logits are an inference-only path")
            ncol = ((s.n_cols + 7) // 8) * 8
            logits = torch.empty(T, ncol, dtype=torch.bfloat16, device=x.device)
            ops.gemm(e, s.w["logits"], logits, T, ncol, E, E, E, ncol)
            return logits[:, : s.n_cols]
        logits = torch.empty(T, s.Vpad, dtype=torch.bfloat16, device=x.device)
        ops.gemm(e, s.w["logits"], logits, T, s.Vpad, E, E, E, s.Vpad)
        loss = None
        sv = {}
        ctx.set_materialize_grads(False)
        if labels is not None:
            loss_out, ws = ops.ce_fwd(logits, labels, s.V, s.ls)
            loss = loss_out[0]
            sv.update(loss_out=loss_out, ws=ws, labels=labels)
        if grad:
            sv.update(x=x, hN=hN, st0=st0, t=t, e=e, st1=st1, logits=logits, w_enc=w_enc, w_ln=w_ln)
            ctx.sv, ctx.spec, ctx.shapes = sv, s, (w_c1.shape, w_c2.shape)
        out_logits = logits[:, : s.V]
        if loss is None:
            return out_logits
        return out_logits, loss

    @staticmethod
    def backward(ctx, d_logits, d_loss=None):
        s, sv = ctx.spec, ctx.sv
        B, n, p, E = s.B, s.n, s.p, s.E
        dev = sv["x"].device
        dl = None
        if d_loss is not None and "labels" in sv:
            dl = ops.ce_bwd(sv["logits"], sv["labels"], sv["ws"], d_loss.to(torch.float32).reshape(1).contiguous(),
                            sv["loss_out"], s.V, s.ls)
        if d_logits is not None:  # gradient arriving through the returned logits (soft-target losses)
            extra = torch.zeros(B * n * n, s.Vpad, dtype=torch.bfloat16, device=dev)
            extra[:, : s.V] = d_logits.to(torch.bfloat16)
            dl = extra if dl is None else dl + extra
        if dl is None:
            raise RuntimeError("MaskGitTransformer head: backward called without any gradient")
        d_e = ops.linear_dgrad(dl, s.w["logits"])
        g_c2 = ops.linear_wgrad_det(dl, sv["e"])[: s.V].reshape(ctx.shapes[1])
        d_t, g_ln = ops.norm_bwd(d_e, sv["t"], _f32(sv["w_ln"]), sv["st1"], torch.bfloat16, rms=s.rms, want_dw=True)
        d_c1 = _to_patches(d_t, B, n, p, E)
        d_hN = ops.linear_dgrad(d_c1, s.w["c1"])
        g_c1 = ops.linear_wgrad_det(d_c1, sv["hN"]).view(ctx.shapes[0])
        grads = [g_c1, g_ln, g_c2]
        if s.use_enc_ln:
            dx, g_enc = ops.norm_bwd(d_hN, sv["x"], _f32(sv["w_enc"]), sv["st0"], torch.float32, rms=s.rms, want_dw=True,
                                     bf16_copy=True)
            grads = [g_enc] + grads
        else:
            dx = d_hN.float()
        ctx.sv = None
        return (dx, None, None, *grads)


class _LayerSpec:
    """Static description of one transformer layer handed to the layer Function."""

    def __init__(self, B, S, H, I, nh, eps, rms, normformer, cross, Skv, E, w, enc_op=None, drop=None, ckpt=False):
        self.B, self.S, self.H, self.I, self.nh = B, S, H, I, nh
        self.ckpt = ckpt  # gradient checkpointing: the backward recomputes the layer's activations from its input
        # dropout of this layer in training mode: (attention p, hidden p, seed tensor, first site id) -- self-attention
        # uses site, cross-attention site + 1, the FFN site + 2; a rate of 0 leaves its site out
        self.p_attn, self.p_hidden, self.seed, self.site = drop if drop is not None else (0.0, 0.0, None, 0)
        self.eps, self.rms, self.normformer, self.cross = eps, rms, normformer, cross
        self.Skv, self.E = Skv, E
        self.enc_op = enc_op  # bf16 copy of the (projected, fp32) encoder states used as the K/V GEMM operand
        self.train = torch.is_grad_enabled()  # Function.forward always runs with grad mode off: record the caller's mode
        self.w = w  # dict of packed bf16 weights for this layer
        self.scale = 1.0 / math.sqrt(H // nh)


class _EncProjFn(torch.autograd.Function):
    """encoder_proj + encoder_proj_layer_norm on the text-encoder states (reference :1239-1241): bf16 GEMM, fp32 norm
    output (the autocast dtype flow); the gradient w.r.t. the raw encoder states is not produced (frozen text encoder)."""

    @staticmethod
    def forward(ctx, ehs, w_packed, eps, rms, w_proj, w_norm):
        y0 = ops.linear_fwd(ehs, w_packed)
        grad = any(ctx.needs_input_grad)
        enc, st = ops.norm_fwd(y0, _f32(w_norm), eps, torch.float32, rms=rms, save_stats=grad)
        if grad:
            ctx.sv = (ehs, y0, st, w_norm, rms)
        ctx.set_materialize_grads(False)
        return enc

    @staticmethod
    def backward(ctx, d_enc):
        ehs, y0, st, w_norm, rms = ctx.sv
        if d_enc is None:
            return (None,) * 6
        d_y0, g_norm = ops.norm_bwd(d_enc.contiguous(), y0, _f32(w_norm), st, torch.bfloat16, rms=rms, want_dw=True)
        g_proj = ops.linear_wgrad_det(d_y0, ehs)
        return None, None, None, None, g_proj, g_norm


def _act_dtype(w):
    """dtype of the activation the pass producing a GEMM operand writes: e4m3 rows (ops.FP8) for an F8 weight
    (set_gemm_precision("fp8")), bf16 otherwise"""
    return ops.FP8 if isinstance(w, ops.F8) else torch.bfloat16


def _act_kw(w, key):
    """_act_dtype as a keyword, for the passes whose bf16 output is the default of `key`: empty for a bf16 weight"""
    dt = _act_dtype(w)
    return {} if dt == torch.bfloat16 else {key: dt}


def _layer_body(x, enc, s, params, save, out=True):
    """The forward of one layer: returns (x3, sv).  save=True keeps in sv (and writes the statistics of) every activation
    the backward reads; save=False computes the same x3 with no statistics written.  out=False stops after ml, the last
    tensor the backward reads: the recompute of a checkpointed layer does not run the wo GEMM (x3 is then None)."""
    it = iter(params)
    w_attn_ln, _, _, _, _ = next(it), next(it), next(it), next(it), next(it)
    w_post = next(it) if s.normformer else None
    w_pre, _, _ = next(it), next(it), next(it)
    w_mid = next(it) if s.normformer else None
    next(it)
    if s.cross:
        w_cln = next(it)
        next(it), next(it), next(it), next(it)
        w_cpost = next(it) if s.normformer else None
    H, I, B, S, nh = s.H, s.I, s.B, s.S, s.nh
    sv = {}
    # ---- self attention
    h1, st1 = ops.norm_fwd(x, _f32(w_attn_ln), s.eps, _act_dtype(s.w["qkv"]), rms=s.rms, save_stats=save)
    qkv = ops.linear_fwd(h1, s.w["qkv"])
    if s.p_attn:
        ctxt, lse, abits = ops.attn_fwd(qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:], B, nh, S, S, s.scale, head_dim=H // nh,
                                        dropout=(s.p_attn, s.seed, s.site))
        sv["abits"] = abits
    else:
        ctxt, lse = ops.attn_fwd(qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:], B, nh, S, S, s.scale, head_dim=H // nh)
    fused_norms = s.normformer and not s.cross and H <= 1024  # post-attention norm + FFN pre-norm in one pass
    h2 = st3 = None
    if fused_norms:
        ao = ops.linear_fwd(ctxt, s.w["ao"])
        x2, h2, st2 = ops.norm2_fwd(ao, x, _f32(w_post), _f32(w_pre), s.eps, rms1=s.rms, rms2=0, save_stats=save,
                                    **_act_kw(s.w["wi"], "h2_dtype"))
    elif s.normformer:
        ao = ops.linear_fwd(ctxt, s.w["ao"])
        x2, st2 = ops.norm_fwd(ao, _f32(w_post), s.eps, torch.float32, res=x, rms=s.rms, save_stats=save)
    else:
        ao, st2 = None, None
        x2 = ops.linear_fwd(ctxt, s.w["ao"], res=x)
    if save:
        sv.update(x=x, h1=h1, st1=st1, qkv=qkv, ctxt=ctxt, lse=lse, ao=ao, st2=st2, x2=x2)
    # ---- cross attention (text conditioning, :886-899)
    if s.cross:
        hc, stc = ops.norm_fwd(x2, _f32(w_cln), s.eps, _act_dtype(s.w["cq"]), rms=s.rms, save_stats=save)
        qc = ops.linear_fwd(hc, s.w["cq"])
        enc_op = s.enc_op if s.enc_op is not None else enc  # bf16 GEMM operand (enc itself may be the fp32 projection)
        kvc = ops.linear_fwd(enc_op, s.w["ckv"])
        if s.p_attn:
            cctx, clse, cbits = ops.attn_fwd(qc, kvc[:, :H], kvc[:, H:], B, nh, S, s.Skv, s.scale, head_dim=H // nh,
                                             dropout=(s.p_attn, s.seed, s.site + 1))
            sv["cbits"] = cbits
        else:
            cctx, clse = ops.attn_fwd(qc, kvc[:, :H], kvc[:, H:], B, nh, S, s.Skv, s.scale, head_dim=H // nh)
        if s.normformer:
            cao = ops.linear_fwd(cctx, s.w["co"])
            x2b, stcp = ops.norm_fwd(cao, _f32(w_cpost), s.eps, torch.float32, res=x2, rms=s.rms, save_stats=save)
        else:
            cao, stcp = None, None
            x2b = ops.linear_fwd(cctx, s.w["co"], res=x2)
        if save:
            sv.update(hc=hc, stc=stc, qc=qc, kvc=kvc, cctx=cctx, clse=clse, cao=cao, stcp=stcp, enc=enc_op)
        x2 = x2b
        if save:
            sv["x2b"] = x2b
    # ---- GLU feed-forward (:785-799)
    if h2 is None:
        h2, st3 = ops.norm_fwd(x2, _f32(w_pre), s.eps, _act_dtype(s.w["wi"]), rms=0, save_stats=save)
    ab = ops.linear_fwd(h2, s.w["wi"])
    # FeedForward.dropout (:797) is fused into the pass that writes ml: ml is then the dropped wo operand (which is
    # also what the wo weight gradient reads), and the keep bits are saved for the backward
    ffn_drop = (s.p_hidden, s.seed, s.site + 2)
    if s.normformer and s.p_hidden:
        ml, st4, sv["fbits"] = ops.norm_fwd(ab, _f32(w_mid), s.eps, torch.bfloat16, act=2, rms=s.rms,
                                            save_stats=save, dropout=ffn_drop)
    elif s.normformer:  # GLU product + mid_mlp_layer_norm in one pass; gelu(a)*b is never written to HBM
        ml, st4 = ops.norm_fwd(ab, _f32(w_mid), s.eps, _act_dtype(s.w["wo"]), act=2, rms=s.rms, save_stats=save)
    elif s.p_hidden:
        (ml, sv["fbits"]), st4 = ops.glu_fwd(ab, dropout=ffn_drop), None
    else:
        ml, st4 = ops.glu_fwd(ab, **_act_kw(s.w["wo"], "out_dtype")), None
    x3 = ops.linear_fwd(ml, s.w["wo"], res=x2) if out else None  # an F8 ml: res + bf16(ml @ wo^T) in the FP8 epilogue
    if save:
        sv.update(h2=h2, st3=st3, ab=ab, ml=ml, st4=st4, fused_norms=fused_norms)
    return x3, sv


class _LayerFn(torch.autograd.Function):
    """One pre-LN (normformer) transformer layer: reference TransformerLayer.forward (:875-904).

    With gradient checkpointing (spec.ckpt) the forward keeps only its input x, the encoder states and the spec (whose seed
    tensor and site ids reproduce the dropout masks); the backward re-runs ``_layer_body`` on them with saving on.  Every
    kernel is run-to-run deterministic, so the recomputed activations, and hence the gradients, are bit-identical to the
    ones a saving forward would have kept."""

    @staticmethod
    def forward(ctx, x, enc, spec, *params):
        s = spec
        grad = s.train and any(ctx.needs_input_grad)  # nothing is saved (no statistics written) under no_grad
        recompute = grad and s.ckpt
        x3, sv = _layer_body(x, enc, s, params, save=grad and not recompute)
        if grad:
            ctx.sv = None if recompute else sv
            ctx.inputs = (x, enc) if recompute else None
            ctx.spec, ctx.params = s, params
        return x3

    @staticmethod
    def backward(ctx, dx3):
        s, sv, params = ctx.spec, ctx.sv, ctx.params
        if ctx.inputs is not None:  # checkpointed: recompute the saved set from the layer's input
            _, sv = _layer_body(*ctx.inputs, s, params, save=True, out=False)
            ctx.inputs = None
        H, I, B, S, nh = s.H, s.I, s.B, s.S, s.nh
        dev = dx3.device
        dx3 = dx3.contiguous()
        d_enc = None
        it = iter(params)
        w_attn_ln = next(it); next(it); next(it); next(it); next(it)
        w_post = next(it) if s.normformer else None
        w_pre = next(it); next(it); next(it)
        w_mid = next(it) if s.normformer else None
        next(it)
        if s.cross:
            w_cln = next(it); next(it); next(it); next(it); next(it)
            w_cpost = next(it) if s.normformer else None
        # ---- FFN
        # every weight gradient below is STORED by a fixed-order reduction (deterministic split-K / ordered column sums):
        # no zero-filled buffers, no atomics, bit-identical from run to run
        dy = ops.take_bf16_copy(dx3)  # written by the norm backward that produced dx3 (the next layer's, or the head's)
        if dy is None:
            dy = ops.cast_bf16(dx3)
        d_ml = ops.linear_dgrad(dy, s.w["wo"])
        g_wo = ops.linear_wgrad_det(dy, sv["ml"])
        if s.normformer and s.p_hidden:  # d_ml is scaled by the keep bits as it is read; the saved ml is the dropped
            # output, so the kernel recomputes the GLU product from [a | b] instead of reading it
            d_ab, g_mid = ops.norm_bwd(d_ml, sv["ab"], _f32(w_mid), sv["st4"], torch.bfloat16, act=2, rms=s.rms,
                                       want_dw=True, dropout=(s.p_hidden, sv["fbits"]))
        elif s.normformer:  # LN backward + GLU backward fused: reads d_ml and [a|b], writes d[a|b]
            d_ab, g_mid = ops.norm_bwd(d_ml, sv["ab"], _f32(w_mid), sv["st4"], torch.bfloat16, act=2, rms=s.rms,
                                       y_fwd=sv["ml"], want_dw=True)
        elif s.p_hidden:
            g_mid, d_ab = None, ops.glu_bwd(sv["ab"], d_ml, dropout=(s.p_hidden, sv["fbits"]))
        else:
            g_mid = None
            d_ab = ops.glu_bwd(sv["ab"], d_ml)
        d_h2 = ops.linear_dgrad(d_ab, s.w["wi"])
        g_wi = ops.linear_wgrad_det(d_ab, sv["h2"])
        x_mid = sv["x2b"] if s.cross else sv["x2"]
        if sv["fused_norms"]:  # FFN pre-norm backward + post-attention norm backward in one pass
            dx2, d_ao, g_post, g_pre = ops.norm2_bwd(d_h2, x_mid, _f32(w_pre), dx3, sv["ao"], _f32(w_post), sv["st2"],
                                                     rms1=s.rms, rms2=0)
        else:
            dx2, g_pre = ops.norm_bwd(d_h2, x_mid, _f32(w_pre), sv["st3"], torch.float32, dres=dx3, rms=0, want_dw=True)
        # ---- cross attention
        cross_grads = []
        if s.cross:
            if s.normformer:
                d_cao, g_cpost = ops.norm_bwd(dx2, sv["cao"], _f32(w_cpost), sv["stcp"], torch.bfloat16, rms=s.rms,
                                              want_dw=True)
            else:
                g_cpost, d_cao = None, ops.cast_bf16(dx2)
            d_cctx = ops.linear_dgrad(d_cao, s.w["co"])
            g_co = ops.linear_wgrad_det(d_cao, sv["cctx"])
            d_qc = torch.empty_like(sv["qc"])
            d_kvc = torch.empty_like(sv["kvc"])
            kvc = sv["kvc"]
            ops.attn_bwd(sv["qc"], kvc[:, :H], kvc[:, H:], sv["cctx"], d_cctx, sv["clse"], d_qc, d_kvc[:, :H],
                         d_kvc[:, H:], B, nh, S, s.Skv, s.scale, head_dim=H // nh,
                         **({"dropout": (s.p_attn, sv["cbits"])} if s.p_attn else {}))
            g_ckv = ops.linear_wgrad_det(d_kvc, sv["enc"])
            if ctx.needs_input_grad[1]:  # projected encoder states: d enc = d[k|v] @ [Wk;Wv], fp32, summed over layers by autograd
                d_enc = ops.linear_dgrad(d_kvc, s.w["ckv"], out_dtype=torch.float32)
            d_hc = ops.linear_dgrad(d_qc, s.w["cq"])
            g_cq = ops.linear_wgrad_det(d_qc, sv["hc"])
            dx2, g_cln = ops.norm_bwd(d_hc, sv["x2"], _f32(w_cln), sv["stc"], torch.float32, dres=dx2, rms=s.rms,
                                      want_dw=True)
            cross_grads = [g_cln, g_cq, g_ckv[:H], g_ckv[H:], g_co] + ([g_cpost] if s.normformer else [])
        # ---- self attention
        if sv["fused_norms"]:
            pass  # d_ao / g_post came out of the fused norm backward above
        elif s.normformer:
            d_ao, g_post = ops.norm_bwd(dx2, sv["ao"], _f32(w_post), sv["st2"], torch.bfloat16, rms=s.rms, want_dw=True)
        else:
            g_post, d_ao = None, ops.cast_bf16(dx2)
        d_ctx = ops.linear_dgrad(d_ao, s.w["ao"])
        g_ao = ops.linear_wgrad_det(d_ao, sv["ctxt"])
        qkv = sv["qkv"]
        d_qkv = torch.empty_like(qkv)
        ops.attn_bwd(qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:], sv["ctxt"], d_ctx, sv["lse"], d_qkv[:, :H],
                     d_qkv[:, H:2 * H], d_qkv[:, 2 * H:], B, nh, S, S, s.scale, head_dim=H // nh,
                     **({"dropout": (s.p_attn, sv["abits"])} if s.p_attn else {}))
        d_h1 = ops.linear_dgrad(d_qkv, s.w["qkv"])
        g_qkv = ops.linear_wgrad_det(d_qkv, sv["h1"])
        dx1, g_attn_ln = ops.norm_bwd(d_h1, sv["x"], _f32(w_attn_ln), sv["st1"], torch.float32, dres=dx2, rms=s.rms,
                                      want_dw=True, bf16_copy=True)  # dx1 is the previous layer's dx3
        grads = [g_attn_ln, g_qkv[:H], g_qkv[H:2 * H], g_qkv[2 * H:], g_ao]
        if s.normformer:
            grads.append(g_post)
        grads += [g_pre, g_wi[:I], g_wi[I:]]
        if s.normformer:
            grads.append(g_mid)
        grads.append(g_wo)
        grads += cross_grads
        ctx.sv = None
        return (dx1, d_enc, None, *grads)


class _HeadSpec:
    def __init__(self, T, H, V, Vpad, eps, rms, use_enc_ln, use_mlm, w, label_smoothing, n_cols=None):
        self.T, self.H, self.V, self.Vpad, self.eps, self.rms = T, H, V, Vpad, eps, rms
        self.use_enc_ln, self.use_mlm, self.w, self.ls = use_enc_ln, use_mlm, w, label_smoothing
        # inference only: compute just the first n_cols logit columns (generate2 reads the codebook_size columns of a
        # vocab_size-wide head, reference :1417 -- the other half of that GEMM would be thrown away)
        self.n_cols = n_cols
        self.train = torch.is_grad_enabled()


class _HeadFn(torch.autograd.Function):
    """encoder_layer_norm -> MlmLayer (dense, GELU, LN, to_logits) -> masked CE (:1268-1280)."""

    @staticmethod
    def forward(ctx, x, labels, spec, *params):
        s = spec
        grad = s.train and any(ctx.needs_input_grad)  # nothing is saved (no statistics written) under no_grad
        it = iter(params)
        w_enc = next(it) if s.use_enc_ln else None
        if s.use_mlm:
            next(it)
            w_mlm_ln = next(it)
        sv = {}
        if s.use_enc_ln:
            hN, st0 = ops.norm_fwd(x, _f32(w_enc), s.eps, torch.bfloat16, rms=s.rms, save_stats=grad)
        else:
            hN, st0 = ops.cast_bf16(x), None
        if s.use_mlm:
            d = ops.linear_fwd(hN, s.w["dense"])
            e, st1 = ops.norm_fwd(d, _f32(w_mlm_ln), s.eps, torch.bfloat16, act=1, rms=s.rms, save_stats=grad)
        else:
            d, e, st1 = None, hN, None
        if s.n_cols is not None:
            if grad or labels is not None:
                raise RuntimeError("column-restricted logits are an inference-only path")
            ncol = ((s.n_cols + 7) // 8) * 8
            logits = torch.empty(s.T, ncol, dtype=torch.bfloat16, device=x.device)
            ops.gemm(e, s.w["logits"], logits, s.T, ncol, s.H, s.H, s.H, ncol)
            return logits[:, : s.n_cols]
        logits = torch.empty(s.T, s.Vpad, dtype=torch.bfloat16, device=x.device)
        ops.gemm(e, s.w["logits"], logits, s.T, s.Vpad, s.H, s.H, s.H, s.Vpad)
        loss = None
        ctx.set_materialize_grads(False)  # an unused logits output must not cost a zero-filled [T,V] gradient
        if labels is not None:
            loss_out, ws = ops.ce_fwd(logits, labels, s.V, s.ls)
            loss = loss_out[0]
            sv.update(loss_out=loss_out, ws=ws, labels=labels)
        if grad:
            sv.update(x=x, hN=hN, st0=st0, d=d, e=e, st1=st1, logits=logits)
            ctx.sv, ctx.spec, ctx.params = sv, s, params
        out_logits = logits[:, : s.V]
        if loss is None:
            return out_logits
        return out_logits, loss

    @staticmethod
    def backward(ctx, d_logits, d_loss=None):
        s, sv, params = ctx.spec, ctx.sv, ctx.params
        dev = sv["x"].device
        it = iter(params)
        w_enc = next(it) if s.use_enc_ln else None
        if s.use_mlm:
            next(it)
            w_mlm_ln = next(it)
        dl = None
        if d_loss is not None and "labels" in sv:
            dl = ops.ce_bwd(sv["logits"], sv["labels"], sv["ws"], d_loss.to(torch.float32).reshape(1).contiguous(),
                            sv["loss_out"], s.V, s.ls)
        if d_logits is not None:  # gradient arriving through the returned logits (rare: custom losses)
            extra = torch.zeros(s.T, s.Vpad, dtype=torch.bfloat16, device=dev)
            extra[:, : s.V] = d_logits.to(torch.bfloat16)
            dl = extra if dl is None else dl + extra
        if dl is None:
            raise RuntimeError("MaskGitTransformer head: backward called without any gradient")
        d_e = ops.linear_dgrad(dl, s.w["logits"])
        g_logits = ops.linear_wgrad_det(dl, sv["e"])
        grads = []
        if s.use_mlm:
            d_d, g_mlm_ln = ops.norm_bwd(d_e, sv["d"], _f32(w_mlm_ln), sv["st1"], torch.bfloat16, act=1, rms=s.rms,
                                         want_dw=True)
            d_hN = ops.linear_dgrad(d_d, s.w["dense"])
            g_dense = ops.linear_wgrad_det(d_d, sv["hN"])
            grads = [g_dense, g_mlm_ln]
        else:
            d_hN = d_e
        if s.use_enc_ln:
            dx, g_enc = ops.norm_bwd(d_hN, sv["x"], _f32(w_enc), sv["st0"], torch.float32, rms=s.rms, want_dw=True,
                                     bf16_copy=True)  # dx is the last layer's dx3
            grads = [g_enc] + grads
        else:
            dx = d_hN.float()
        grads.append(g_logits[: s.V])
        ctx.sv = None
        return (dx, None, None, *grads)


# --------------------------------------------------------------------------------------------
# The model
# --------------------------------------------------------------------------------------------
class MaskGitTransformer(ModelMixin, ConfigMixin):
    _supports_gradient_checkpointing = True

    @register_to_config
    def __init__(
        self,
        vocab_size,  # codebook_size + 1 (mask token) [+ num_classes for class-conditional models]
        hidden_size=768,
        embedding_size=None,
        num_hidden_layers=12,
        num_attention_heads=12,
        intermediate_size=3072,
        hidden_dropout=0.1,
        attention_dropout=0.1,
        max_position_embeddings=256,
        add_cross_attention=False,
        encoder_hidden_size=1024,
        project_encoder_hidden_states=False,
        initializer_range=0.02,
        norm_type="layernorm",
        layer_norm_eps=1e-5,
        use_normformer=True,
        use_encoder_layernorm=True,
        use_mlm_layer=True,
        use_mlm_layernorm=True,
        use_bias=False,
        codebook_size=1024,
        num_vq_tokens=256,
        num_classes=None,
        use_codebook_size_for_output=False,
        use_conv_in_out=False,
        patch_size=1,
        **kwargs,
    ):
        super().__init__()
        if use_bias:
            raise NotImplementedError("open_muse_b200: use_bias=True is not supported (no reference config enables it)")
        if use_conv_in_out and not isinstance(embedding_size, int):
            # the reference hands the raw ``embedding_size`` to ConvEmbed (:1133-1135): left unset -- as in the two yaml files
            # that enable the flag, configs/cc12m_movq.yaml and imagenet_text2image_movq_conv.yaml -- nn.Embedding(vocab, None)
            # raises this TypeError there too
            raise TypeError("use_conv_in_out=True needs an explicit integer embedding_size (the reference raises in "
                            "nn.Embedding(vocab_size, None) when it is left unset)")
        if use_conv_in_out and (patch_size < 1 or (embedding_size * patch_size ** 2) % 8 or embedding_size % 8):
            raise NotImplementedError("open_muse_b200: use_conv_in_out needs embedding_size to be a multiple of 8 (16-byte "
                                      "rows for the TMA operands)")
        # without use_conv_in_out the reference ignores embedding_size: Embed is built with hidden_size twice (:1143-1146, Q5)
        if use_conv_in_out and not use_mlm_layer:
            raise NotImplementedError("open_muse_b200: use_conv_in_out without use_mlm_layer (logits on the patch grid) is "
                                      "not supported")
        if use_mlm_layer and not use_mlm_layernorm and not use_conv_in_out:
            raise NotImplementedError("open_muse_b200: use_mlm_layer without use_mlm_layernorm is not supported yet")
        if hidden_size % num_attention_heads or hidden_size // num_attention_heads not in (48, 64, 96, 128):
            if hidden_size % num_attention_heads:
                raise ValueError(
                    f"embed_dim must be divisible by num_heads (got `embed_dim`: {hidden_size} and `num_heads`:"
                    f" {num_attention_heads})."
                )
            raise NotImplementedError("open_muse_b200: head_dim must be 48, 64, 96 or 128 (the reference configs use 64, "
                                      "and 48 in configs/imagenet.yaml / imagenet_movq.yaml: hidden 768, 16 heads)")
        self.vocab_size = vocab_size
        self.hidden_size = hidden_size
        self.num_hidden_layers = num_hidden_layers
        self.num_attention_heads = num_attention_heads
        self.intermediate_size = intermediate_size
        self.hidden_dropout = hidden_dropout
        self.attention_dropout = attention_dropout
        self.max_position_embeddings = max_position_embeddings
        self.initializer_range = initializer_range
        self.embedding_size = embedding_size or hidden_size
        self.register_to_config(mask_token_id=vocab_size - 1)

        # construction order == reference (:1130-1197) so seeded initialisation is identical
        if use_conv_in_out:  # (:1132-1141; ConvEmbed keeps its own max_position_embeddings default of 256)
            self.embed = ConvEmbed(vocab_size, embedding_size, hidden_size, patch_size=patch_size, norm_type=norm_type,
                                   layer_norm_eps=layer_norm_eps, use_bias=use_bias)
        else:
            self.embed = Embed(vocab_size, hidden_size, hidden_dropout, max_position_embeddings)
        if add_cross_attention is not None and project_encoder_hidden_states:  # (:1154-1157)
            self.encoder_proj = nn.Linear(encoder_hidden_size, hidden_size, bias=use_bias)
            self.encoder_proj_layer_norm = _norm(norm_type, hidden_size, layer_norm_eps, use_bias)
            encoder_hidden_size = hidden_size
        self.transformer_layers = nn.ModuleList(
            [
                TransformerLayer(hidden_size, intermediate_size, num_attention_heads, encoder_hidden_size,
                                 add_cross_attention, hidden_dropout, attention_dropout, norm_type, layer_norm_eps,
                                 use_normformer, use_bias)
                for _ in range(num_hidden_layers)
            ]
        )
        if use_encoder_layernorm:
            self.encoder_layer_norm = _norm(norm_type, hidden_size, layer_norm_eps, use_bias)
        self.output_size = codebook_size if use_codebook_size_for_output else vocab_size
        self.padded_output_size = ((self.output_size + 63) // 64) * 64  # TMA-friendly logits pitch
        if use_mlm_layer and use_conv_in_out:  # (:1182-1191)
            self.mlm_layer = ConvMlmLayer(self.output_size, embedding_size, hidden_size, patch_size=patch_size,
                                          norm_type=norm_type, layer_norm_eps=layer_norm_eps, use_bias=use_bias)
        elif use_mlm_layer:
            self.mlm_layer = MlmLayer(hidden_size, self.output_size, norm_type, layer_norm_eps, use_mlm_layernorm, use_bias)
        else:
            self.to_logits = nn.Linear(hidden_size, self.output_size, bias=use_bias)
        self.gradient_checkpointing = False
        self.apply(self._init_weights)
        self._gemm_precision = "bf16"
        self._packed = _PackedWeights(self)

    def _init_weights(self, module):
        # truncated normal for Linear / Embedding, ones for norm weights (reference :1201-1219)
        if isinstance(module, nn.Linear):
            nn.init.trunc_normal_(module.weight, std=self.config.initializer_range)
            if module.bias is not None:
                module.bias.data.zero_()
        elif isinstance(module, nn.Embedding):
            nn.init.trunc_normal_(module.weight, std=self.config.initializer_range)
        elif isinstance(module, (nn.LayerNorm, RMSNorm)):
            if getattr(module, "weight", None) is not None:
                module.weight.data.fill_(1.0)

    def _set_gradient_checkpointing(self, module, value=False):
        self.gradient_checkpointing = True  # (reference quirk Q6: ``value`` is ignored)

    # ------------------------------------------------------------------ GEMM precision
    def set_gemm_precision(self, mode: str):
        """"bf16" (default: the reference's autocast recipe) or "fp8": inference only -- forward under torch.no_grad() in
        eval mode, and generate2 -- with the e4m3 tensor cores for each layer's [q;k;v], cross-attention q, [wi_0;wi_1]
        and wo GEMMs (wo with its residual add fused into the FP8 epilogue).  Their activations come out of the norm / GLU
        passes that produce them as e4m3 with one scale per row, the weights are quantized per output row; every other
        GEMM stays bf16 (DESIGN.md section 5).  Not a config key: save_pretrained / from_pretrained do not see it.
        "fp8" needs hidden_size and intermediate_size to be multiples of 16 (the e4m3 rows are fed by TMA, whose row
        pitches are multiples of 16 bytes), hidden_size <= 1024 (the warp-per-row norm passes) and intermediate_size <=
        4096 (the GLU + mid-norm pass holds the row in registers)."""
        if mode not in ("bf16", "fp8"):
            raise ValueError(f"gemm precision must be 'bf16' or 'fp8', got {mode!r}")
        H, I = self.hidden_size, self.intermediate_size
        if mode == "fp8":
            bad = {k: v for k, v in dict(hidden_size=H, intermediate_size=I).items() if v % 16}
            if bad:
                raise ValueError(f"gemm precision 'fp8' needs widths that are multiples of 16, got {bad}")
            if H > 1024 or I > 4096:
                raise ValueError(f"gemm precision 'fp8' needs hidden_size <= 1024 and intermediate_size <= 4096, got "
                                 f"{H} and {I}")
        self._gemm_precision = mode  # part of the operand cache key: the next forward rebuilds the operands
        return self

    @property
    def gemm_precision(self) -> str:
        return self._gemm_precision

    def _check_fp8_inference(self):
        if self._gemm_precision == "fp8" and (self.training or torch.is_grad_enabled()):
            raise RuntimeError("MaskGitTransformer in FP8 GEMM precision is inference only: call model.eval() and run under "
                               "torch.no_grad(), or set_gemm_precision('bf16') to train")

    # ------------------------------------------------------------------ parameter lists (Function order)
    def _layer_params(self, layer):
        c = self.config
        a, f = layer.attention, layer.ffn
        ps = [layer.attn_layer_norm.weight, a.query.weight, a.key.weight, a.value.weight, a.out.weight]
        if c.use_normformer:
            ps.append(layer.post_attn_layer_norm.weight)
        ps += [f.pre_mlp_layer_norm.weight, f.wi_0.weight, f.wi_1.weight]
        if c.use_normformer:
            ps.append(f.mid_mlp_layer_norm.weight)
        ps.append(f.wo.weight)
        if c.add_cross_attention:
            x = layer.crossattention
            ps += [layer.crossattn_layer_norm.weight, x.query.weight, x.key.weight, x.value.weight, x.out.weight]
            if c.use_normformer:
                ps.append(layer.post_crossattn_layer_norm.weight)
        return ps

    def _head_params(self):
        c = self.config
        ps = [self.encoder_layer_norm.weight] if c.use_encoder_layernorm else []
        if c.use_mlm_layer and c.use_conv_in_out:
            ps += [self.mlm_layer.conv1.weight, self.mlm_layer.layer_norm.norm.weight, self.mlm_layer.conv2.weight]
        elif c.use_mlm_layer:
            ps += [self.mlm_layer.mlm_dense.weight, self.mlm_layer.mlm_ln.weight, self.mlm_layer.to_logits.weight]
        else:
            ps.append(self.to_logits.weight)
        return ps

    # ------------------------------------------------------------------ forward
    def forward(
        self,
        input_ids,
        encoder_hidden_states=None,
        encoder_attention_mask=None,
        labels=None,
        label_smoothing=0.0,
        cond_dropout_prob=0.0,
        _raw_bf16=False,
        _logit_cols=None,
        **kwargs,  # cond_embeds / loss_weight / micro_conds from train_muse.py:742-750 are accepted and ignored
    ):
        c = self.config
        if c.add_cross_attention and encoder_hidden_states is None:
            raise ValueError("If `add_cross_attention` is True, `encoder_hidden_states` should be provided.")
        if encoder_attention_mask is not None:
            raise TypeError("encoder_attention_mask is not supported (it raises in the reference too: quirk Q2)")
        if not input_ids.is_cuda:
            raise RuntimeError("open_muse_b200.MaskGitTransformer runs on CUDA (sm_90a) only; move inputs to the GPU")
        self._check_fp8_inference()
        B, S = input_ids.shape
        if _CHECK_IDS:  # debug switch (MUSE_B200_CHECK_IDS=1): torch raises a device assert on out-of-range ids / labels,
            # the kernels clamp silently -- this host-side check (one sync) catches class-offset / vocab mix-ups
            lo, hi = int(input_ids.min()), int(input_ids.max())
            if lo < 0 or hi >= self.vocab_size:
                raise IndexError(f"input_ids out of range [0, {self.vocab_size}): min {lo}, max {hi}")
            if labels is not None:
                bad = (labels != -100) & ((labels < 0) | (labels >= self.output_size))
                if bool(bad.any()):
                    raise IndexError(f"labels out of range [0, {self.output_size}) (other than -100)")
        H = self.hidden_size
        rms = 0 if c.norm_type == "layernorm" else 1
        S_out, conv = S, None  # use_conv_in_out: S tokens outside the transformer, S / patch^2 inside
        if c.use_conv_in_out:
            n, p = math.isqrt(S), c.patch_size
            if n * n != S or n % p:
                raise ValueError(f"use_conv_in_out: the {S} tokens must form a square grid divisible by patch_size {p}")
            S = S // (p * p)
            if S > self.embed.max_position_embeddings:
                raise IndexError(f"{S} patches exceed ConvEmbed's {self.embed.max_position_embeddings} positions")
        elif S > self.max_position_embeddings:
            raise IndexError(f"sequence length {S} exceeds max_position_embeddings {self.max_position_embeddings}")
        packed = self._packed.refresh()
        ids = input_ids.contiguous().to(torch.int64)
        # nn.Dropout is active iff the module is in training mode (also under no_grad).  One seed per forward, drawn on the
        # device from torch's default generator: torch.manual_seed reproduces the masks, and a captured CUDA graph draws
        # a fresh seed on every replay without a host sync.  Site ids: 0 the embedding, 1 + 3 i .. 3 + 3 i layer i.
        p_hidden, p_attn, seed = 0.0, 0.0, None
        if self.training and (self.hidden_dropout > 0.0 or self.attention_dropout > 0.0):
            p_hidden, p_attn = float(self.hidden_dropout), float(self.attention_dropout)
            seed = torch.randint(-2 ** 63, 2 ** 63 - 1, (1,), dtype=torch.int64, device=input_ids.device)
        if c.use_conv_in_out:
            conv = _ConvSpec(B, n, p, self.embedding_size, H, c.layer_norm_eps, rms, packed.head)
            x = _ConvEmbedFn.apply(ids, conv, self.embed.embeddings.weight, self.embed.layer_norm.weight,
                                   self.embed.conv.weight, self.embed.position_embeddings.weight)
        else:
            x = _EmbedFn.apply(ids, self.embed.word_embeddings.weight, self.embed.position_embeddings.weight,
                               (p_hidden, seed, 0) if p_hidden else None)

        enc = None
        Skv = E = 0
        if c.add_cross_attention and encoder_hidden_states is not None:
            if encoder_hidden_states.requires_grad:
                raise NotImplementedError("gradients w.r.t. encoder_hidden_states are not implemented")
            ehs = encoder_hidden_states
            if self.training and cond_dropout_prob > 0.0:  # classifier-free-guidance dropout (:1244-1247)
                keep = torch.zeros((ehs.shape[0], 1, 1), device=ehs.device).float().uniform_(0, 1) < (1.0 - cond_dropout_prob)
                ehs = ehs * keep
            Skv, E = ehs.shape[1], ehs.shape[2]
            enc = ehs.reshape(B * Skv, E).to(torch.bfloat16).contiguous()
        enc_op = None
        # (:1239-1241). The reference drops conditioning after this projection; dropping the raw states first is the same
        # function and the same gradients because the projection and the norm have no bias (zero rows stay zero).
        if enc is not None and c.project_encoder_hidden_states:
            enc = _EncProjFn.apply(enc, packed.head["eproj"], c.layer_norm_eps, rms, self.encoder_proj.weight,
                                   self.encoder_proj_layer_norm.weight)
            E = H
            enc_op = ops.cast_bf16(enc.detach())
        for i, layer in enumerate(self.transformer_layers):
            spec = _LayerSpec(B, S, H, self.intermediate_size, self.num_attention_heads, c.layer_norm_eps, rms,
                              c.use_normformer, enc is not None, Skv, E, packed.layers[i], enc_op,
                              drop=(p_attn, p_hidden, seed, 1 + 3 * i) if seed is not None else None,
                              ckpt=self.gradient_checkpointing)
            x = _LayerFn.apply(x, enc, spec, *self._layer_params(layer))

        flat_labels = labels.reshape(-1).contiguous().to(torch.int64) if labels is not None else None
        if _logit_cols is not None and (_logit_cols >= self.output_size or labels is not None or torch.is_grad_enabled()):
            _logit_cols = None
        if conv is not None:
            hspec = _ConvSpec(B, conv.n, conv.p, conv.E, H, c.layer_norm_eps, rms, packed.head, V=self.output_size,
                              Vpad=self.padded_output_size, use_enc_ln=c.use_encoder_layernorm,
                              label_smoothing=label_smoothing, n_cols=_logit_cols)
            out = _ConvHeadFn.apply(x, flat_labels, hspec, *self._head_params())
        else:
            hspec = _HeadSpec(B * S, H, self.output_size, self.padded_output_size, c.layer_norm_eps, rms,
                              c.use_encoder_layernorm, c.use_mlm_layer, packed.head, label_smoothing, n_cols=_logit_cols)
            out = _HeadFn.apply(x, flat_labels, hspec, *self._head_params())
        if labels is not None:
            logits, loss = out
        else:
            logits, loss = out, None
        logits = logits.unflatten(0, (B, S_out))
        if _raw_bf16:
            return logits, loss
        if not torch.is_autocast_enabled("cuda"):
            logits = logits.float()  # the reference returns fp32 logits outside autocast
        if labels is not None:
            return logits, loss
        return logits

    # ------------------------------------------------------------------ generation
    def generate(self, *args, **kwargs):
        raise AttributeError(
            "MaskGitTransformer.generate is broken in the reference at this commit (quirk Q1: `None.scatter`); "
            "use generate2, which is what PipelineMuse calls"
        )

    @torch.no_grad()
    def generate2(
        self,
        input_ids: torch.LongTensor = None,
        class_ids: torch.LongTensor = None,
        encoder_hidden_states: torch.FloatTensor = None,
        negative_embeds: torch.FloatTensor = None,
        temperature=1.0,
        timesteps=18,
        guidance_scale=0,
        noise_schedule=cosine_schedule,
        generator: torch.Generator = None,
        _noise=None,
        _trace=None,
        **kwargs,
    ):
        """MaskGIT iterative parallel decoding, same semantics as the reference (:1363-1456).

        The whole loop -- ``timesteps`` x (forward, Exp(1) / uniform draws from the torch generator, fused sample /
        confidence / re-mask kernel) -- is captured once per (shape, schedule) into ONE CUDA graph and replayed: a call
        costs a handful of host launches instead of ~80 per step.  ``use_cuda_graph=False`` (or the private test hooks
        ``_noise`` = per-step (q_exp, u) tensors, ``_trace`` = list collecting per-step state) run the same kernels launched
        one by one."""
        c = self.config
        if self.training and (self.hidden_dropout > 0.0 or self.attention_dropout > 0.0):
            # the reference would sample with dropout applied to every forward of the decode loop
            raise RuntimeError("generate2 on a MaskGitTransformer in training mode would sample with dropout > 0 active; "
                               "call model.eval() first")
        mask_id, seq_len, n_codes = c.mask_token_id, c.num_vq_tokens, c.codebook_size
        batch = len(class_ids) if class_ids is not None else encoder_hidden_states.shape[0]
        if class_ids is not None:
            class_ids += n_codes  # in place on the caller's tensor, like the reference (quirk Q3)
        if input_ids is None:
            input_ids = torch.full((batch, seq_len), mask_id, dtype=torch.long, device=self.device)
        input_ids = input_ids.contiguous()
        use_graph = kwargs.pop("use_cuda_graph", None)
        if use_graph is None:
            use_graph = _os.environ.get("MUSE_B200_GENERATE_GRAPH", "1") != "0"
        use_graph = bool(use_graph) and _noise is None and _trace is None and input_ids.is_cuda
        args = (input_ids, class_ids, encoder_hidden_states, negative_embeds)
        sched = (float(temperature), int(timesteps), float(guidance_scale), noise_schedule)
        if not use_graph:
            return self._generate2_loop(*args, *sched, generator, _noise, _trace)
        return self._generate2_graphed(args, sched, generator)

    def _generate2_loop(self, input_ids, class_ids, encoder_hidden_states, negative_embeds, temperature, timesteps,
                        guidance_scale, noise_schedule, generator, noise=None, trace=None):
        c = self.config
        mask_id, n_codes = c.mask_token_id, c.codebook_size
        batch, seq_len = input_ids.shape  # every shape below follows the ids (inpainting may pass its own length)
        use_cfg = encoder_hidden_states is not None and guidance_scale > 0
        if use_cfg:
            uncond = torch.zeros_like(encoder_hidden_states) if negative_embeds is None else negative_embeds
            cfg_states = torch.cat([encoder_hidden_states, uncond])
        sampled_ids = input_ids
        for step in range(timesteps):
            model_in = input_ids if class_ids is None else torch.cat([class_ids[:, None], input_ids], dim=1)
            if use_cfg:
                both, _ = self(torch.cat([model_in] * 2), encoder_hidden_states=cfg_states, _raw_bf16=True, _logit_cols=n_codes)
                logits, logits_unc = both[:batch], both[batch:]
            else:
                logits, _ = self(model_in, encoder_hidden_states=encoder_hidden_states, _raw_bf16=True, _logit_cols=n_codes)
                logits_unc = None
            # the generator is consumed exactly like the reference: multinomial(n=1) draws Exp(1) noise of the
            # probabilities' shape (ATen), mask_by_random_topk draws one uniform per token (sampling.py:13-15)
            if noise is not None:
                q_exp, u = noise[step]
            else:
                q_exp = torch.empty(batch * seq_len, n_codes, dtype=torch.float32, device=logits.device).exponential_(1, generator=generator)
                u = torch.zeros(batch, seq_len, dtype=torch.float32, device=logits.device).uniform_(0, 1, generator=generator)
            ratio = 1.0 * (step + 1) / timesteps
            mask_len = int((seq_len * noise_schedule(torch.tensor(ratio))).floor())
            temperature = temperature * (1.0 - ratio)  # compounds across steps (quirk Q4)
            prev = input_ids
            sampled_ids, input_ids = ops.sample_step(
                logits, input_ids, q_exp, u, n_codes, mask_id, mask_len, temperature, logits_unc=logits_unc,
                guidance=guidance_scale, skip_first_token=class_ids is not None)
            if trace is not None:
                off = 1 if class_ids is not None else 0
                trace.append(dict(step=step, input_ids=prev.clone(), logits=logits[:, off:, :n_codes].clone(),
                                  logits_unc=None if logits_unc is None else logits_unc[:, off:, :n_codes].clone(),
                                  sampled=sampled_ids.clone(), next_ids=input_ids.clone(), mask_len=mask_len,
                                  temperature=temperature))
        return sampled_ids

    def _generate2_graphed(self, args, sched, generator):
        """Replay (capturing on first use) the whole decode loop as one CUDA graph.  Static input buffers; the torch
        generator is registered with the graph, so replays consume its stream exactly like the launched-one-by-one path."""
        packed = self._packed.refresh()  # outside the graph: replays must see the current weights in the same buffers
        key = (tuple((tuple(a.shape), a.dtype, a.device) if a is not None else None for a in args), sched,
               None if generator is None else id(generator), getattr(packed, "layout_key", None),
               torch.is_autocast_enabled("cuda"), self._gemm_precision)
        cache = self.__dict__.setdefault("_gen_graphs", {})
        entry = cache.get(key)
        if entry is None:
            static = [None if a is None else a.clone() for a in args]
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            dev = args[0].device
            state = torch.cuda.get_rng_state(dev) if generator is None else generator.get_state()
            with torch.cuda.stream(side):  # lazy initialisation (kernel attributes, allocator) off the capture
                self._generate2_loop(*static, *sched, generator)
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize(dev)
            if generator is not None:  # the warm-up run must not advance the caller's random stream
                generator.set_state(state)
            else:
                torch.cuda.set_rng_state(state, dev)
            graph = torch.cuda.CUDAGraph()
            if generator is not None:
                graph.register_generator_state(generator)
            with torch.cuda.graph(graph):
                out = self._generate2_loop(*static, *sched, generator)
            if len(cache) >= 8:
                cache.pop(next(iter(cache)))
            entry = cache[key] = (graph, static, out, generator)
        graph, static, out, _ = entry
        for dst, src in zip(static, args):
            if dst is not None:
                dst.copy_(src, non_blocking=True)
        graph.replay()
        return out.clone()
