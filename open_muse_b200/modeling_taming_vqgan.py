"""``VQGANModel`` -- the taming-transformers tokenizer every text-to-image config of the reference uses
(muse/modeling_taming_vqgan.py), behind the reference's surface: same constructor / config keys, parameter names
(``encoder.down.{l}.block.{b}.conv1.weight``, ``encoder.down.{l}.attn.{b}.q.weight``, ``encoder.down.{l}.downsample.conv``,
``decoder.up.{l}.upsample.conv``, ``quant_conv``, ``post_quant_conv``, ``quantize.embedding.weight``), construction order
(seeded initialisation identical) and methods ``encode / decode / decode_code / get_code / forward``.

Inference only (the tokenizer is frozen in both training scripts).  Everything runs in libmuse_b200, NHWC fp32 between
layers with fp32-faithful tensor-core convolutions (csrc/conv_tc.cu):
  * ResnetBlock (:65-134): GroupNorm+SiLU(+split) -> 3x3 conv -> GroupNorm+SiLU -> 3x3 conv (+ x or nin_shortcut(x) fused
    as the residual of the second conv's epilogue); all convolutions carry a bias here.
  * Downsample (:47-62): pad (0,1,0,1) + 3x3 stride 2 = space-to-depth + a stride-1 2x2 convolution over 4*C channels.
  * Upsample (:27-44): nearest x2 + 3x3 conv as four 2x2 parity convolutions on the low-resolution input.
  * AttnBlock (:137-174): GroupNorm -> q, k, v 1x1 convs -> one 512-wide head over the 16x16 tokens; both attention
    products are 1x1 convolutions with per-image weights (keys / values), softmax in fp32 -> proj_out (+ residual).
  * quantiser: the bit-exact arg-min / lookup kernels of MaskGitVQGAN.

The blocks also build the MoVQ tokenizer (modeling_movq.py): ``norm`` makes its decoder norms SpatialNorms, modulated by
the latent ``zq`` that ``run`` then passes down, and ``linear`` gives the AttnBlocks nn.Linear projections.
"""
from __future__ import annotations

import math
from functools import partial
from typing import Tuple

import torch
from torch import nn

from . import ops
from .modeling_utils import ConfigMixin, ModelMixin, register_to_config

_GN = dict(num_groups=32, eps=1e-6, affine=True)


def _gn(norm, silu=1):
    return (norm.weight, norm.bias, 32, 1e-6, silu)


def _group_norm(channels):
    return nn.GroupNorm(num_channels=channels, **_GN)


def _norm(norm, zq, silu=1):
    """ops.conv2d / ops.groupnorm_silu arguments of a block norm: an nn.GroupNorm, or with the latent zq (fp32 NHWC) a MoVQ
    SpatialNorm, whose GroupNorm output is modulated by its 1x1 conv_y / conv_b of zq."""
    if zq is None:
        return dict(gn=_gn(norm, silu))
    return dict(gn=_gn(norm.norm_layer, silu), spatial=(zq, norm.conv_y, norm.conv_b))


def _conv1x1(w):
    """the [C, C, 1, 1] weight ops.conv2d takes, for an nn.Conv2d or an nn.Linear [C, C] weight; the Linear's view is kept on
    the parameter so that the packed-weight caches, keyed per tensor, keep hitting"""
    if w.dim() == 4:
        return w
    v = getattr(w, "_conv_view", None)
    if v is None or v.data_ptr() != w.data_ptr() or v.device != w.device:
        v = w.detach().view(*w.shape, 1, 1)
        w._conv_view = v
    return v


class Upsample(nn.Module):
    def __init__(self, in_channels, with_conv):
        super().__init__()
        self.with_conv = with_conv
        if with_conv:
            self.conv = nn.Conv2d(in_channels, in_channels, kernel_size=3, stride=1, padding=1)

    def run(self, x):
        if not self.with_conv:
            raise NotImplementedError("open_muse_b200.VQGANModel: resample_with_conv=False is not supported")
        return ops.conv2d(x, self.conv.weight, bias=self.conv.bias, upsample2x=True)


class Downsample(nn.Module):
    def __init__(self, in_channels, with_conv):
        super().__init__()
        self.with_conv = with_conv
        if with_conv:
            self.conv = nn.Conv2d(in_channels, in_channels, kernel_size=3, stride=2, padding=0)

    def run(self, x):
        if not self.with_conv:
            return ops.avg_pool2x2(x)
        return ops.conv2d_down(x, self.conv.weight, bias=self.conv.bias)


class ResnetBlock(nn.Module):
    def __init__(self, in_channels, out_channels=None, use_conv_shortcut=False, dropout_prob=0.0, norm=_group_norm):
        super().__init__()
        self.in_channels = in_channels
        self.out_channels_ = in_channels if out_channels is None else out_channels
        self.use_conv_shortcut = use_conv_shortcut
        self.norm1 = norm(in_channels)
        self.conv1 = nn.Conv2d(in_channels, self.out_channels_, kernel_size=3, stride=1, padding=1)
        self.norm2 = norm(self.out_channels_)
        self.dropout = nn.Dropout(dropout_prob)
        self.conv2 = nn.Conv2d(self.out_channels_, self.out_channels_, kernel_size=3, stride=(1, 1), padding=1)
        if self.in_channels != self.out_channels_:
            if use_conv_shortcut:
                self.conv_shortcut = nn.Conv2d(in_channels, self.out_channels_, kernel_size=3, stride=1, padding=1)
            else:
                self.nin_shortcut = nn.Conv2d(in_channels, self.out_channels_, kernel_size=1, stride=1, padding=0)

    def run(self, x, zq=None):
        h = ops.conv2d(x, self.conv1.weight, bias=self.conv1.bias, **_norm(self.norm1, zq))
        res = x
        if self.in_channels != self.out_channels_:
            sc = self.conv_shortcut if self.use_conv_shortcut else self.nin_shortcut
            res = ops.conv2d(x, sc.weight, bias=sc.bias)
        return ops.conv2d(h, self.conv2.weight, bias=self.conv2.bias, residual=res, **_norm(self.norm2, zq))


class AttnBlock(nn.Module):
    def __init__(self, in_channels, norm=_group_norm, linear=False):
        super().__init__()
        self.in_channels = in_channels
        if linear:  # MoVQ: nn.Linear(C, C) projections over the tokens, the same products as 1x1 convolutions
            conv = partial(nn.Linear, in_channels, in_channels)
        else:
            conv = partial(nn.Conv2d, in_channels, in_channels, kernel_size=1, stride=1, padding=0)
        self.norm = norm(in_channels)
        self.q, self.k, self.v = conv(), conv(), conv()
        self.proj_out = conv()

    def run(self, x, zq=None):
        B, hh, ww, C = x.shape
        a = _norm(self.norm, zq, silu=0)
        n = ops.groupnorm_silu(x, *a.pop("gn"), **a)
        q = ops.conv2d(n, _conv1x1(self.q.weight), bias=self.q.bias)
        k = ops.conv2d(n, _conv1x1(self.k.weight), bias=self.k.bias)
        v = ops.conv2d(n, _conv1x1(self.v.weight), bias=self.v.bias)
        a = ops.attention_single_head(q.view(-1, C), k.view(-1, C), v.view(-1, C), B, hh, ww).view(B, hh, ww, C)
        return ops.conv2d(a, _conv1x1(self.proj_out.weight), bias=self.proj_out.bias, residual=x)


class UpsamplingBlock(nn.Module):
    def __init__(self, config, curr_res, block_idx, norm=_group_norm, linear=False):
        super().__init__()
        self.block_idx = block_idx
        if block_idx == config.num_resolutions - 1:
            block_in = config.hidden_channels * config.channel_mult[-1]
        else:
            block_in = config.hidden_channels * config.channel_mult[block_idx + 1]
        block_out = config.hidden_channels * config.channel_mult[block_idx]
        res_blocks, attn_blocks = [], []
        for _ in range(config.num_res_blocks + 1):  # creation order interleaved like the reference (seeded init)
            res_blocks.append(ResnetBlock(block_in, block_out, dropout_prob=config.dropout, norm=norm))
            block_in = block_out
            if curr_res in config.attn_resolutions:
                attn_blocks.append(AttnBlock(block_in, norm=norm, linear=linear))
        self.block = nn.ModuleList(res_blocks)
        self.attn = nn.ModuleList(attn_blocks)
        self.upsample = Upsample(block_in, config.resample_with_conv) if block_idx != 0 else None

    def run(self, x, zq=None):
        for i, blk in enumerate(self.block):
            x = blk.run(x, zq)
            if len(self.attn) > 1:  # (sic, :211)
                x = self.attn[i].run(x, zq)
        return self.upsample.run(x) if self.upsample is not None else x


class DownsamplingBlock(nn.Module):
    def __init__(self, config, curr_res, block_idx, linear=False):
        super().__init__()
        in_mult = (1,) + tuple(config.channel_mult)
        block_in = config.hidden_channels * in_mult[block_idx]
        block_out = config.hidden_channels * config.channel_mult[block_idx]
        res_blocks, attn_blocks = nn.ModuleList(), nn.ModuleList()
        for _ in range(config.num_res_blocks):
            res_blocks.append(ResnetBlock(block_in, block_out, dropout_prob=config.dropout))
            block_in = block_out
            if curr_res in config.attn_resolutions:
                attn_blocks.append(AttnBlock(block_in, linear=linear))
        self.block = res_blocks
        self.attn = attn_blocks
        self.downsample = Downsample(block_in, config.resample_with_conv) if block_idx != config.num_resolutions - 1 else None

    def run(self, x):
        for i, blk in enumerate(self.block):
            x = blk.run(x)
            if len(self.attn) > 1:  # (sic, :250)
                x = self.attn[i].run(x)
        return self.downsample.run(x) if self.downsample is not None else x


class MidBlock(nn.Module):
    def __init__(self, config, in_channels, no_attn, dropout, norm=_group_norm, linear=False):
        super().__init__()
        self.no_attn = no_attn
        self.block_1 = ResnetBlock(in_channels, in_channels, dropout_prob=dropout, norm=norm)
        if not no_attn:
            self.attn_1 = AttnBlock(in_channels, norm=norm, linear=linear)
        self.block_2 = ResnetBlock(in_channels, in_channels, dropout_prob=dropout, norm=norm)

    def run(self, x, zq=None):
        x = self.block_1.run(x, zq)
        if not self.no_attn:
            x = self.attn_1.run(x, zq)
        return self.block_2.run(x, zq)


class Encoder(nn.Module):
    """linear: nn.Linear attention projections (MoVQ, whose configs have no no_attn_mid_block: the mid attention is always
    built)"""

    def __init__(self, config, linear=False):
        super().__init__()
        self.conv_in = nn.Conv2d(config.num_channels, config.hidden_channels, kernel_size=3, stride=1, padding=1)
        curr_res, blocks = config.resolution, []
        for i in range(config.num_resolutions):
            blocks.append(DownsamplingBlock(config, curr_res, block_idx=i, linear=linear))
            if i != config.num_resolutions - 1:
                curr_res //= 2
        self.down = nn.ModuleList(blocks)
        mid = config.hidden_channels * config.channel_mult[-1]
        self.mid = MidBlock(config, mid, getattr(config, "no_attn_mid_block", False), config.dropout, linear=linear)
        self.norm_out = nn.GroupNorm(num_channels=mid, **_GN)
        self.conv_out = nn.Conv2d(mid, config.z_channels, kernel_size=3, stride=1, padding=1)

    def run(self, pixels):
        h = ops.conv2d(pixels, self.conv_in.weight, bias=self.conv_in.bias)
        for blk in self.down:
            h = blk.run(h)
        h = self.mid.run(h)
        return ops.conv2d(h, self.conv_out.weight, bias=self.conv_out.bias, gn=_gn(self.norm_out))


class Decoder(nn.Module):
    """norm / linear: the MoVQ decoder (SpatialNorm norms, nn.Linear attention projections, mid attention always built),
    whose run() takes the latent zq every norm is modulated by"""

    def __init__(self, config, norm=_group_norm, linear=False):
        super().__init__()
        block_in = config.hidden_channels * config.channel_mult[config.num_resolutions - 1]
        curr_res = config.resolution // 2 ** (config.num_resolutions - 1)
        self.z_shape = (1, config.z_channels, curr_res, curr_res)
        self.conv_in = nn.Conv2d(config.z_channels, block_in, kernel_size=3, stride=1, padding=1)
        self.mid = MidBlock(config, block_in, getattr(config, "no_attn_mid_block", False), config.dropout, norm=norm,
                            linear=linear)
        ups = []
        for i in reversed(range(config.num_resolutions)):
            ups.append(UpsamplingBlock(config, curr_res, block_idx=i, norm=norm, linear=linear))
            if i != 0:
                curr_res *= 2
        self.up = nn.ModuleList(list(reversed(ups)))
        block_out = config.hidden_channels * config.channel_mult[0]
        self.norm_out = norm(block_out)
        self.conv_out = nn.Conv2d(block_out, config.num_channels, kernel_size=3, stride=1, padding=1)

    def run(self, z, zq=None):
        h = ops.conv2d(z, self.conv_in.weight, bias=self.conv_in.bias)
        h = self.mid.run(h, zq)
        for blk in reversed(self.up):
            h = blk.run(h, zq)
        return ops.conv2d(h, self.conv_out.weight, bias=self.conv_out.bias, **_norm(self.norm_out, zq))


class VectorQuantizer(nn.Module):
    def __init__(self, num_embeddings, embedding_dim, commitment_cost):
        super().__init__()
        self.num_embeddings, self.embedding_dim, self.commitment_cost = num_embeddings, embedding_dim, commitment_cost
        self.embedding = nn.Embedding(num_embeddings, embedding_dim)
        self.embedding.weight.data.uniform_(-1.0 / num_embeddings, 1.0 / num_embeddings)

    def get_code_nhwc(self, z_nhwc):
        b = z_nhwc.shape[0]
        return ops.vq_argmin(z_nhwc.reshape(-1, self.embedding_dim), self.embedding.weight.float()).view(b, -1)

    def get_code(self, z_nchw):
        return self.get_code_nhwc(ops.to_nhwc(z_nchw.float().contiguous()))

    def get_codebook_entry(self, indices):
        b, t = indices.shape
        s = int(math.sqrt(t))
        return ops.vq_lookup_nchw(indices.contiguous(), self.embedding.weight.float()).view(b, -1, s, s)

    def get_soft_code_nhwc(self, z_nhwc, temp=1.0, stochastic=False, generator=None):
        b = z_nhwc.shape[0]
        z = z_nhwc.reshape(-1, self.embedding_dim)
        q = None
        if stochastic:
            q = torch.empty(z.shape[0], self.num_embeddings, dtype=torch.float32, device=z.device).exponential_(generator=generator)
        soft, ids = ops.vq_soft_code(z, self.embedding.weight.float(), temp, q)
        return soft.view(b, -1, self.num_embeddings), ids.view(b, -1)


class VQGANModel(ModelMixin, ConfigMixin):
    @register_to_config
    def __init__(
        self,
        resolution: int = 256,
        num_channels: int = 3,
        hidden_channels: int = 128,
        channel_mult: Tuple = (1, 1, 2, 2, 4),
        num_res_blocks: int = 2,
        attn_resolutions: int = (16,),
        no_attn_mid_block: bool = False,
        z_channels: int = 256,
        num_embeddings: int = 1024,
        quantized_embed_dim: int = 256,
        dropout: float = 0.0,
        resample_with_conv: bool = True,
        commitment_cost: float = 0.25,
    ):
        super().__init__()
        self.config.num_resolutions = len(channel_mult)
        self.config.reduction_factor = 2 ** (self.config.num_resolutions - 1)
        self.config.latent_size = resolution // self.config.reduction_factor
        self.encoder = Encoder(self.config)
        self.decoder = Decoder(self.config)
        self.quantize = VectorQuantizer(self.config.num_embeddings, self.config.quantized_embed_dim, self.config.commitment_cost)
        self.quant_conv = nn.Conv2d(self.config.z_channels, self.config.quantized_embed_dim, kernel_size=1)
        self.post_quant_conv = nn.Conv2d(self.config.quantized_embed_dim, self.config.z_channels, kernel_size=1)
        self.conv_precision = "bf16x3"

    def set_conv_precision(self, mode: str):
        """See MaskGitVQGAN.set_conv_precision: "bf16x3" (fp32-faithful, default) or "bf16" (single pass; the AttnBlock
        attention products stay fp32-faithful)."""
        with ops.conv_precision(mode):
            pass
        self.conv_precision = mode
        return self

    def _encode_nhwc(self, pixel_values):
        if not pixel_values.is_cuda:
            raise RuntimeError("open_muse_b200.VQGANModel runs on CUDA (sm_90a) only; move inputs to the GPU")
        with ops.conv_precision(self.conv_precision):
            h = self.encoder.run(ops.to_nhwc(pixel_values.float().contiguous()))
            return ops.conv2d(h, self.quant_conv.weight, bias=self.quant_conv.bias)

    def _quantize_nhwc(self, z_nhwc, return_loss):
        ids = self.quantize.get_code_nhwc(z_nhwc)
        z_q = self.quantize.get_codebook_entry(ids)
        loss = None
        if return_loss:  # value only (the tokenizer is not trained on this path)
            loss = torch.mean((z_q - ops.to_nchw(z_nhwc)) ** 2) * (1.0 + self.config.commitment_cost)
        return z_q, ids, loss

    @torch.no_grad()
    def encode(self, pixel_values, return_loss=False):
        z_q, ids, loss = self._quantize_nhwc(self._encode_nhwc(pixel_values), return_loss)
        return (z_q, ids, loss) if return_loss else (z_q, ids)

    @torch.no_grad()
    def decode(self, quantized_states):
        with ops.conv_precision(self.conv_precision):
            z = ops.to_nhwc(quantized_states.float().contiguous())
            h = ops.conv2d(z, self.post_quant_conv.weight, bias=self.post_quant_conv.bias)
            return ops.to_nchw(self.decoder.run(h))

    @torch.no_grad()
    def decode_code(self, codebook_indices):
        return self.decode(self.quantize.get_codebook_entry(codebook_indices))

    @torch.no_grad()
    def decode_code_uint8(self, codebook_indices):
        """ids -> display bytes uint8 [B, H, W, 3]: the decoder's NHWC output through the reference's clamp / truncation recipe
        on the device (pipeline_muse.py:245-252).  Extension used by PipelineMuse for output_type="pil"."""
        z_q = self.quantize.get_codebook_entry(codebook_indices)
        with ops.conv_precision(self.conv_precision):
            z = ops.to_nhwc(z_q.float().contiguous())
            h = ops.conv2d(z, self.post_quant_conv.weight, bias=self.post_quant_conv.bias)
            return ops.image_to_uint8(self.decoder.run(h))

    @torch.no_grad()
    def get_code(self, pixel_values):
        return self.quantize.get_code_nhwc(self._encode_nhwc(pixel_values))

    @torch.no_grad()
    def get_soft_code(self, pixel_values, temp=1.0, stochastic=False):
        return self.quantize.get_soft_code_nhwc(self._encode_nhwc(pixel_values), temp, stochastic)

    @torch.no_grad()
    def forward(self, pixel_values, return_loss=False):
        z_q, ids, loss = self._quantize_nhwc(self._encode_nhwc(pixel_values), return_loss)
        rec = self.decode(z_q)
        return (rec, z_q, ids, loss) if return_loss else (rec, z_q, ids)
