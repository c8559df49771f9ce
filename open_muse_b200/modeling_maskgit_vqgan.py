"""``MaskGitVQGAN`` (f16, 256 px -> 16x16 tokens) with the reference's surface (muse/modeling_maskgit_vqgan.py).

Same constructor / config keys / parameter names (``encoder.down.{l}.block.{b}.conv1.weight`` ...,
``quantize.embedding.weight``) and the same methods: ``encode``, ``decode``, ``decode_code``, ``get_code``,
``get_soft_code``, ``forward``.

Hot-path status (see DESIGN.md):
  * tokenise search (``VectorQuantizer``: distances + arg-min, :303-316,342-348) and detokenise lookup
    (``get_codebook_entry``, :318-324) run in libmuse_b200 kernels with a bit-exact contract (csrc/vq.cu).
  * the convolutional encoder / decoder (GroupNorm+SiLU+3x3 conv stacks) run as wgmma implicit-GEMM convolutions
    with fp32-level accuracy (operands carried as bf16 hi/lo planes, three products, fp32 accumulation:
    csrc/conv_tc.cu) fed by a fused GroupNorm+SiLU(+split) kernel; the 3-channel stem/head and odd geometries use the
    fp32 SIMT kernel (csrc/conv.cu).  fp32-faithful because token ids must match the fp32 reference (single-pass
    bf16/TF32 products flip ~2 % of ids, SURVEY H1).
The tokenizer is frozen in both training scripts (train_maskgit_imagenet.py:220-226), so only forward exists.
"""
from __future__ import annotations

import math
from typing import Tuple

import torch
import torch.nn.functional as F
from torch import nn

from . import ops
from .modeling_utils import ConfigMixin, ModelMixin, register_to_config


class Conv2dSame(nn.Conv2d):
    """Parameter container for a stride-1 'same' convolution (reference :33-45)."""


class ResnetBlock(nn.Module):
    def __init__(self, in_channels, out_channels=None, dropout_prob=0.0):
        super().__init__()
        self.in_channels = in_channels
        self.out_channels_ = in_channels if out_channels is None else out_channels
        self.norm1 = nn.GroupNorm(32, in_channels, eps=1e-6, affine=True)
        self.conv1 = Conv2dSame(in_channels, self.out_channels_, kernel_size=3, bias=False)
        self.norm2 = nn.GroupNorm(32, self.out_channels_, eps=1e-6, affine=True)
        self.dropout = nn.Dropout(dropout_prob)
        self.conv2 = Conv2dSame(self.out_channels_, self.out_channels_, kernel_size=3, bias=False)
        if in_channels != self.out_channels_:
            self.nin_shortcut = Conv2dSame(self.out_channels_, self.out_channels_, kernel_size=1, bias=False)

    def run(self, x):
        h = ops.conv2d(x, self.conv1.weight, gn=(self.norm1.weight, self.norm1.bias, 32, 1e-6))
        gn2 = (self.norm2.weight, self.norm2.bias, 32, 1e-6)
        if self.in_channels != self.out_channels_:
            h = ops.conv2d(h, self.conv2.weight, gn=gn2)
            # quirk Q8 (:82-85): shortcut of the post-conv2 activation, block input dropped
            return ops.conv2d(h, self.nin_shortcut.weight, residual=h)
        return ops.conv2d(h, self.conv2.weight, residual=x, gn=gn2)


class DownsamplingBlock(nn.Module):
    def __init__(self, config, block_idx):
        super().__init__()
        mult = (1,) + tuple(config.channel_mult)
        c_in = config.hidden_channels * mult[block_idx]
        c_out = config.hidden_channels * config.channel_mult[block_idx]
        blocks = nn.ModuleList()
        for _ in range(config.num_res_blocks):
            blocks.append(ResnetBlock(c_in, c_out, dropout_prob=config.dropout))
            c_in = c_out
        self.block = blocks
        self.downsample = block_idx != config.num_resolutions - 1

    def run(self, x):
        for b in self.block:
            x = b.run(x)
        return ops.avg_pool2x2(x) if self.downsample else x


class UpsamplingBlock(nn.Module):
    def __init__(self, config, block_idx):
        super().__init__()
        if block_idx == config.num_resolutions - 1:
            c_in = config.hidden_channels * config.channel_mult[-1]
        else:
            c_in = config.hidden_channels * config.channel_mult[block_idx + 1]
        c_out = config.hidden_channels * config.channel_mult[block_idx]
        blocks = []
        for _ in range(config.num_res_blocks):
            blocks.append(ResnetBlock(c_in, c_out, dropout_prob=config.dropout))
            c_in = c_out
        self.block = nn.ModuleList(blocks)
        self.add_upsample = block_idx != 0
        if self.add_upsample:
            self.upsample_conv = Conv2dSame(c_out, c_out, kernel_size=3)

    def run(self, x):
        for b in self.block:
            x = b.run(x)
        if self.add_upsample:  # nearest x2 folded into the convolution's input gather
            x = ops.conv2d(x, self.upsample_conv.weight, bias=self.upsample_conv.bias, upsample2x=True)
        return x


class Encoder(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.conv_in = Conv2dSame(config.num_channels, config.hidden_channels, kernel_size=3, bias=False)
        self.down = nn.ModuleList([DownsamplingBlock(config, i) for i in range(config.num_resolutions)])
        mid = config.hidden_channels * config.channel_mult[-1]
        self.mid = nn.ModuleList([ResnetBlock(mid, mid, dropout_prob=config.dropout) for _ in range(config.num_res_blocks)])
        self.norm_out = nn.GroupNorm(32, mid, eps=1e-6, affine=True)
        self.conv_out = Conv2dSame(mid, config.z_channels, kernel_size=1)

    def run(self, pixels):
        h = ops.conv2d(pixels, self.conv_in.weight)
        for blk in self.down:
            h = blk.run(h)
        for blk in self.mid:
            h = blk.run(h)
        return ops.conv2d(h, self.conv_out.weight, bias=self.conv_out.bias,
                          gn=(self.norm_out.weight, self.norm_out.bias, 32, 1e-6))


class Decoder(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        c = config.hidden_channels * config.channel_mult[config.num_resolutions - 1]
        res = config.resolution // 2 ** (config.num_resolutions - 1)
        self.z_shape = (1, config.z_channels, res, res)
        self.conv_in = Conv2dSame(config.z_channels, c, kernel_size=3)
        self.mid = nn.ModuleList([ResnetBlock(c, c, dropout_prob=config.dropout) for _ in range(config.num_res_blocks)])
        ups = [UpsamplingBlock(config, i) for i in reversed(range(config.num_resolutions))]
        self.up = nn.ModuleList(list(reversed(ups)))
        c0 = config.hidden_channels * config.channel_mult[0]
        self.norm_out = nn.GroupNorm(32, c0, eps=1e-6, affine=True)
        self.conv_out = Conv2dSame(c0, config.num_channels, kernel_size=3)

    def run(self, z):
        h = ops.conv2d(z, self.conv_in.weight, bias=self.conv_in.bias)
        for blk in self.mid:
            h = blk.run(h)
        for blk in reversed(self.up):
            h = blk.run(h)
        return ops.conv2d(h, self.conv_out.weight, bias=self.conv_out.bias,
                          gn=(self.norm_out.weight, self.norm_out.bias, 32, 1e-6))


class VectorQuantizer(nn.Module):
    def __init__(self, num_embeddings, embedding_dim, commitment_cost):
        super().__init__()
        self.num_embeddings, self.embedding_dim, self.commitment_cost = num_embeddings, embedding_dim, commitment_cost
        self.embedding = nn.Embedding(num_embeddings, embedding_dim)
        self.embedding.weight.data.uniform_(-1.0 / num_embeddings, 1.0 / num_embeddings)

    def get_code_nhwc(self, z_nhwc):
        """z in NHWC is already the [B*H*W, C] row layout of compute_distances (:305): no permute needed."""
        b = z_nhwc.shape[0]
        return ops.vq_argmin(z_nhwc.reshape(-1, self.embedding_dim), self.embedding.weight.float()).view(b, -1)

    def get_code(self, z_nchw):
        return self.get_code_nhwc(ops.to_nhwc(z_nchw.float().contiguous()))

    def get_codebook_entry(self, indices):
        b, t = indices.shape
        s = int(math.sqrt(t))
        return ops.vq_lookup_nchw(indices.contiguous(), self.embedding.weight.float()).view(b, -1, s, s)

    def forward(self, z_nchw, return_loss=False):
        ids = self.get_code(z_nchw)
        z_q = self.get_codebook_entry(ids).view_as(z_nchw)
        loss = None
        if return_loss:  # training of the tokenizer itself is out of scope; value provided for API parity
            loss = torch.mean((z_q - z_nchw) ** 2) * (1.0 + self.commitment_cost)
        return z_q, ids, loss

    def quantize_nhwc(self, z_nhwc, return_loss=False):
        ids = self.get_code_nhwc(z_nhwc)
        z_q = self.get_codebook_entry(ids)
        loss = None
        if return_loss:
            loss = torch.mean((z_q - ops.to_nchw(z_nhwc)) ** 2) * (1.0 + self.commitment_cost)
        return z_q, ids, loss

    def get_soft_code_nhwc(self, z_nhwc, temp=1.0, stochastic=False, generator=None):
        """soft targets of train_maskgit_imagenet.py:101-117,364-367 (reference :327-340). stochastic=True draws the
        Exp(1) noise of torch.multinomial(soft, 1) with torch and takes argmax soft/q in the kernel."""
        b = z_nhwc.shape[0]
        z = z_nhwc.reshape(-1, self.embedding_dim)
        q = None
        if stochastic:
            q = torch.empty(z.shape[0], self.num_embeddings, dtype=torch.float32, device=z.device).exponential_(generator=generator)
        soft, ids = ops.vq_soft_code(z, self.embedding.weight.float(), temp, q)
        return soft.view(b, -1, self.num_embeddings), ids.view(b, -1)

    def get_soft_code(self, z_nchw, temp=1.0, stochastic=False):
        return self.get_soft_code_nhwc(ops.to_nhwc(z_nchw.float().contiguous()), temp, stochastic)


class MaskGitVQGAN(ModelMixin, ConfigMixin):
    @register_to_config
    def __init__(
        self,
        resolution: int = 256,
        num_channels: int = 3,
        hidden_channels: int = 128,
        channel_mult: Tuple = (1, 1, 2, 2, 4),
        num_res_blocks: int = 2,
        attn_resolutions: int = (16,),
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
        self.conv_precision = "bf16x3"

    def set_conv_precision(self, mode: str):
        """"bf16x3" (default): fp32-faithful tensor-core convolutions, the mode of the bit-exact token-id contract.
        "bf16": single-pass bf16 operands, ~2.5x faster tokenise / detokenise at the accuracy class the reference's own
        GPU path has (TF32 convolutions); ids differ from the exact ones only near arg-min ties."""
        with ops.conv_precision(mode):
            pass
        self.conv_precision = mode
        return self

    def _encode_nhwc(self, pixel_values):
        if not pixel_values.is_cuda:
            raise RuntimeError("open_muse_b200.MaskGitVQGAN runs on CUDA (sm_90a) only; move inputs to the GPU")
        with ops.conv_precision(self.conv_precision):
            return self.encoder.run(ops.to_nhwc(pixel_values.float().contiguous()))

    @torch.no_grad()
    def encode(self, pixel_values, return_loss=False):
        z_q, ids, loss = self.quantize.quantize_nhwc(self._encode_nhwc(pixel_values), return_loss)
        return (z_q, ids, loss) if return_loss else (z_q, ids)

    @torch.no_grad()
    def decode(self, quantized_states):
        with ops.conv_precision(self.conv_precision):
            return ops.to_nchw(self.decoder.run(ops.to_nhwc(quantized_states.float().contiguous())))

    @torch.no_grad()
    def decode_code(self, codebook_indices):
        return self.decode(self.quantize.get_codebook_entry(codebook_indices))

    @torch.no_grad()
    def decode_code_uint8(self, codebook_indices):
        """ids -> display bytes uint8 [B, H, W, 3] (HWC per image, what PIL wants): the decoder's native NHWC output goes
        straight through the reference's clamp / truncation recipe on the device (pipeline_muse.py:245-252) -- no NCHW
        round trip, a 4x smaller device->host copy.  Extension used by PipelineMuse for output_type="pil"."""
        z_q = self.quantize.get_codebook_entry(codebook_indices)
        with ops.conv_precision(self.conv_precision):
            return ops.image_to_uint8(self.decoder.run(ops.to_nhwc(z_q.float().contiguous())))

    @torch.no_grad()
    def get_soft_code(self, pixel_values, temp=1.0, stochastic=False):
        return self.quantize.get_soft_code_nhwc(self._encode_nhwc(pixel_values), temp, stochastic)

    @torch.no_grad()
    def get_code(self, pixel_values):
        return self.quantize.get_code_nhwc(self._encode_nhwc(pixel_values))

    @torch.no_grad()
    def forward(self, pixel_values, return_loss=False):
        z_q, ids, loss = self.quantize.quantize_nhwc(self._encode_nhwc(pixel_values), return_loss)
        rec = self.decode(z_q)
        return (rec, z_q, ids, loss) if return_loss else (rec, z_q, ids)
