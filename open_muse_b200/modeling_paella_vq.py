"""``PaellaVQModel`` -- the Paella f4 / f8 tokenizer of the reference's ``paella_vq`` configs (muse/modeling_paella_vq.py),
behind the reference's surface: same constructor and config keys, parameter and buffer names (``in_block.1``,
``down_blocks.{i}``, ``vquantizer.codebook``, ``up_blocks.{i}``, ``out_block.0``, the BatchNorm running statistics), module
construction order (seeded initialisation identical) and methods ``encode / decode / decode_code / get_code / forward``.

Inference only (the reference's own TODO; the tokenizer is frozen in every script).  Everything runs in libmuse_b200, NHWC
fp32 between layers, on the tensor cores with fp32-faithful bf16x3 operands where the geometry has a TMA tiling and on the
fp32 SIMT kernels elsewhere (for example the 48- and 96-wide levels of f8):
  * in_block: PixelUnshuffle(2) + 1x1 conv as one 1x1 convolution over an im2col of the 2x2 blocks (ops.conv2d_unshuffle).
  * ResBlock (:112-145): LN1 statistics, one spatial pass (replication-padded depthwise 3x3 of LN1, + residual, LN2 written
    as the next operand), Linear + GELU (GELU epilogue), Linear + residual: four launches.  The six gammas are folded into
    the weights on the host and cached on the parameter versions.
  * Conv2d(4, 2, 1) and ConvTranspose2d(4, 2, 1): space-to-depth + 3x3, and four 2x2 parity convolutions.
  * The latent 1x1 conv + eval-mode BatchNorm2d: one convolution with the BatchNorm folded into its weight and bias.
  * quantiser: the bit-exact arg-min / lookup kernels of MaskGitVQGAN (D = 4 zero-filled to the kernel's k step).
  * out_block: 1x1 conv + PixelShuffle(2), the shuffle folded into the convolution's store.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F
from torch import nn

from . import ops
from .modeling_utils import ConfigMixin, ModelMixin, register_to_config

_EPS = 1e-6


def _versions(*ts):
    return tuple((t.data_ptr(), t._version, t.device) for t in ts)


class VectorQuantizer(nn.Module):
    def __init__(self, num_embeddings, embedding_dim, commitment_cost=0.25):
        super().__init__()
        self.num_embeddings = num_embeddings
        self.codebook_dim = embedding_dim
        self.commitment_cost = commitment_cost
        self.codebook = nn.Embedding(num_embeddings, embedding_dim)
        self.codebook.weight.data.uniform_(-1.0 / num_embeddings, 1.0 / num_embeddings)

    def _flat(self, z_nhwc):
        return z_nhwc.reshape(-1, self.codebook_dim)

    def get_code_nhwc(self, z_nhwc):
        return ops.vq_argmin(self._flat(z_nhwc), self.codebook.weight.float()).view(z_nhwc.shape[0], -1)

    def get_code(self, hidden_states):
        return self.get_code_nhwc(ops.to_nhwc(hidden_states.float().contiguous()))

    @torch.no_grad()
    def forward(self, hidden_states, return_loss=False):
        """(z_q NCHW, ids [B, tokens], loss): z_q holds exact codebook rows, loss the value only (inference)."""
        z = ops.to_nhwc(hidden_states.float().contiguous())
        ids = self.get_code_nhwc(z)
        b, h, w = z.shape[:3]
        z_q = ops.vq_lookup_nchw(ids, self.codebook.weight.float()).view(b, -1, h, w)
        loss = None
        if return_loss:
            loss = torch.mean((z_q - hidden_states) ** 2) * (1.0 + self.commitment_cost)
        return z_q, ids, loss

    def get_codebook_entry(self, indices):
        """(sic, :76-82) assumes a square token grid."""
        batch, num_tokens = indices.shape
        s = int(math.sqrt(num_tokens))
        return ops.vq_lookup_nchw(indices.contiguous(), self.codebook.weight.float()).view(batch, -1, s, s)

    @torch.no_grad()
    def get_soft_code(self, hidden_states, temp=1.0, stochastic=False):
        z = self._flat(ops.to_nhwc(hidden_states.float().contiguous()))
        q = None
        if stochastic:
            q = torch.empty(z.shape[0], self.num_embeddings, dtype=torch.float32, device=z.device).exponential_()
        soft, ids = ops.vq_soft_code(z, self.codebook.weight.float(), temp, q)
        b = hidden_states.shape[0]
        return soft.view(b, -1, self.num_embeddings), ids.view(b, -1)


class ResBlock(nn.Module):
    def __init__(self, c, c_hidden):
        super().__init__()
        if c % 8 != 0 or c > 1024:
            raise NotImplementedError(f"open_muse_b200.PaellaVQModel: ResBlock width {c} (needs a multiple of 8, <= 1024)")
        self.norm1 = nn.LayerNorm(c, elementwise_affine=False, eps=1e-6)
        self.depthwise = nn.Sequential(nn.ReplicationPad2d(1), nn.Conv2d(c, c, kernel_size=3, groups=c))
        self.norm2 = nn.LayerNorm(c, elementwise_affine=False, eps=1e-6)
        self.channelwise = nn.Sequential(nn.Linear(c, c_hidden), nn.GELU(), nn.Linear(c_hidden, c))
        self.gammas = nn.Parameter(torch.zeros(6), requires_grad=True)

        def _basic_init(module):
            if isinstance(module, nn.Linear) or isinstance(module, nn.Conv2d):
                torch.nn.init.xavier_uniform_(module.weight)
                if module.bias is not None:
                    nn.init.constant_(module.bias, 0)

        self.apply(_basic_init)

    def _folded(self):
        """x + g2 * dw(LN1(x) * (1 + g0) + g1) = x + dw'(LN1(x)) with dw' = g2 (1 + g0) w, bias g2 (b + g1 sum(w)) (every
        output sees all nine taps under replication padding); Lin1(LN2 * (1 + g3) + g4) = Lin1'(LN2) and g5 * Lin2 = Lin2'.
        Folded in fp64, cached on the parameter versions."""
        dw, l1, l2 = self.depthwise[1], self.channelwise[0], self.channelwise[2]
        params = (self.gammas, dw.weight, dw.bias, l1.weight, l1.bias, l2.weight, l2.bias)
        key = _versions(*params)
        hit = getattr(self, "_fold_cache", None)
        if hit is not None and hit[0] == key:
            return hit[1]
        g, w, b, w1, b1, w2, b2 = (t.detach().double() for t in params)
        c = w.shape[0]
        w9 = w.reshape(c, 9)
        wk = (g[2] * (1 + g[0]) * w9).t().contiguous()
        bias = g[2] * (b + g[1] * w9.sum(1))
        fw1 = ((1 + g[3]) * w1)[:, :, None, None]
        fb1 = b1 + g[4] * w1.sum(1)
        fw2 = (g[5] * w2)[:, :, None, None]
        fb2 = g[5] * b2
        out = tuple(t.float().contiguous() for t in (wk, bias, fw1, fb1, fw2, fb2))
        self._fold_cache = (key, out)
        return out

    def run(self, x):
        return ops.paella_resblock(x, *self._folded(), eps=self.norm1.eps)


def _latent_folded(seq):
    """Conv2d(c, c_latent, 1, bias=False) + eval-mode BatchNorm2d -> one 1x1 conv weight and bias (fp64 fold, cached)."""
    conv, bn = seq[0], seq[1]
    params = (conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var)
    key = _versions(*params)
    hit = getattr(seq, "_fold_cache", None)
    if hit is not None and hit[0] == key:
        return hit[1]
    w, gamma, beta, mean, var = (t.detach().double() for t in params)
    s = gamma / torch.sqrt(var + bn.eps)
    out = ((w * s[:, None, None, None]).float().contiguous(), (beta - mean * s).float().contiguous())
    seq._fold_cache = (key, out)
    return out


class PaellaVQModel(ModelMixin, ConfigMixin):
    @register_to_config
    def __init__(
        self, levels=2, bottleneck_blocks=12, c_hidden=384, c_latent=4, codebook_size=8192, scale_factor=0.3764
    ):
        super().__init__()
        self.c_latent = c_latent
        self.scale_factor = scale_factor
        c_levels = [c_hidden // (2**i) for i in reversed(range(levels))]

        self.in_block = nn.Sequential(nn.PixelUnshuffle(2), nn.Conv2d(3 * 4, c_levels[0], kernel_size=1))
        down_blocks = []
        for i in range(levels):
            if i > 0:
                down_blocks.append(nn.Conv2d(c_levels[i - 1], c_levels[i], kernel_size=4, stride=2, padding=1))
            block = ResBlock(c_levels[i], c_levels[i] * 4)
            down_blocks.append(block)
        down_blocks.append(
            nn.Sequential(
                nn.Conv2d(c_levels[-1], c_latent, kernel_size=1, bias=False),
                nn.BatchNorm2d(c_latent),
            )
        )
        self.down_blocks = nn.Sequential(*down_blocks)

        self.codebook_size = codebook_size
        self.vquantizer = VectorQuantizer(codebook_size, c_latent)

        up_blocks = [nn.Sequential(nn.Conv2d(c_latent, c_levels[-1], kernel_size=1))]
        for i in range(levels):
            for j in range(bottleneck_blocks if i == 0 else 1):
                block = ResBlock(c_levels[levels - 1 - i], c_levels[levels - 1 - i] * 4)
                up_blocks.append(block)
            if i < levels - 1:
                up_blocks.append(
                    nn.ConvTranspose2d(
                        c_levels[levels - 1 - i], c_levels[levels - 2 - i], kernel_size=4, stride=2, padding=1
                    )
                )
        self.up_blocks = nn.Sequential(*up_blocks)
        self.out_block = nn.Sequential(
            nn.Conv2d(c_levels[0], 3 * 4, kernel_size=1),
            nn.PixelShuffle(2),
        )
        self.conv_precision = "bf16x3"

    def set_conv_precision(self, mode: str):
        """"bf16x3" (fp32-faithful, default) or "bf16" (single tensor-core pass per product, bf16-operand accuracy)."""
        with ops.conv_precision(mode):
            pass
        self.conv_precision = mode
        return self

    # ---------------------------------------------------------------------------------------------- NHWC fp32 passes
    def _encode_nhwc(self, pixel_values):
        if not pixel_values.is_cuda:
            raise RuntimeError("open_muse_b200.PaellaVQModel runs on CUDA (sm_90a) only; move inputs to the GPU")
        latent = self.down_blocks[-1]
        if latent[1].training:
            raise NotImplementedError(
                "open_muse_b200.PaellaVQModel is inference only: call .eval() (in training mode the reference's BatchNorm "
                "would use batch statistics)")
        with ops.conv_precision(self.conv_precision):
            conv = self.in_block[1]
            h = ops.conv2d_unshuffle(ops.to_nhwc(pixel_values.float().contiguous()), conv.weight, conv.bias)
            for blk in self.down_blocks[:-1]:
                h = blk.run(h) if isinstance(blk, ResBlock) else ops.conv2d_s2p1(h, blk.weight, blk.bias)
            w, b = _latent_folded(latent)
            return ops.conv2d(h, w, bias=b)

    def _decode_nhwc(self, z_nhwc):
        with ops.conv_precision(self.conv_precision):
            conv = self.up_blocks[0][0]
            h = ops.conv2d(z_nhwc, conv.weight, bias=conv.bias)
            for blk in self.up_blocks[1:]:
                h = blk.run(h) if isinstance(blk, ResBlock) else ops.conv_transpose2d_s2(h, blk.weight, blk.bias)
            out = self.out_block[0]
            return ops.conv1x1_pixel_shuffle(h, out.weight, out.bias)

    def _quantize(self, z_nhwc):
        ids = self.vquantizer.get_code_nhwc(z_nhwc)
        b, h, w = z_nhwc.shape[:3]
        return ops.vq_lookup_nchw(ids, self.vquantizer.codebook.weight.float()).view(b, -1, h, w), ids

    # ---------------------------------------------------------------------------------------------- reference surface
    @torch.no_grad()
    def encode(self, x):
        """(z_q / scale_factor, ids, None): three values, as the reference returns (sic: two-value unpacking raises)."""
        z_q, ids = self._quantize(self._encode_nhwc(x))
        return z_q / self.scale_factor, ids, None

    @torch.no_grad()
    def decode(self, x):
        x = x * self.scale_factor
        return ops.to_nchw(self._decode_nhwc(ops.to_nhwc(x.float().contiguous())))

    @torch.no_grad()
    def decode_code(self, codebook_indices):
        """(sic) no scale_factor here, unlike decode()."""
        z = self.vquantizer.get_codebook_entry(codebook_indices)
        return ops.to_nchw(self._decode_nhwc(ops.to_nhwc(z.contiguous())))

    @torch.no_grad()
    def decode_code_uint8(self, codebook_indices):
        """ids -> display bytes uint8 [B, H, W, 3]: the decoder's NHWC output through the reference's clamp / truncation
        recipe on the device (pipeline_muse.py:245-252).  Extension used by PipelineMuse for output_type="pil"."""
        z = self.vquantizer.get_codebook_entry(codebook_indices)
        return ops.image_to_uint8(self._decode_nhwc(ops.to_nhwc(z.contiguous())))

    @torch.no_grad()
    def get_code(self, pixel_values):
        return self.vquantizer.get_code_nhwc(self._encode_nhwc(pixel_values))

    @torch.no_grad()
    def forward(self, x, quantize=False):
        qe = self.encode(x)[0]
        return self.decode(qe)
