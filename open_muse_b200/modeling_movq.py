"""``MOVQ`` -- the MoVQ f8 tokenizer of the reference's ``movq`` configs (muse/modeling_movq.py), behind the reference's
surface: same constructor and config keys, parameter names (``decoder.mid.block_1.norm1.norm_layer.weight``,
``...norm1.conv_y.weight``, ``encoder.mid.attn_1.q.weight`` as [C, C] Linear weights, ``quantize.embedding.weight``,
``quant_conv``, ``post_quant_conv``), construction order (seeded initialisation identical) and methods
``encode / decode / decode_code / get_code / forward``.

Inference only (the tokenizer is frozen in both training scripts).  It runs on the taming VQGAN's blocks
(modeling_taming_vqgan.py), NHWC fp32 between layers with fp32-faithful tensor-core convolutions:
  * encoder: the taming encoder with nn.Linear attention projections (the same products as the 1x1 convolutions) and the
    mid-block attention always present.
  * quantiser: the bit-exact arg-min / lookup kernels of MaskGitVQGAN; the arg-min of the reference's Euclidean cdist is
    the arg-min of the squared distance.
  * decoder: the taming decoder with every GroupNorm a SpatialNorm, GN(f) * conv_y(up(zq)) + conv_b(up(zq)) with zq the
    codebook rows (before post_quant_conv) and `up` the nearest resize to f's grid.  The modulation is computed per pixel
    inside the GroupNorm apply pass (ops.conv2d / ops.groupnorm_silu with spatial=...), so neither up(zq) nor the two
    modulation tensors are ever written.
"""
from __future__ import annotations

from functools import partial
from typing import Tuple

import torch
from torch import nn

from . import ops
from .modeling_taming_vqgan import Decoder, Encoder, VectorQuantizer as _TamingVectorQuantizer, _GN
from .modeling_utils import ConfigMixin, ModelMixin, register_to_config


class SpatialNorm(nn.Module):
    """GroupNorm(f) * conv_y(up(zq)) + conv_b(up(zq)) (muse/modeling_movq.py:21-49); run by the blocks that hold it."""

    def __init__(self, f_channels, zq_channels, norm_layer=nn.GroupNorm, freeze_norm_layer=False, add_conv=False,
                 **norm_layer_params):
        super().__init__()
        if add_conv:  # no MOVQ path enables it (Normalize passes add_conv=False)
            raise NotImplementedError("open_muse_b200.MOVQ: SpatialNorm(add_conv=True) is not supported")
        self.norm_layer = norm_layer(num_channels=f_channels, **norm_layer_params)
        if freeze_norm_layer:
            for p in self.norm_layer.parameters():
                p.requires_grad = False
        self.add_conv = add_conv
        self.conv_y = nn.Conv2d(zq_channels, f_channels, kernel_size=1, stride=1, padding=0)
        self.conv_b = nn.Conv2d(zq_channels, f_channels, kernel_size=1, stride=1, padding=0)


def _spatial_norm(zq_channels, channels):
    return SpatialNorm(channels, zq_channels, **_GN)


class VectorQuantizer(_TamingVectorQuantizer):
    def __init__(self, num_embeddings, embedding_dim, commitment_cost, legacy=True):
        super().__init__(num_embeddings, embedding_dim, commitment_cost)
        self.legacy = legacy

    def forward_nhwc(self, z_nhwc, return_loss=False):
        """(z_q NCHW, ids [B, tokens], loss): z_q holds exact codebook rows"""
        ids = self.get_code_nhwc(z_nhwc)
        b, h, w = z_nhwc.shape[:3]
        z_q = ops.vq_lookup_nchw(ids, self.embedding.weight.float()).view(b, -1, h, w)
        loss = None
        if return_loss:
            # (sic, :500-508) the loss reads self.beta, which the class never sets: AttributeError, as upstream
            loss = self.beta * torch.mean((z_q - ops.to_nchw(z_nhwc)) ** 2)
        return z_q, ids, loss

    @torch.no_grad()
    def forward(self, hidden_states, return_loss=False):
        return self.forward_nhwc(ops.to_nhwc(hidden_states.float().contiguous()), return_loss)

    def get_soft_code(self, hidden_states, temp=1.0, stochastic=False):
        """Not built: nothing in the reference calls it (MOVQ has no get_soft_code), and its softmax is over Euclidean
        cdist distances, which the arg-min kernels do not compute (they rank squared distances)."""
        raise NotImplementedError("open_muse_b200.MOVQ: quantize.get_soft_code is not supported (the reference model has "
                                  "no get_soft_code; use get_code)")

    get_soft_code_nhwc = get_soft_code


class MOVQ(ModelMixin, ConfigMixin):
    @register_to_config
    def __init__(
        self,
        resolution: int = 256,
        num_channels=3,
        out_channels=3,
        hidden_channels=128,
        channel_mult: Tuple = (1, 2, 2, 4),
        num_res_blocks=2,
        attn_resolutions=(32,),
        z_channels=4,
        double_z=False,
        num_embeddings=16384,
        quantized_embed_dim=4,
        dropout=0.0,
        resample_with_conv: bool = True,
        commitment_cost: float = 0.25,
    ):
        super().__init__()
        # (sic) out_channels and double_z are accepted and unused, as upstream
        self.config.num_resolutions = len(channel_mult)
        self.config.reduction_factor = 2 ** (self.config.num_resolutions - 1)
        self.config.latent_size = resolution // self.config.reduction_factor
        self.encoder = Encoder(self.config, linear=True)
        self.decoder = Decoder(self.config, norm=partial(_spatial_norm, quantized_embed_dim), linear=True)
        self.quantize = VectorQuantizer(num_embeddings, quantized_embed_dim, commitment_cost=commitment_cost)
        self.quant_conv = nn.Conv2d(z_channels, quantized_embed_dim, 1)
        self.post_quant_conv = nn.Conv2d(quantized_embed_dim, z_channels, 1)
        self.conv_precision = "bf16x3"

    def set_conv_precision(self, mode: str):
        """"bf16x3" (fp32-faithful, default) or "bf16" (single pass; the AttnBlock attention products stay
        fp32-faithful)."""
        with ops.conv_precision(mode):
            pass
        self.conv_precision = mode
        return self

    # ---------------------------------------------------------------------------------------------- NHWC fp32 passes
    def _encode_nhwc(self, pixel_values):
        if not pixel_values.is_cuda:
            raise RuntimeError("open_muse_b200.MOVQ runs on CUDA (sm_90a) only; move inputs to the GPU")
        with ops.conv_precision(self.conv_precision):
            h = self.encoder.run(ops.to_nhwc(pixel_values.float().contiguous()))
            return ops.conv2d(h, self.quant_conv.weight, bias=self.quant_conv.bias)

    def _decode_nhwc(self, quant):
        """quant: the codebook rows, NCHW -> decoded image NHWC; every norm of the decoder is modulated by quant itself"""
        with ops.conv_precision(self.conv_precision):
            zq = ops.to_nhwc(quant.float().contiguous())
            h = ops.conv2d(zq, self.post_quant_conv.weight, bias=self.post_quant_conv.bias)
            return self.decoder.run(h, zq)

    # ---------------------------------------------------------------------------------------------- reference surface
    @torch.no_grad()
    def encode(self, pixel_values, return_loss=False):
        """(z_q, ids): two values, unlike VQGANModel; return_loss=True raises AttributeError as upstream"""
        z_q, ids, loss = self.quantize.forward_nhwc(self._encode_nhwc(pixel_values), return_loss)
        return (z_q, ids, loss) if return_loss else (z_q, ids)

    @torch.no_grad()
    def decode(self, quant):
        return ops.to_nchw(self._decode_nhwc(quant))

    @torch.no_grad()
    def decode_code(self, codebook_indices):
        return self.decode(self.quantize.get_codebook_entry(codebook_indices))

    @torch.no_grad()
    def decode_code_uint8(self, codebook_indices):
        """ids -> display bytes uint8 [B, H, W, 3]: the decoder's NHWC output through the reference's clamp / truncation
        recipe on the device (pipeline_muse.py:245-252).  Extension used by PipelineMuse for output_type="pil"."""
        return ops.image_to_uint8(self._decode_nhwc(self.quantize.get_codebook_entry(codebook_indices)))

    @torch.no_grad()
    def get_code(self, pixel_values):
        return self.quantize.get_code_nhwc(self._encode_nhwc(pixel_values))

    @torch.no_grad()
    def forward(self, pixel_values, return_loss=False):
        """(reconstruction, ids): two values, unlike VQGANModel"""
        z_q, ids, loss = self.quantize.forward_nhwc(self._encode_nhwc(pixel_values), return_loss)
        rec = self.decode(z_q)
        return (rec, ids, loss) if return_loss else (rec, ids)
