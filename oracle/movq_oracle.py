"""ORACLE (test infrastructure only): fp64 functional restatement of the MoVQ tokenizer ``MOVQ`` (muse/modeling_movq.py),
written from its behaviour and driven by a reference-named ``state_dict``.  Pinned against tests/golden/micro_movq.pt
(outputs of the unmodified reference)."""
from __future__ import annotations

import math
from typing import Dict

import torch
import torch.nn.functional as F

F64 = torch.float64


def _d(p):
    return {k: v.detach().to(F64) for k, v in p.items() if v.is_floating_point()}


def _conv(x, p, pre, stride=1, padding=1):
    return F.conv2d(x, p[pre + "weight"], p.get(pre + "bias"), stride=stride, padding=padding)


def _norm(x, p, pre, zq):
    """nn.GroupNorm(32, eps 1e-6), or with zq the SpatialNorm: GN(x) * conv_y(up(zq)) + conv_b(up(zq)), up = nearest"""
    if zq is None:
        return F.group_norm(x, 32, p[pre + "weight"], p[pre + "bias"], 1e-6)
    z = F.interpolate(zq, size=x.shape[-2:], mode="nearest")
    n = F.group_norm(x, 32, p[pre + "norm_layer.weight"], p[pre + "norm_layer.bias"], 1e-6)
    return n * _conv(z, p, pre + "conv_y.", padding=0) + _conv(z, p, pre + "conv_b.", padding=0)


def resnet_block(x, p, pre, zq=None):
    h = _conv(F.silu(_norm(x, p, pre + "norm1.", zq)), p, pre + "conv1.")
    h = _conv(F.silu(_norm(h, p, pre + "norm2.", zq)), p, pre + "conv2.")
    if pre + "conv_shortcut.weight" in p:
        x = _conv(x, p, pre + "conv_shortcut.")
    elif pre + "nin_shortcut.weight" in p:
        x = _conv(x, p, pre + "nin_shortcut.", padding=0)
    return h + x


def attn_block(x, p, pre, zq=None):
    """one head of width C over the h*w tokens, nn.Linear projections"""
    b, c, hh, ww = x.shape
    n = _norm(x, p, pre + "norm.", zq).reshape(b, c, hh * ww).transpose(1, 2)
    lin = lambda t, name: F.linear(t, p[pre + name + ".weight"], p[pre + name + ".bias"])  # noqa: E731
    q, k, v = lin(n, "q"), lin(n, "k"), lin(n, "v")
    w = torch.softmax(q @ k.transpose(1, 2) / math.sqrt(c), dim=-1)
    return lin(w @ v, "proj_out").transpose(1, 2).reshape(b, c, hh, ww) + x


def _level(h, p, pre, n_blocks, zq=None):
    n_attn = len({k.split(".attn.")[1].split(".")[0] for k in p if k.startswith(pre + "attn.")})
    for i in range(n_blocks):
        h = resnet_block(h, p, f"{pre}block.{i}.", zq)
        if n_attn > 1:  # attention runs only where a level holds more than one block
            h = attn_block(h, p, f"{pre}attn.{i}.", zq)
    return h


def _mid(h, p, pre, zq=None):
    h = resnet_block(h, p, pre + "block_1.", zq)
    h = attn_block(h, p, pre + "attn_1.", zq)
    return resnet_block(h, p, pre + "block_2.", zq)


def encoder(sd: Dict[str, torch.Tensor], cfg: dict, pixels):
    """Encoder + quant_conv: z [B, D, h, w] in fp64"""
    p = _d(sd)
    n_res = len(cfg["channel_mult"])
    h = _conv(pixels.to(F64), p, "encoder.conv_in.")
    for lvl in range(n_res):
        h = _level(h, p, f"encoder.down.{lvl}.", cfg["num_res_blocks"])
        if lvl != n_res - 1:
            h = _conv(F.pad(h, (0, 1, 0, 1)), p, f"encoder.down.{lvl}.downsample.conv.", stride=2, padding=0)
    h = _mid(h, p, "encoder.mid.")
    h = _conv(F.silu(_norm(h, p, "encoder.norm_out.", None)), p, "encoder.conv_out.")
    return _conv(h, p, "quant_conv.", padding=0)


def distances(sd, z):
    """squared Euclidean distances [B*h*w, n_codes] (same arg-min as the reference's cdist)"""
    cb = sd["quantize.embedding.weight"].detach().to(F64)
    zf = z.to(F64).permute(0, 2, 3, 1).reshape(-1, cb.shape[1])
    return (zf[:, None, :] - cb[None].to(zf.device)).pow(2).sum(-1)


def decode(sd, cfg, quant):
    """post_quant_conv + MoVQDecoder, every norm modulated by quant (the codebook rows)"""
    p = _d(sd)
    zq = quant.to(F64)
    n_res = len(cfg["channel_mult"])
    h = _conv(_conv(zq, p, "post_quant_conv.", padding=0), p, "decoder.conv_in.")
    h = _mid(h, p, "decoder.mid.", zq)
    for lvl in reversed(range(n_res)):
        h = _level(h, p, f"decoder.up.{lvl}.", cfg["num_res_blocks"] + 1, zq)
        if lvl != 0:
            h = _conv(F.interpolate(h, scale_factor=2.0, mode="nearest"), p, f"decoder.up.{lvl}.upsample.conv.")
    return _conv(F.silu(_norm(h, p, "decoder.norm_out.", zq)), p, "decoder.conv_out.")


def decode_code(sd, cfg, ids):
    cb = sd["quantize.embedding.weight"].detach().to(F64)
    b, t = ids.shape
    s = int(math.sqrt(t))
    return decode(sd, cfg, cb.to(ids.device)[ids].reshape(b, s, s, -1).permute(0, 3, 1, 2))
