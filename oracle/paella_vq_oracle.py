"""ORACLE (test infrastructure only): fp64 functional restatement of ``PaellaVQModel`` (muse/modeling_paella_vq.py), driven by
a reference-named ``state_dict`` and the model's config dict.  The GPU tests use it as the fp64 reference of the encoder,
the quantiser distances and the decoder; it is pinned against tests/golden/micro_paella_vq.pt (outputs of the unmodified
reference) on the CPU."""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn.functional as F

D64 = torch.float64


def _levels(cfg):
    return [cfg["c_hidden"] // (2**i) for i in reversed(range(cfg["levels"]))]


def _ln(x):
    """LayerNorm over channels (NCHW dim 1), no affine, eps 1e-6"""
    mean = x.mean(1, keepdim=True)
    var = x.var(1, unbiased=False, keepdim=True)
    return (x - mean) / torch.sqrt(var + 1e-6)


def resblock(x, p, pre):
    """ResBlock.forward (:137-145)"""
    g = p[pre + "gammas"]
    c = x.shape[1]
    t = _ln(x) * (1 + g[0]) + g[1]
    t = F.conv2d(F.pad(t, (1, 1, 1, 1), mode="replicate"), p[pre + "depthwise.1.weight"], p[pre + "depthwise.1.bias"], groups=c)
    x = x + t * g[2]
    t = (_ln(x) * (1 + g[3]) + g[4]).permute(0, 2, 3, 1)
    t = F.linear(F.gelu(F.linear(t, p[pre + "channelwise.0.weight"], p[pre + "channelwise.0.bias"])),
                 p[pre + "channelwise.2.weight"], p[pre + "channelwise.2.bias"])
    return x + t.permute(0, 3, 1, 2) * g[5]


def _p64(sd):
    return {k: v.to(D64) if v.is_floating_point() else v for k, v in sd.items()}


def encoder(sd: Dict[str, torch.Tensor], cfg: dict, pixels):
    """in_block + down_blocks (eval-mode BatchNorm): pre-quantisation z, NCHW fp64"""
    p = _p64(sd)
    lv = _levels(cfg)
    h = F.conv2d(F.pixel_unshuffle(pixels.to(D64), 2), p["in_block.1.weight"], p["in_block.1.bias"])
    i = 0
    for lvl in range(len(lv)):
        if lvl > 0:
            h = F.conv2d(h, p[f"down_blocks.{i}.weight"], p[f"down_blocks.{i}.bias"], stride=2, padding=1)
            i += 1
        h = resblock(h, p, f"down_blocks.{i}.")
        i += 1
    h = F.conv2d(h, p[f"down_blocks.{i}.0.weight"])
    return F.batch_norm(h, p[f"down_blocks.{i}.1.running_mean"], p[f"down_blocks.{i}.1.running_var"],
                        p[f"down_blocks.{i}.1.weight"], p[f"down_blocks.{i}.1.bias"], False, 0.0, 1e-5)


def distances(sd, z_nchw):
    """squared euclidean distances [tokens, codes] in fp64 (cdist is their square root: same arg-min)"""
    cb = sd["vquantizer.codebook.weight"].to(D64)
    z = z_nchw.to(D64).permute(0, 2, 3, 1).reshape(-1, cb.shape[1])
    return (z[:, None, :] - cb[None]).pow(2).sum(-1)


def decoder(sd, cfg, z_nchw):
    """up_blocks + out_block (decode without the scale factor, i.e. decode_code's path)"""
    p = _p64(sd)
    lv = _levels(cfg)
    h = F.conv2d(z_nchw.to(D64), p["up_blocks.0.0.weight"], p["up_blocks.0.0.bias"])
    i = 1
    for lvl in range(len(lv)):
        for _ in range(cfg["bottleneck_blocks"] if lvl == 0 else 1):
            h = resblock(h, p, f"up_blocks.{i}.")
            i += 1
        if lvl < len(lv) - 1:
            h = F.conv_transpose2d(h, p[f"up_blocks.{i}.weight"], p[f"up_blocks.{i}.bias"], stride=2, padding=1)
            i += 1
    return F.pixel_shuffle(F.conv2d(h, p["out_block.0.weight"], p["out_block.0.bias"]), 2)


def decode_code(sd, cfg, ids):
    cb = sd["vquantizer.codebook.weight"].to(D64)
    b, t = ids.shape
    s = int(t ** 0.5)
    return decoder(sd, cfg, cb[ids].reshape(b, s, s, -1).permute(0, 3, 1, 2))
