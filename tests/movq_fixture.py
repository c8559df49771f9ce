"""The MOVQ fixture (tests/golden/micro_movq.pt): two micro configs of the UNMODIFIED reference (muse/modeling_movq.py),
recorded on the CPU in fp32.
  * tc: 64 px, widths 64 / 64 / 128, attention at 16 x 16: every heavy layer takes the tensor-core route, and the
    decoder's SpatialNorms see the latent at ratios 1, 2 and 4.
  * f8: the class-default level structure (1, 2, 2, 4) at width 32, attention at 8 x 8: the narrow and 8 x 8 layers take
    the fp32 SIMT route, and the SpatialNorm ratios go up to 8.
Both have active attention blocks (2 per encoder level, 3 per decoder level, plus the mid blocks).  Test infrastructure
only.

With the reference init every GroupNorm affine is (1, 0) and the +-1/n codebook maps nearly every token onto a couple of
codes.  So ``micro_model`` builds the seeded model and then sets random GroupNorm affines (plain and spatial) from a second
seeded generator, and the recorder sets a codebook with the spread of z.  The weights are not stored: ``micro_model``
rebuilds them from the seeds with any class that has the reference's construction order (the reference's own class when
recording, ``open_muse_b200.MOVQ`` in the tests), and ``state_dict`` checks the rebuilt tensors against the signature
(fp64 sum and norm per tensor) of the reference's.  Only the codebook, the images and the outputs are stored.

Regenerate, in the build container only (the GPU box has no reference checkout):

    python tests/movq_fixture.py
"""
import os
import sys

import torch
from torch import nn

HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(HERE, "golden", "micro_movq.pt")

CONFIGS = {"tc": (dict(resolution=64, hidden_channels=64, channel_mult=(1, 1, 2), num_res_blocks=2, attn_resolutions=(16,),
                       num_embeddings=512), 80),
           "f8": (dict(resolution=64, hidden_channels=32, channel_mult=(1, 2, 2, 4), num_res_blocks=2,
                       attn_resolutions=(8,), num_embeddings=512), 90)}


def _signature(sd):
    return {k: (float(x.double().sum()), float(x.double().norm())) for k, x in sd.items()}


def micro_model(cls, name):
    """the seeded model of config `name` with random GroupNorm affines (the codebook is the reference init)"""
    cfg, seed = CONFIGS[name]
    torch.manual_seed(seed)
    m = cls(**cfg)
    init_sig = _signature(m.state_dict())
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for _, mod in m.named_modules():
            if isinstance(mod, nn.GroupNorm):
                mod.weight.copy_(1.0 + 0.3 * torch.randn(mod.num_channels, generator=g))
                mod.bias.copy_(0.3 * torch.randn(mod.num_channels, generator=g))
    return m.eval(), init_sig, g


def state_dict(cls, gold, name):
    """the recorded state dict of config `name`, rebuilt with `cls` and checked tensor by tensor against the signature"""
    m, _, _ = micro_model(cls, name)
    with torch.no_grad():
        m.quantize.embedding.weight.copy_(gold[name]["codebook"])
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    assert list(sd) == list(gold[name]["state_signature"])
    for k, (s, n) in _signature(sd).items():  # fp64 reductions: the summation order may differ between CPUs
        rs, rn = gold[name]["state_signature"][k]
        assert abs(s - rs) <= 1e-12 * max(1.0, abs(rs)) and abs(n - rn) <= 1e-12 * max(1.0, rn), k
    return sd


def record(muse_pkg):
    from muse.modeling_movq import MOVQ

    out = {}
    for name, (cfg, seed) in CONFIGS.items():
        m, init_sig, g = micro_model(MOVQ, name)
        img = torch.rand(2, 3, 64, 64, generator=g) * 2 - 1
        with torch.no_grad():
            z = m.quant_conv(m.encoder(img))
            m.quantize.embedding.weight.copy_(torch.randn(cfg["num_embeddings"], 4, generator=g) * z.std() + z.mean())
            z_q, ids = m.encode(img)
            d = m.quantize.compute_distances(z.permute(0, 2, 3, 1).contiguous())
            top2 = d.topk(2, dim=1, largest=False).values
            dec = m.decode_code(ids)
            fwd, fwd_ids = m(img)
        assert torch.equal(fwd_ids, ids)
        margin = top2[:, 1] - top2[:, 0]
        print(f"micro movq {name}: tokens {margin.numel()}, distinct ids {ids.unique().numel()}, "
              f"margin > 1e-3: {int((margin > 1e-3).sum())}")
        out[name] = dict(config=dict(m.config), seed=seed, init_signature=init_sig,
                         state_signature=_signature(m.state_dict()), codebook=m.quantize.embedding.weight.detach().clone(),
                         image=img, z=z, ids=ids, margin=margin, z_q=z_q, decode_code=dec, forward=fwd)
    torch.save(out, PATH)
    print(PATH, os.path.getsize(PATH) // 1024, "KiB")


if __name__ == "__main__":
    sys.path.insert(0, os.path.join(HERE, "golden"))
    from make_golden import import_reference

    record(import_reference())
