"""The PaellaVQModel fixture (tests/golden/micro_paella_vq.pt): an f4 and an f8 micro config of the UNMODIFIED reference
(muse/modeling_paella_vq.py), recorded on the CPU in fp32.  Test infrastructure only.

With the reference init every ResBlock is the identity (gammas = 0), the BatchNorm statistics are the defaults and the
+-1/8192 codebook makes nearly every token a near-tie.  So ``micro_model`` builds the seeded model and then sets random
non-zero gammas and random BatchNorm statistics and affine from a second seeded generator, and the recorder sets a codebook
with the spread of z.  The weights are not stored: ``micro_model`` rebuilds them from the seeds with any class that has the
reference's construction order (the reference's own class when recording, ``open_muse_b200.PaellaVQModel`` in the tests),
and ``state_dict`` checks the rebuilt tensors against the signature (fp64 sum and norm per tensor) of the reference's.
Only the codebook, the images and the outputs are stored.

Regenerate, in the build container only (the GPU box has no /root/reference):

    python tests/paella_fixture.py
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(HERE, "golden", "micro_paella_vq.pt")

CONFIGS = {"f4": (dict(levels=2, c_hidden=128, bottleneck_blocks=2, codebook_size=512), 60),
           "f8": (dict(levels=3, c_hidden=192, bottleneck_blocks=1, codebook_size=512), 70)}


def _signature(sd):
    return {k: (float(x.double().sum()), float(x.double().norm())) for k, x in sd.items()}


def micro_model(cls, name):
    """the seeded model of config `name` with its gammas and BatchNorm set (the codebook is the reference init)"""
    cfg, seed = CONFIGS[name]
    torch.manual_seed(seed)
    m = cls(**cfg)
    init_sig = _signature(m.state_dict())
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for k, prm in m.named_parameters():
            if k.endswith("gammas"):
                prm.copy_(torch.randn(6, generator=g) * 0.5)
        bn = m.down_blocks[-1][1]
        bn.running_mean.copy_(torch.randn(bn.num_features, generator=g) * 0.2)
        bn.running_var.copy_(torch.rand(bn.num_features, generator=g) + 0.5)
        bn.weight.copy_(1.0 + 0.3 * torch.randn(bn.num_features, generator=g))
        bn.bias.copy_(0.3 * torch.randn(bn.num_features, generator=g))
        bn.num_batches_tracked.fill_(123)
    return m.eval(), init_sig, g


def state_dict(cls, gold, name):
    """the recorded state dict of config `name`, rebuilt with `cls` and checked tensor by tensor against the signature"""
    m, _, _ = micro_model(cls, name)
    with torch.no_grad():
        m.vquantizer.codebook.weight.copy_(gold[name]["codebook"])
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    assert list(sd) == list(gold[name]["state_signature"])
    for k, (s, n) in _signature(sd).items():  # fp64 reductions: the summation order may differ between CPUs
        rs, rn = gold[name]["state_signature"][k]
        assert abs(s - rs) <= 1e-12 * max(1.0, abs(rs)) and abs(n - rn) <= 1e-12 * max(1.0, rn), k
    return sd


def record(muse_pkg):
    from muse.modeling_paella_vq import PaellaVQModel

    out = {}
    for name, (cfg, seed) in CONFIGS.items():
        m, init_sig, g = micro_model(PaellaVQModel, name)
        img = torch.rand(2, 3, 64, 64, generator=g) * 2 - 1
        with torch.no_grad():
            z = m.down_blocks(m.in_block(img))
            m.vquantizer.codebook.weight.copy_(torch.randn(cfg["codebook_size"], 4, generator=g) * z.std() + z.mean())
            z_q, ids, loss = m.encode(img)
            d = m.vquantizer.compute_distances(z.permute(0, 2, 3, 1).contiguous())
            top2 = d.topk(2, dim=1, largest=False).values
            dec = m.decode_code(ids)
            fwd = m(img)
        assert loss is None
        margin = top2[:, 1] - top2[:, 0]
        print(f"micro paella vq {name}: tokens {margin.numel()}, margin > 1e-4: {int((margin > 1e-4).sum())}")
        out[name] = dict(config=dict(m.config), seed=seed, init_signature=init_sig,
                         state_signature=_signature(m.state_dict()), codebook=m.vquantizer.codebook.weight.detach().clone(),
                         image=img, z=z, ids=ids, margin=margin, z_q=z_q, decode_code=dec, forward=fwd)
    torch.save(out, PATH)
    print(PATH, os.path.getsize(PATH) // 1024, "KiB")


if __name__ == "__main__":
    sys.path.insert(0, os.path.join(HERE, "golden"))
    from make_golden import import_reference

    record(import_reference())
