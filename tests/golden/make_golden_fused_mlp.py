#!/usr/bin/env python
"""Generates micro_uvit_v2_fused_mlp.pt in this directory: MaskGiTUViT_v2 with use_fused_mlp=True (FusedGeLUFeedForward,
muse/modeling_transformer_v2.py:954-996) run by the UNMODIFIED reference on the CPU in fp32 (make_golden.py's method).
Run from the repo root, where the reference is mounted:

    python tests/golden/make_golden_fused_mlp.py

The fixture stores no weights: ``seeded_model`` rebuilds them from the seeds for any class with the reference's
constructor, and the fixture keeps per-tensor signatures of the reference's initial and final weights to pin that.  Nor
does it store whole gradients: ``signature`` keeps each gradient's norm, its first 8 elements and its projections on
four seeded Gaussian vectors, which ``signature_error`` turns into an estimate of a rel-L2 gradient error (a projection of
the error on a standard Gaussian vector has the error's norm as its rms).  This module is also imported by the tests for
``seeded_model``, the signatures and ``fused_mlp_standin``; only ``main`` needs the reference."""
import contextlib
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, "micro_uvit_v2_fused_mlp.pt")
# make_golden.MICRO_V2 with hidden 64 and one head; 176 = 11 * 16 is not a power of two and fits the FP8 mode's
# multiple-of-16 widths
CONFIG = dict(hidden_size=64, num_attention_heads=1, in_channels=64, block_out_channels=(64,), block_num_heads=1,
              num_res_blocks=1, num_hidden_layers=2, intermediate_size=176, vocab_size=72, codebook_size=64,
              encoder_hidden_size=32, cond_embed_dim=16, micro_cond_encode_dim=8, micro_cond_embed_dim=40,
              norm_type="rmsnorm", use_fused_mlp=True)
SEED, DRAW_SEED, GEN_SEED, PROJ_SEED = 70, 71, 72, 73


def tensor_signature(x):
    return float(x.double().sum()), float(x.double().norm())


def seeded_model(cls, **over):
    """torch.manual_seed(SEED); cls(**CONFIG), then the zero- / one-initialised tensors (adaLN mappers, GRN gamma / beta,
    mlm conv1, norm weights) re-drawn as make_golden.py's fixture (6) does, so that every branch contributes.  Returns
    (model, initial signatures, re-drawn names, the generator of the re-draw, which then draws the fixture's batch)."""
    torch.manual_seed(SEED)
    m = cls(**dict(CONFIG, **over))
    init_sig = {k: tensor_signature(x) for k, x in m.state_dict().items()}
    redrawn = []
    g = torch.Generator().manual_seed(DRAW_SEED)
    with torch.no_grad():
        for k, x in m.state_dict().items():
            if "adaLN_modulation.mapper" in k or k.endswith("gamma") or k.endswith("beta") or k == "mlm_layer.conv1.weight":
                x.copy_(torch.randn(x.shape, generator=g) * 0.05)
                redrawn.append(k)
            elif k.endswith("norm.weight"):
                x.copy_(1.0 + 0.1 * torch.randn(x.shape, generator=g))
                redrawn.append(k)
    return m, init_sig, redrawn, g


def _directions(n):
    return torch.randn(n, 4, generator=torch.Generator().manual_seed(PROJ_SEED + n), dtype=torch.float64)


def signature(t):
    f = t.detach().double().cpu().flatten()
    return dict(norm=float(f.norm()), head=f[:8].clone(), proj=f @ _directions(f.numel()))


def signature_error(t, sig):
    """estimated rel-L2 error of t against the tensor sig was taken of: the largest of the norm difference and the four
    projections of the difference, over the reference's norm"""
    s = signature(t)
    d = max(abs(s["norm"] - sig["norm"]), float((s["proj"] - sig["proj"]).abs().max()))
    return d / max(sig["norm"], 1e-30)


@contextlib.contextmanager
def fused_mlp_standin():
    """Lets the unmodified reference run ``use_fused_mlp=True`` on a CPU box for the duration of the block, touching none
    of its files.  FusedGeLUFeedForward.forward (:963-996) calls flash_attn's ``fused_mlp_func``, which is not installed,
    and asks ``torch.cuda.get_device_capability`` unconditionally.  On an H100 it gets (9, 0) and passes
    ``heuristic=-1``, for which flash_attn's FusedMLPFunc runs plain torch ops under the caller's autocast dtype: F.linear,
    F.gelu(approximate="tanh"), F.linear.  The stand-in restates that branch (read from flash_attn/ops/fused_dense.py, not
    run next to flash_attn itself).  The reference's ``muse.modeling_transformer_v2`` must be imported already."""
    import torch.nn.functional as F

    mt = sys.modules["muse.modeling_transformer_v2"]

    def fused_mlp_func(x, weight1, weight2, bias1=None, bias2=None, activation="gelu_approx", save_pre_act=True,
                       return_residual=False, checkpoint_lvl=0, heuristic=0, process_group=None, sequence_parallel=True):
        assert heuristic == -1 and activation == "gelu_approx" and not return_residual and process_group is None
        if torch.is_autocast_enabled():
            dtype = torch.get_autocast_gpu_dtype()
            x, weight1, weight2 = [a.to(dtype=dtype) for a in (x, weight1, weight2)]
            bias1 = bias1.to(dtype=dtype) if bias1 is not None else None
            bias2 = bias2.to(dtype=dtype) if bias2 is not None else None
        return F.linear(F.gelu(F.linear(x, weight1, bias1), approximate="tanh"), weight2, bias2)

    saved = mt.fused_mlp_func, torch.cuda.get_device_capability
    mt.fused_mlp_func, torch.cuda.get_device_capability = fused_mlp_func, lambda device=None: (9, 0)
    try:
        yield
    finally:
        mt.fused_mlp_func, torch.cuda.get_device_capability = saved


def main():
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from tests.golden.make_golden import import_reference

    import_reference()
    from muse.modeling_transformer_v2 import MaskGiTUViT_v2

    torch.set_num_threads(4)
    with fused_mlp_standin():
        v2, init_sig, redrawn, g = seeded_model(MaskGiTUViT_v2)
        v2.train()
        ids = torch.randint(0, 64, (3, 16), generator=g)
        mask = torch.rand(3, 16, generator=g) < 0.6
        inp = torch.where(mask, 71, ids)
        lab = torch.where(mask, ids, -100)
        enc = torch.randn(3, 5, 32, generator=g)
        ce = torch.randn(3, 16, generator=g)
        mc = torch.tensor([[256.0, 256.0, 0.0, 0.0, 6.0], [512.0, 384.0, 10.0, 20.0, 5.5], [128.0, 256.0, 3.0, 0.0, 7.25]])
        logits, loss = v2(inp, enc, ce, mc, labels=lab, label_smoothing=0.1)
        loss.backward()
        grads = {n: signature(p.grad) for n, p in v2.named_parameters()}
        v2.zero_grad()
        lw = torch.rand(3, 16, generator=g)
        _, loss_w = v2(inp, enc, ce, mc, labels=lab, loss_weight=lw)
        loss_w.backward()
        grads_w = {n: signature(p.grad) for n, p in v2.named_parameters()}
        v2.eval()
        empty_e, empty_c = torch.randn(1, 5, 32, generator=g), torch.randn(1, 16, generator=g)
        with torch.no_grad():
            gen_ids = v2.generate2(enc, ce, mc[:1], empty_e, empty_c, temperature=(2.0, 0.0), timesteps=4,
                                   guidance_scale=3.0, seq_len=16, generator=torch.Generator().manual_seed(GEN_SEED))
    sd = v2.state_dict()
    assert not any("wi_1" in k for k in sd) and any(k.endswith("ffn.wi_0.weight") for k in sd)
    torch.save(dict(config=CONFIG, init_signature=init_sig, redrawn=redrawn,
                    state_signature={k: tensor_signature(x) for k, x in sd.items()}, input_ids=inp, labels=lab,
                    encoder_hidden_states=enc, cond_embeds=ce, micro_conds=mc, logits=logits.detach(), loss=loss.detach(),
                    grads=grads, loss_weight=lw, loss_weighted=loss_w.detach(), grads_weighted=grads_w,
                    empty_embeds=empty_e, empty_cond_embeds=empty_c, gen_seed=GEN_SEED, gen_ids=gen_ids.clone()), FIXTURE)
    print("micro uvit v2 fused mlp: loss", float(loss.detach()), "weighted", float(loss_w.detach()),
          "logits std", float(logits.detach().std()), os.path.getsize(FIXTURE) // 1024, "KiB")


if __name__ == "__main__":
    main()
