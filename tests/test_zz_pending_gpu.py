"""GPU tests of compositions whose parts are validated elsewhere:

  * ``use_conv_in_out=True`` (ConvEmbed / ConvMlmLayer, reference muse/modeling_transformer.py:988-1080) against the unmodified
    reference's fp32 outputs in tests/golden/micro_conv_transformer.pt;
  * the UNMODIFIED training/train_muse.py through the real kernels;
  * MaskGiTUViT_v2 at head_dim 48 (the attention kernels are validated at that width through MaskGitTransformer).

Their host side is also checked numerically on the CPU (tests/test_v1_numeric_cpu.py::test_conv_in_out_*: logits 1e-7, every
gradient < 2e-4 of the reference; tests/test_train_muse_script_cpu.py: the script trains on the kernels' torch restatements)
and every kernel they launch is covered by tests/test_kernels_gpu.py / test_uvit_v2_gpu.py."""
import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]

DEV = "cuda"


def _rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-20))


def test_conv_in_out_vs_reference(golden):
    from open_muse_b200.modeling_transformer import MaskGitTransformer

    g = golden("micro_conv_transformer.pt")
    m = MaskGitTransformer(**g["config"])
    m.load_state_dict(g["state_dict"])
    m.to(DEV).train()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        logits, loss = m(g["input_ids"].to(DEV), encoder_hidden_states=g["encoder_hidden_states"].to(DEV),
                         labels=g["labels"].to(DEV), label_smoothing=g["label_smoothing"])
    loss.backward()
    torch.cuda.synchronize()
    assert logits.shape == g["logits"].shape
    assert _rel(logits, g["logits"]) < 1e-2
    assert abs(float(loss) - float(g["loss"])) < 2e-3 * abs(float(g["loss"]))
    errs = {}
    for n, p in m.named_parameters():
        assert p.grad is not None and p.grad.shape == p.shape, n
        errs[n] = _rel(p.grad, g["grads"][n])
    # same rule as tests/test_model_gpu.py: only the ~1e-6 query / key gradients may sit above 6e-2 (bf16 noise of the recipe)
    bad = {n: e for n, e in errs.items() if e >= 6e-2 and not ("attention.query" in n or "attention.key" in n)}
    assert not bad and max(errs.values()) < 0.5, (bad, max(errs.values()))
    print("conv in/out on the GPU: logits", _rel(logits, g["logits"]), "worst gradient", max(errs.values()))
    m.eval()
    with torch.no_grad():
        ids = m.generate2(encoder_hidden_states=g["encoder_hidden_states"].to(DEV), timesteps=4, guidance_scale=2.0,
                          generator=torch.Generator(DEV).manual_seed(3))
    assert ids.shape == (2, 64) and int(ids.min()) >= 0 and int(ids.max()) < g["config"]["codebook_size"]


def test_reference_train_muse_script_trains_on_gpu(tmp_path, monkeypatch):
    """GPU twin of tests/test_train_muse_script_cpu.py: the UNMODIFIED training/train_muse.py through the real kernels (CLIP
    text encoder with projection, taming VQGAN tokenizer, MaskGiTUViT_v2 with pooled + micro conditioning, bf16 autocast,
    name-grouped AdamW, EMA, checkpoint rotation)."""
    import json
    import math
    import os

    from tests.train_script_harness import find_script, make_muse_config, run_script

    script = find_script("train_muse.py")
    if script is None:
        pytest.skip("reference training script not available (build() snapshots it into oracle/_ref)")
    monkeypatch.setenv("WANDB_MODE", "disabled")
    steps = 6
    cfg, out = make_muse_config(str(tmp_path), steps=steps, batch=8, mixed_precision="bf16", save_every=3, use_ema=True,
                                extra_experiment={"checkpoints_total_limit": 1})
    from open_muse_b200 import ops

    n0 = ops.launches()
    acc = run_script(script, cfg)
    assert ops.launches() - n0 > 100 * steps
    losses = [v["step_loss"] for v, s in acc.logged if "step_loss" in v]
    assert len(losses) == steps and all(math.isfinite(x) for x in losses)
    assert abs(losses[0] - math.log(64)) < 0.6 and losses[-1] < losses[0]
    cks = sorted(d for d in os.listdir(out) if d.startswith("checkpoint"))
    assert len(cks) == 1 and json.load(open(os.path.join(out, cks[0], "metadata.json")))["global_step"] == steps


def test_uvit_head_dim_48_vs_oracle():
    """MaskGiTUViT_v2 with head_dim 48 in the transformer layers and the block attentions (96 / 2, 48 / 1) against the oracle's
    fp32 forward / autograd: the attention kernels are validated at head_dim 48 through MaskGitTransformer, this composition
    (the U-ViT passing head width and 1 / sqrt(48)) has only run on the CPU restatements."""
    from open_muse_b200 import MaskGiTUViT_v2
    from oracle import transformer_v2_oracle as V2

    cfg = dict(hidden_size=96, num_attention_heads=2, in_channels=48, block_out_channels=(48,), block_num_heads=1,
               num_res_blocks=1, num_hidden_layers=2, intermediate_size=128, vocab_size=72, codebook_size=64,
               encoder_hidden_size=32, cond_embed_dim=16, micro_cond_encode_dim=8, micro_cond_embed_dim=40, norm_type="rmsnorm")
    torch.manual_seed(3)
    m = MaskGiTUViT_v2(**cfg)
    with torch.no_grad():
        for p in m.parameters():
            p.add_((0.1 if p.dim() == 1 else 0.02) * torch.randn_like(p))
    g = torch.Generator().manual_seed(4)
    ids, lab = torch.randint(0, 64, (2, 16), generator=g), torch.randint(0, 64, (2, 16), generator=g)
    enc, ce, mc = torch.randn(2, 5, 32, generator=g), torch.randn(2, 16, generator=g), torch.rand(2, 5, generator=g) * 100
    q = {k: v.detach().clone().requires_grad_(True) for k, v in m.state_dict().items()}
    ref_logits, ref_loss = V2.forward(q, dict(m.config), ids, enc, ce, mc, labels=lab, label_smoothing=0.1)
    ref_loss.backward()
    m.to(DEV).train()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        logits, loss = m(ids.to(DEV), enc.to(DEV), ce.to(DEV), mc.to(DEV), labels=lab.to(DEV), label_smoothing=0.1)
    loss.backward()
    torch.cuda.synchronize()
    assert _rel(logits, ref_logits) < 2e-2 and abs(float(loss) - float(ref_loss)) < 2e-3 * float(ref_loss)
    bad = {n: _rel(p.grad, q[n].grad) for n, p in m.named_parameters()
           if _rel(p.grad, q[n].grad) > 8e-2 and not (".query." in n or ".key." in n)}
    assert not bad, bad
