"""GPU twin of tests/test_train_script_cpu.py: the UNMODIFIED reference training script (taken from oracle/_ref/training, the
git-ignored snapshot __graft_entry__.build() makes, or /root/reference when present) trains the drop-in MaskGitTransformer
on the GPU through the real kernels: frozen MaskGitVQGAN tokeniser (wgmma / SIMT convolutions + bit-exact arg-min) ->
masking -> bf16-autocast forward + fused CE -> backward -> clip -> AdamW -> checkpoints."""
import json
import math
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from tests.train_script_harness import find_script, make_config, run_script  # noqa: E402

SCRIPT = find_script()


@pytest.mark.skipif(SCRIPT is None, reason="reference training script not available (build() snapshots it into oracle/_ref)")
@pytest.mark.parametrize("soft_targets", [False, True])
def test_reference_training_script_trains_on_gpu(tmp_path, soft_targets, monkeypatch):
    monkeypatch.setenv("WANDB_MODE", "disabled")
    steps = 6
    cfg, out = make_config(str(tmp_path), steps=steps, batch=8, mixed_precision="bf16", soft_targets=soft_targets, save_every=3)
    from open_muse_b200 import ops

    n0 = ops.launches()
    acc = run_script(SCRIPT, cfg)
    assert ops.launches() - n0 > 100 * steps  # the step really ran through libmuse_b200
    losses = [v["step_loss"] for v, s in acc.logged if "step_loss" in v]
    assert len(losses) == steps and all(math.isfinite(x) for x in losses)
    assert abs(losses[0] - math.log(64 if soft_targets else 75)) < 0.5  # random init: ~uniform prediction
    assert losses[-1] < losses[0]                                        # lr 1e-3 AdamW moves it within 6 steps
    ev = [v["eval_loss"] for v, s in acc.logged if "eval_loss" in v]
    assert ev and math.isfinite(ev[-1])
    assert json.load(open(os.path.join(out, "checkpoint-3", "metadata.json"))) == {"global_step": 3}
    # the exported model loads back into the drop-in class and differs from a fresh init
    from open_muse_b200 import MaskGitTransformer

    m = MaskGitTransformer.from_pretrained(out)
    sd = torch.load(os.path.join(out, "checkpoint-3", "unwrapped_model", "pytorch_model.bin"), map_location="cpu")
    w = "transformer_layers.0.ffn.wi_0.weight"
    assert not torch.equal(m.state_dict()[w], sd[w]) and bool(torch.isfinite(m.state_dict()[w]).all())
    print(f"reference train script on GPU ({'soft' if soft_targets else 'hard'} targets): losses {[round(x, 4) for x in losses]}, "
          f"eval {ev[-1]:.4f}")
