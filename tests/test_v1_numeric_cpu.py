"""Host logic of MaskGitTransformer checked NUMERICALLY without a GPU: the product's own autograd Functions, packed-operand
table, gradient routing and generate2 loop run on the CPU with the C-ABI kernels replaced by torch restatements of their
contracts (tests/cpu_math_ops.py) and are compared with what the UNMODIFIED reference computed (tests/golden/*.pt, written
by tests/golden/make_golden.py from /root/reference).

exact mode (every "bf16" tensor carries fp32 values): logits, loss and EVERY parameter gradient must equal the reference's
fp32 results to ~1e-4 -- a gradient routed to the wrong parameter, a missing residual term or a wrong statistics row cannot
hide under bf16 noise as it could in the GPU tests' 1e-2 / 6e-2 tolerances.
recipe mode (bf16 where the kernels write bf16): the precision recipe of the hot path itself stays within the GPU tests'
tolerances on the same fixtures.
The kernels are NOT exercised here (tests/test_kernels_gpu.py, tests/test_model_gpu.py do that on the GPU)."""
import pytest
import torch

from open_muse_b200 import MaskGitTransformer
from tests import cpu_math_ops


def _rel(a, b):
    a, b = a.detach().float(), b.detach().float()
    return float((a - b).norm() / b.norm().clamp_min(1e-20))


def _run(g, exact, monkeypatch, **fwd):
    cpu_math_ops.install(monkeypatch, exact=exact)
    m = MaskGitTransformer(**g["config"])
    m.load_state_dict(g["state_dict"])
    m.train()
    logits, loss = m(**fwd)
    loss.backward()
    return m, logits, loss


def _inputs(g):
    if "batch" in g:
        return dict(input_ids=g["batch"]["input_ids"], labels=g["batch"]["labels"], label_smoothing=g.get("label_smoothing", 0.0))
    return dict(input_ids=g["input_ids"], labels=g["labels"], encoder_hidden_states=g["encoder_hidden_states"])


FIXTURES = ["micro_transformer.pt", "micro_t2i_transformer.pt", "micro_t2i_proj_transformer.pt"]


@pytest.mark.parametrize("name", FIXTURES)
def test_host_wiring_reproduces_the_reference_in_fp32(golden, monkeypatch, name):
    g = golden(name)
    m, logits, loss = _run(g, True, monkeypatch, **_inputs(g))
    assert logits.shape == g["logits"].shape
    assert _rel(logits, g["logits"]) < 2e-5
    assert abs(float(loss.detach()) - float(g["loss"])) < 2e-6 * abs(float(g["loss"])) + 1e-7
    assert set(n for n, _ in m.named_parameters()) == set(g["grads"])
    worst = 0.0
    for n, p in m.named_parameters():
        assert p.grad is not None and p.grad.dtype == torch.float32, n
        e = _rel(p.grad, g["grads"][n])
        worst = max(worst, e)
        assert e < 2e-4, (n, e)
    print(f"{name}: logits {_rel(logits, g['logits']):.2e}, worst gradient {worst:.2e}")


@pytest.mark.parametrize("name", FIXTURES)
def test_precision_recipe_on_the_cpu_stays_within_the_gpu_tolerances(golden, monkeypatch, name):
    """bf16 GEMM operands / activations, fp32 accumulation, residual stream, statistics and weight gradients -- the dtype of
    every tensor exactly as the kernels write it"""
    g = golden(name)
    m, logits, loss = _run(g, False, monkeypatch, **_inputs(g))
    assert _rel(logits, g["logits"]) < 1e-2
    assert abs(float(loss) - float(g["loss"])) < 2e-3 * abs(float(g["loss"]))
    above = []
    for n, p in m.named_parameters():
        e = _rel(p.grad, g["grads"][n])
        if e >= 6e-2:
            above.append((n, e))
    # the reference's own bf16-autocast recipe is this noisy on the ~1e-6 query / key gradients (tests/test_model_gpu.py)
    assert all("attention.query" in n or "attention.key" in n for n, _ in above) and len(above) <= 2, above


@pytest.mark.parametrize("name,stride", [("tiny_transformer.pt", (16, 25)), ("hd48_transformer.pt", (8, 16))])
def test_seeded_construction_and_wiring_at_config_widths(golden, monkeypatch, name, stride):
    """BASELINE config 1 and configs/imagenet.yaml widths (head_dim 48): seeded construction reproduces the reference's
    initial weights, and the host wiring its loss / logits / gradient signatures"""
    g = golden(name)
    cpu_math_ops.install(monkeypatch, exact=True)
    torch.manual_seed(g["seed"])
    m = MaskGitTransformer(**g["config"]).train()
    logits, loss = m(g["batch"]["input_ids"], labels=g["batch"]["labels"], label_smoothing=g.get("label_smoothing", 0.0))
    loss.backward()
    assert abs(float(loss) - float(g["loss"])) < 1e-5 * abs(float(g["loss"]))
    torch.testing.assert_close(logits[:, ::stride[0], ::stride[1]], g["logits_slice"], rtol=2e-4, atol=2e-5)
    grads = dict((n, p.grad) for n, p in m.named_parameters())
    for k, n in g["grad_norms"].items():
        torch.testing.assert_close(grads[k].norm(), n, rtol=5e-4, atol=1e-8)
        torch.testing.assert_close(grads[k].flatten()[:8], g["grad_heads"][k], rtol=5e-3, atol=1e-7)


def test_logits_only_forward_and_external_loss(golden, monkeypatch):
    """the soft-target route of training/train_maskgit_imagenet.py: forward without labels returns fp32 logits, and a loss
    computed by the caller back-propagates through the head to every parameter"""
    g = golden("micro_transformer.pt")
    cpu_math_ops.install(monkeypatch, exact=True)
    m = MaskGitTransformer(**g["config"])
    m.load_state_dict(g["state_dict"])
    m.train()
    b = g["batch"]
    logits = m(b["input_ids"])
    assert logits.dtype == torch.float32 and _rel(logits, g["logits"]) < 2e-5
    loss = torch.nn.functional.cross_entropy(logits.reshape(-1, logits.shape[-1]), b["labels"].reshape(-1), ignore_index=-100,
                                             label_smoothing=g["label_smoothing"])
    loss.backward()
    for n, p in m.named_parameters():
        assert _rel(p.grad, g["grads"][n]) < 2e-4, n


def test_generate2_host_loop_reproduces_the_reference_id_trace(golden, monkeypatch):
    """generate2's host loop (class token, codebook-restricted logits, ATen noise drawn from the caller's generator in the
    reference's order, mask_len / temperature schedule) against the ids the unmodified reference produced"""
    g = golden("micro_generate2.pt")
    p = golden("micro_transformer.pt")
    cpu_math_ops.install(monkeypatch, exact=True)
    m = MaskGitTransformer(**p["config"])
    m.load_state_dict(p["state_dict"])
    m.eval()
    monkeypatch.setattr(MaskGitTransformer, "device", property(lambda self: torch.device("cpu")), raising=False)
    for steps in (4, 7):
        gen = torch.Generator().manual_seed(g["seed"])
        cls = g["class_ids"].clone()
        ids = m.generate2(class_ids=cls, timesteps=steps, temperature=g["temperature"], generator=gen, use_cuda_graph=False)
        assert torch.equal(cls, g["class_ids"] + p["config"]["codebook_size"])  # quirk Q3: the caller's tensor is shifted
        assert torch.equal(ids, g["ids"][f"micro_generate2_steps{steps}"])


def test_generate2_classifier_free_guidance_host_loop(golden, monkeypatch):
    w = golden("micro_t2i_transformer.pt")
    g = golden("micro_t2i_generate2.pt")
    cpu_math_ops.install(monkeypatch, exact=True)
    m = MaskGitTransformer(**w["config"])
    m.load_state_dict(w["state_dict"])
    m.eval()
    monkeypatch.setattr(MaskGitTransformer, "device", property(lambda self: torch.device("cpu")), raising=False)
    ids = m.generate2(encoder_hidden_states=g["encoder_hidden_states"], timesteps=4, temperature=1.0, guidance_scale=3.0,
                      generator=torch.Generator().manual_seed(5), use_cuda_graph=False)
    assert torch.equal(ids, g["cfg_ids"])
    ids = m.generate2(input_ids=g["start"].clone(), encoder_hidden_states=g["encoder_hidden_states"],
                      negative_embeds=g["negative_embeds"], timesteps=3, temperature=0.7, guidance_scale=1.5,
                      generator=torch.Generator().manual_seed(6), use_cuda_graph=False)
    assert torch.equal(ids, g["neg_ids"])


# ---------------------------------------------------------------------------------------------------------------------
# use_conv_in_out (ConvEmbed / ConvMlmLayer, reference muse/modeling_transformer.py:988-1080)
def test_conv_in_out_seeded_construction_matches_the_reference(golden):
    g = golden("micro_conv_transformer.pt")
    torch.manual_seed(g["seed"])
    m = MaskGitTransformer(**g["config"])
    sd = m.state_dict()
    assert list(sd) == list(g["init_norms"])  # names AND registration order (= RNG order, = checkpoint keys)
    for k, n in g["init_norms"].items():
        assert abs(float(sd[k].double().norm()) - n) <= 1e-6 * n, k
    assert all(sd[k].shape == v.shape for k, v in g["state_dict"].items())
    # the two yaml files that enable the flag leave embedding_size unset: the reference cannot construct them
    assert g["embedding_size_unset"].startswith("TypeError")
    with pytest.raises(TypeError):
        MaskGitTransformer(**{k: v for k, v in g["config"].items() if k != "embedding_size"})


def test_conv_in_out_host_wiring_reproduces_the_reference_in_fp32(golden, monkeypatch):
    """patch gather in PixelUnshuffle channel order, the 1x1 convolutions as GEMMs on the packed [out, in] weights, position
    rows through the residual epilogue, PixelShuffle + Norm2D + logits on the outer grid, and every gradient back in the
    Conv2d / Embedding parameter layouts"""
    g = golden("micro_conv_transformer.pt")
    m, logits, loss = _run(g, True, monkeypatch, input_ids=g["input_ids"], labels=g["labels"],
                           encoder_hidden_states=g["encoder_hidden_states"], label_smoothing=g["label_smoothing"])
    assert logits.shape == g["logits"].shape == (2, 64, 64)
    assert _rel(logits, g["logits"]) < 2e-5
    assert abs(float(loss) - float(g["loss"])) < 2e-6 * abs(float(g["loss"]))
    assert set(n for n, _ in m.named_parameters()) == set(g["grads"])
    for n, p in m.named_parameters():
        assert p.grad is not None and p.grad.shape == p.shape, n
        assert _rel(p.grad, g["grads"][n]) < 2e-4, (n, _rel(p.grad, g["grads"][n]))


def test_conv_in_out_precision_recipe_and_inference_paths(golden, monkeypatch):
    g = golden("micro_conv_transformer.pt")
    m, logits, loss = _run(g, False, monkeypatch, input_ids=g["input_ids"], labels=g["labels"],
                           encoder_hidden_states=g["encoder_hidden_states"], label_smoothing=g["label_smoothing"])
    assert _rel(logits, g["logits"]) < 1e-2 and abs(float(loss) - float(g["loss"])) < 2e-3 * abs(float(g["loss"]))
    for n, p in m.named_parameters():
        assert _rel(p.grad, g["grads"][n]) < 6e-2, n
    m.eval()
    with torch.no_grad():
        full = m(g["input_ids"], encoder_hidden_states=g["encoder_hidden_states"])
        part, _ = m(g["input_ids"], encoder_hidden_states=g["encoder_hidden_states"], _raw_bf16=True, _logit_cols=40)
    assert full.shape == (2, 64, 64) and part.shape == (2, 64, 40)
    assert torch.equal(part.float(), full[..., :40])  # column-restricted logits (generate2) = the same GEMM, fewer columns
    with pytest.raises(ValueError):
        m(g["input_ids"][:, :60], encoder_hidden_states=g["encoder_hidden_states"])  # not a square grid


def test_conv_in_out_external_loss_through_the_returned_logits(golden, monkeypatch):
    """soft-target style training with use_conv_in_out: the caller's loss back-propagates through the returned logits"""
    g = golden("micro_conv_transformer.pt")
    cpu_math_ops.install(monkeypatch, exact=True)
    m = MaskGitTransformer(**g["config"])
    m.load_state_dict(g["state_dict"])
    m.train()
    logits = m(g["input_ids"], encoder_hidden_states=g["encoder_hidden_states"])
    assert logits.dtype == torch.float32 and _rel(logits, g["logits"]) < 2e-5
    loss = torch.nn.functional.cross_entropy(logits.reshape(-1, logits.shape[-1]), g["labels"].reshape(-1), ignore_index=-100,
                                             label_smoothing=g["label_smoothing"])
    loss.backward()
    for n, p in m.named_parameters():
        assert _rel(p.grad, g["grads"][n]) < 2e-4, n


def test_packed_operand_cache_follows_every_kind_of_weight_update(golden, monkeypatch):
    """The bf16 operand cache is keyed on (storage, version counter) of every Linear weight: an optimizer step, a
    load_state_dict, ``EMAModel.copy_to`` / ``restore`` (train_muse.py:857-908 validates with the EMA weights) and a plain
    in-place edit must each be visible in the very next forward -- checked against a freshly built model holding the same
    weights (the ADVICE r1 'stale packed operands' bug class, on the CPU)."""
    from open_muse_b200 import EMAModel

    g = golden("micro_transformer.pt")
    cpu_math_ops.install(monkeypatch, exact=True)
    ids = g["batch"]["input_ids"]

    def fresh(sd):
        f = MaskGitTransformer(**g["config"])
        f.load_state_dict(sd)
        return f.eval()(ids)

    m = MaskGitTransformer(**g["config"])
    m.load_state_dict(g["state_dict"])
    m.eval()
    with torch.no_grad():
        base = m(ids)
        assert torch.equal(base, fresh(m.state_dict()))
        # (1) optimizer step
        m.train()
    _, loss = m(ids, labels=g["batch"]["labels"])
    loss.backward()
    opt = torch.optim.SGD(m.parameters(), lr=0.5)
    opt.step()
    m.eval()
    with torch.no_grad():
        after_step = m(ids)
        assert not torch.equal(after_step, base) and torch.equal(after_step, fresh(m.state_dict()))
        # (2) EMA copy_to / restore
        ema = EMAModel(m.parameters(), decay=0.5)
        for s in ema.shadow_params:
            s.mul_(0.9)
        ema.store(m.parameters())
        ema.copy_to(m.parameters())
        with_ema = m(ids)
        assert not torch.equal(with_ema, after_step) and torch.equal(with_ema, fresh(m.state_dict()))
        ema.restore(m.parameters())
        assert torch.equal(m(ids), after_step)
        # (3) load_state_dict and (4) a plain in-place edit of one weight
        m.load_state_dict(g["state_dict"])
        assert torch.equal(m(ids), base)
        m.transformer_layers[1].ffn.wo.weight.mul_(1.5)
        edited = m(ids)
        assert not torch.equal(edited, base) and torch.equal(edited, fresh(m.state_dict()))
