"""Gradient checkpointing on the GPU.  A checkpointed layer (MaskGitTransformer) or block / layer (MaskGiTUViT_v2) keeps
only its inputs and re-runs its forward kernels in its backward; every kernel is run-to-run deterministic and the dropout
masks follow from the device-side seed, so logits, loss and every gradient must be bit-identical with checkpointing on and
off -- launched one by one, replayed from a captured CUDA graph, and after fused optimizer steps.  The exception is the
weight gradients of MaskGiTUViT_v2, which its kernels accumulate with fp32 atomics: they are equal up to the summation
order in any two runs (tests/test_uvit_dropout_gpu.py), checkpointed or not; its logits and loss are bit-identical.  The
memory held between forward and backward is measured per layer: with checkpointing a layer keeps its inputs and nothing
else."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from open_muse_b200 import FusedAdamW, MaskGiTUViT_v2  # noqa: E402
from open_muse_b200.graphs import GraphedStep  # noqa: E402
from open_muse_b200.modeling_transformer import MaskGitTransformer  # noqa: E402
from oracle import transformer_oracle as T  # noqa: E402

DEV = "cuda"
BASE = dict(vocab_size=2025, max_position_embeddings=257, hidden_size=512, num_hidden_layers=3, num_attention_heads=8,
            intermediate_size=2048, codebook_size=1024, num_vq_tokens=256, num_classes=1000)
UVIT_ARGS = ("input_ids", "encoder_hidden_states", "cond_embeds", "micro_conds")


def _class_batch(B, seed=5):
    g = torch.Generator().manual_seed(seed)
    tokens = torch.randint(0, 1024, (B, 256), generator=g)
    cls = torch.randint(0, 1000, (B,), generator=g)
    inp, lab = T.mask_tokens(tokens, cls, torch.rand(B, generator=g), torch.rand(B, 256, generator=g), 1024, 2024)
    return dict(input_ids=inp.to(DEV), labels=lab.to(DEV))


def _cross_case(head_dim):
    H = 512
    cfg = dict(vocab_size=1025, max_position_embeddings=256, hidden_size=H, num_hidden_layers=2,
               num_attention_heads=H // head_dim, intermediate_size=1024, add_cross_attention=True, encoder_hidden_size=384,
               project_encoder_hidden_states=True, codebook_size=1024, num_vq_tokens=256, use_codebook_size_for_output=True)
    g = torch.Generator().manual_seed(3)
    B = 4
    ids = torch.randint(0, 1024, (B, 256), generator=g)
    mask = torch.rand(B, 256, generator=g) < 0.5
    fwd = dict(input_ids=torch.where(mask, 1024, ids).to(DEV), labels=torch.where(mask, ids, -100).to(DEV),
               encoder_hidden_states=torch.randn(B, 77, 384, generator=g).to(DEV))
    return cfg, fwd


def _v1(cfg, p, ckpt, sd=None):
    torch.manual_seed(0)
    m = MaskGitTransformer(**dict(cfg, hidden_dropout=p, attention_dropout=p))
    if sd is not None:
        m.load_state_dict(sd)
    m.to(DEV).train()
    if ckpt:
        m.enable_gradient_checkpointing()
    return m


def _run(m, fwd):
    torch.manual_seed(11)  # the dropout seed is drawn from the default CUDA generator
    m.zero_grad(set_to_none=True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        logits, loss = m(**fwd)
    loss.backward()
    torch.cuda.synchronize()
    return logits.detach().clone(), loss.detach().clone(), {n: p.grad.clone() for n, p in m.named_parameters()}


def _rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / b.norm().clamp_min(1e-20))


def _assert_bit_equal(a, b):
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert a[2].keys() == b[2].keys()
    for n in a[2]:
        assert torch.equal(a[2][n], b[2][n]), n


@pytest.mark.parametrize("p", [0.0, 0.1])
def test_base_model_is_bit_identical_with_checkpointing(p):
    fwd = _class_batch(12)
    _assert_bit_equal(_run(_v1(BASE, p, False), fwd), _run(_v1(BASE, p, True), fwd))


@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("head_dim", [64, 128])
def test_cross_attention_model_is_bit_identical_with_checkpointing(head_dim, p):
    cfg, fwd = _cross_case(head_dim)
    _assert_bit_equal(_run(_v1(cfg, p, False), fwd), _run(_v1(cfg, p, True), fwd))


@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("name", ["micro_uvit_v2.pt", "micro_uvit_v2_downup.pt"])
def test_uvit_fixtures_match_with_checkpointing(golden, name, p):
    g = golden(name)
    fwd = dict(zip(UVIT_ARGS, [g[k].to(DEV) for k in UVIT_ARGS]), labels=g["labels"].to(DEV), label_smoothing=0.1)
    runs = []
    for ckpt in (False, True):
        m = MaskGiTUViT_v2(**dict(g["config"], hidden_dropout=p, attention_dropout=p))
        m.load_state_dict(g["state_dict"])
        m.to(DEV).train()
        if ckpt:
            m.enable_gradient_checkpointing()
            assert m.down_blocks[0].gradient_checkpointing and m.up_blocks[0].gradient_checkpointing
        runs.append(_run(m, fwd))
    (l0, s0, g0), (l1, s1, g1) = runs
    assert torch.equal(l0, l1) and torch.equal(s0, s1)
    assert g0.keys() == g1.keys()
    for n in g0:  # fp32-atomic weight gradients: equal up to the order of the summation
        assert torch.equal(g0[n], g1[n]) or _rel(g0[n], g1[n]) < 1e-4, (n, _rel(g0[n], g1[n]))


def test_graphed_checkpointed_step_replays_the_eager_plain_step():
    fwd = _class_batch(12)
    m = _v1(BASE, 0.0, True)

    def step(i, l_):
        m.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            logits, loss = m(i, labels=l_)
        loss.backward()
        return logits, loss

    # graph first (see tests/test_model_gpu.py: an eager backward before the capture would tie the AccumulateGrad nodes to
    # the legacy default stream)
    graphed = GraphedStep(step, (fwd["input_ids"], fwd["labels"]))
    for _ in range(2):
        logits, loss = graphed(fwd["input_ids"], fwd["labels"])
    torch.cuda.synchronize()
    replay = (logits.clone(), loss.clone(), {n: p.grad.clone() for n, p in m.named_parameters()})
    _assert_bit_equal(replay, _run(_v1(BASE, 0.0, False), fwd))


def test_fused_adamw_steps_are_bit_identical_with_checkpointing():
    fwd = _class_batch(8)
    params = []
    for ckpt in (False, True):
        m = _v1(BASE, 0.1, ckpt)
        opt = FusedAdamW(m.parameters(), lr=1e-3, weight_decay=0.01, model=m)
        for _ in range(2):
            _run(m, fwd)
            opt.step()
        torch.cuda.synchronize()
        params.append({n: p.detach().clone() for n, p in m.named_parameters()})
    for n in params[0]:
        assert torch.equal(params[0][n], params[1][n]), n


# ------------------------------------------------------------------------------------------------ memory
def _held_after_forward(m, fwd):
    """bytes allocated by a training forward and still held when the backward would start"""
    _run(m, fwd)  # builds the operand cache, the attention workspaces and the gradients' first allocations
    m.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        out = m(**fwd)
    torch.cuda.synchronize()
    held = torch.cuda.memory_allocated() - before
    del out
    return held


def _r512(n):
    return -(-n // 512) * 512  # the caching allocator's rounding of small blocks


MiB = 2 ** 20  # a large-pool block is not split when less than 1 MiB would remain: up to 1 MiB of slack per tensor


def test_v1_layer_memory_held_between_forward_and_backward():
    B, S, H, I = 8, 257, BASE["hidden_size"], BASE["intermediate_size"]
    T_ = B * S
    fwd = _class_batch(B)
    per_layer = {}
    for ckpt in (False, True):
        held = [_held_after_forward(_v1(dict(BASE, num_hidden_layers=L), 0.0, ckpt), fwd) for L in (2, 4)]
        per_layer[ckpt] = (held[1] - held[0]) / 2
    # checkpointed: the layer's fp32 input x
    assert abs(per_layer[True] - 4 * H * T_) <= MiB, per_layer
    # plain: fp32 x, x2; bf16 h1, qkv, ctxt, ao, h2, [a|b], ml (22 H + 6 I bytes per token), plus the statistics and the
    # attention log-sum-exp rows
    full = (22 * H + 6 * I) * T_
    assert full <= per_layer[False] <= full + (32 + 4 * BASE["num_attention_heads"]) * T_ + 4 * MiB, per_layer
    print(f"per layer, B={B}: plain {per_layer[False] / 2**20:.2f} MiB, checkpointed {per_layer[True] / 2**20:.3f} MiB")


def test_uvit_layer_memory_held_between_forward_and_backward(golden):
    g = golden("micro_uvit_v2.pt")
    cfg = dict(g["config"], hidden_dropout=0.0, attention_dropout=0.0)
    B = 2
    fwd = dict(zip(UVIT_ARGS, [g[k][:B].to(DEV) for k in UVIT_ARGS]), labels=g["labels"][:B].to(DEV))
    H, S = cfg["hidden_size"], g["input_ids"].shape[1]
    per_layer = {}
    for ckpt in (False, True):
        held = []
        for L in (2, 4):
            torch.manual_seed(0)
            m = MaskGiTUViT_v2(**dict(cfg, num_hidden_layers=L)).to(DEV).train()
            if ckpt:
                m.gradient_checkpointing = True  # the transformer layers only: the stages are the same in both models
            held.append(_held_after_forward(m, fwd))
        per_layer[ckpt] = (held[1] - held[0]) / 2
    # checkpointed: bf16 hidden x, fp32 residual r and the fp32 adaLN rows (3 x (scale | shift)) of the layer
    expect = _r512(2 * H * B * S) + _r512(4 * H * B * S) + _r512(4 * 6 * H * B)
    assert abs(per_layer[True] - expect) <= 1024, (per_layer, expect)
    assert per_layer[False] > 4 * per_layer[True], per_layer
