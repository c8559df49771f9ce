"""Dropout of MaskGiTUViT_v2 on the GPU: the GRN dropout kernels' keep bits against the generator's restatement
(tests/test_dropout_cpu.py) and their math against the undropped kernels, model parity with the unmodified reference given
the recorded masks, determinism under torch.manual_seed, and mask statistics and training at the U-ViT default widths."""
import math

import pytest
import torch

from open_muse_b200 import MaskGiTUViT_v2, ops
from tests.test_dropout_cpu import elem_keep, keep_scale, pack_bits, threshold, unpack_bits
from tests.test_uvit_dropout_cpu import ARGS, _columns, _replayed_reference, expected_sites

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-20))


def _seed(v):
    return torch.tensor([v], dtype=torch.int64, device=DEV)


def _rand(shape, seed, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(shape, generator=g, device=DEV) * scale).to(torch.bfloat16)


def _frac_ok(k, p):
    r = 1 - threshold(p) / 65536
    return abs(float(k.float().mean()) - r) <= 6 * math.sqrt(r * (1 - r) / k.numel())


@pytest.mark.parametrize("B,HW,C", [(2, 256, 3072), (3, 64, 256), (2, 16, 72)])
def test_grn_dropout_bits_and_math(B, HW, C):
    """the ResBlock's dropout fused into GELU + GRN: the stored bits equal the restatement (pad bits 0), the output is the
    undropped one times Z, and the backward equals the undropped backward of bf16(dout * Z)"""
    p, seed, site = 0.1, -7654321987654321, 9
    rows = B * HW
    x = _rand((rows, C), 1)
    g = torch.Generator(device=DEV).manual_seed(2)
    gamma = torch.randn(C, generator=g, device=DEV) * 0.3
    beta = torch.randn(C, generator=g, device=DEV) * 0.1
    out, st, bits = ops.grn(x, gamma, beta, B, HW, save_stats=True, dropout=(p, _seed(seed), site))
    out0, st0 = ops.grn(x, gamma, beta, B, HW, save_stats=True)
    assert torch.equal(st, st0)  # dropout follows GRN: its statistics do not change
    keep = elem_keep(seed, site, rows, C, p)
    assert bits.shape == (rows, (C + 31) // 32)
    assert torch.equal(bits.cpu(), pack_bits(keep))
    if C % 32:
        assert int(((bits[:, -1].long() & 0xFFFFFFFF) >> (C % 32)).max()) == 0  # pad bits
    kd = keep.to(DEV)
    z = kd.float() * keep_scale(p)
    assert _rel(out, out0.float() * z) < 1e-2 and bool((out[~kd] == 0).all())
    dout = _rand((rows, C), 3)
    dg, db = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    dx = ops.grn_bwd(x, dout, st, gamma, dg, db, B, HW, dropout=(p, bits))
    dg0, db0 = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    dx0 = ops.grn_bwd(x, (dout.float() * z).to(torch.bfloat16), st, gamma, dg0, db0, B, HW)
    assert _rel(dx, dx0) < 1e-2 and _rel(dg, dg0) < 1e-2 and _rel(db, db0) < 1e-2


def _train(g, seed, weighted=False):
    cfg = dict(g["config"], hidden_dropout=0.1, attention_dropout=0.1)
    m = MaskGiTUViT_v2(**cfg)
    m.load_state_dict(g["state_dict"])
    m.to(DEV).train()
    kw = dict(labels=g["labels"].to(DEV), label_smoothing=0.1)
    if weighted:
        kw["loss_weight"] = g["loss_weight"].to(DEV)
    torch.manual_seed(seed)
    with ops.dropout_record() as log:
        with torch.autocast("cuda", dtype=torch.bfloat16):
            logits, loss = m(*[g[k].to(DEV) for k in ARGS], **kw)
    loss.backward()
    grads = {n: p.grad.clone() for n, p in m.named_parameters()}
    return cfg, logits.detach(), loss.detach(), grads, [(s, b.clone()) for s, b in log]


@pytest.mark.parametrize("name,weighted", [("micro_uvit_v2.pt", True), ("micro_uvit_v2_downup.pt", False)])
def test_model_parity_with_the_reference_given_the_same_masks(golden, name, weighted):
    g = golden(name)
    cfg, logits, loss, grads, log = _train(g, 3, weighted)
    assert [s for s, _ in log] == expected_sites(cfg, 0.1, 0.1)
    masks = {s: b.cpu() for s, b in log}
    S, Skv = g["input_ids"].shape[1], g["encoder_hidden_states"].shape[1]
    ref = _replayed_reference(cfg, g["state_dict"], masks, S, Skv, 0.1, 0.1, device=DEV)
    kw = dict(labels=g["labels"].to(DEV), label_smoothing=0.1)
    if weighted:
        kw["loss_weight"] = g["loss_weight"].to(DEV)
    r_logits, r_loss = ref(*[g[k].to(DEV) for k in ARGS], **kw)
    r_loss.backward()
    assert abs(float(loss) - float(r_loss.detach())) / float(r_loss.detach()) < 2e-3
    errs = {n: _rel(grads[n], p.grad) for n, p in ref.named_parameters()}
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:6]
    print("worst grad rel-L2:", ", ".join(f"{k}={v:.2e}" for k, v in worst))
    bad = {k: v for k, v in errs.items() if v > 8e-2 and not (".query." in k or ".key." in k)}
    assert not bad, bad
    cos = {n: float(torch.nn.functional.cosine_similarity(grads[n].float().flatten(), p.grad.float().flatten(), dim=0))
           for n, p in ref.named_parameters()}
    assert min(cos.values()) > 0.95, sorted(cos.items(), key=lambda kv: kv[1])[:5]


def test_same_seed_gives_identical_masks_logits_and_loss(golden):
    g = golden("micro_uvit_v2.pt")
    r1, r2 = _train(g, 11), _train(g, 11)
    assert [s for s, _ in r1[4]] == [s for s, _ in r2[4]]
    assert all(torch.equal(a, b) for (_, a), (_, b) in zip(r1[4], r2[4]))
    assert torch.equal(r1[1], r2[1]) and torch.equal(r1[2], r2[2])
    # the U-ViT weight gradients accumulate with fp32 atomics: equal up to the summation order
    assert all(_rel(r1[3][n], r2[3][n]) < 1e-4 for n in r1[3])
    r3 = _train(g, 12)
    assert all(not torch.equal(a, b) for (_, a), (_, b) in zip(r1[4], r3[4]))


def test_default_widths_train_with_dropout():
    """hidden 1024 / 16 heads, blocks 768 / 12 heads with kv_mapper, 256 tokens, 77 text states, 2 layers, 1 res block"""
    cfg = dict(num_hidden_layers=2, num_res_blocks=1, vocab_size=1032, codebook_size=1024, intermediate_size=2816,
               hidden_dropout=0.1, attention_dropout=0.1)
    torch.manual_seed(0)
    m = MaskGiTUViT_v2(**cfg)
    gen = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for k, x in m.state_dict().items():
            if "adaLN_modulation.mapper" in k or k.endswith("gamma") or k.endswith("beta") or k == "mlm_layer.conv1.weight":
                x.copy_(torch.randn(x.shape, generator=gen) * 0.03)
    B = 4
    ids = torch.randint(0, 1024, (B, 256), generator=gen)
    mask = torch.rand(B, 256, generator=gen) < 0.5
    inp, lab = torch.where(mask, 1031, ids).to(DEV), torch.where(mask, ids, -100).to(DEV)
    enc = torch.randn(B, 77, 768, generator=gen).to(DEV)
    ce = torch.randn(B, 768, generator=gen).to(DEV)
    mc = torch.tensor([[256.0, 256.0, 0.0, 0.0, 6.0]]).repeat(B, 1).to(DEV)
    m.to(DEV).train()
    opt = torch.optim.AdamW(m.parameters(), lr=1e-3)
    losses = []
    for step in range(6):
        with ops.dropout_record() as log, torch.autocast("cuda", dtype=torch.bfloat16):
            _, loss = m(inp, enc, ce, mc, labels=lab)
        loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
        losses.append(float(loss))
        if step == 0:
            assert [s for s, _ in log] == list(range(12))
            cols = _columns(dict(m.config), 256, 77)
            masks = dict(log)
            assert _frac_ok(unpack_bits(masks[0].cpu(), cols[0]), 0.1)  # GRN of the down ResBlock: [B * 256, 3072]
            assert _frac_ok(unpack_bits(masks[1].cpu(), cols[1]), 0.1)  # its attention: [B, 12, 256, 77]
    assert all(math.isfinite(x) for x in losses)
    assert losses[-1] < losses[0], losses
    m.eval()
    with torch.no_grad():
        a, b = m(inp, enc, ce, mc), m(inp, enc, ce, mc)
    assert torch.equal(a, b)
