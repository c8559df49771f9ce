"""Attention head widths 96 and 128 without a GPU: which widths the models accept, seeded construction against the
unmodified reference (the oracle/_ref snapshot, run in a subprocess), and the host wiring of MaskGitTransformer /
MaskGiTUViT_v2 on the torch restatements of the kernels (tests/cpu_math_ops.py, exact fp32 mode) against the oracle's
logits and gradients."""
import json
import os
import subprocess
import sys

import pytest
import torch

from open_muse_b200 import MaskGiTUViT_v2, MaskGitTransformer
from oracle import ref_snapshot
from oracle import transformer_oracle as T
from oracle import transformer_v2_oracle as V2
from tests import cpu_math_ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

V1 = dict(vocab_size=72, max_position_embeddings=17, num_hidden_layers=2, num_attention_heads=2, intermediate_size=128,
          codebook_size=64, num_vq_tokens=16, num_classes=7, hidden_dropout=0.0, attention_dropout=0.0)
UVIT = dict(hidden_size=256, num_attention_heads=2, in_channels=192, block_out_channels=(192,), block_num_heads=2,
            num_res_blocks=1, num_hidden_layers=2, intermediate_size=128, vocab_size=72, codebook_size=64,
            encoder_hidden_size=32, cond_embed_dim=16, micro_cond_encode_dim=8, micro_cond_embed_dim=40, norm_type="rmsnorm")
# hidden 256 / 2 heads = head_dim 128 everywhere; hidden 192 / 2 heads = 96
V1_WIDTHS = {128: dict(V1, hidden_size=256), 96: dict(V1, hidden_size=192)}
UVIT_WIDTHS = {"layers 128, blocks 96": UVIT,
               "layers 96, blocks 128": dict(UVIT, hidden_size=192, in_channels=256, block_out_channels=(256,))}


def _rel(a, b):
    a, b = a.detach().float(), b.detach().float()
    return float((a - b).norm() / b.norm().clamp_min(1e-20))


@pytest.mark.parametrize("hidden,heads", [(384, 12), (320, 4), (512, 2), (160, 1)])  # head_dim 32, 80, 256, 160
def test_other_head_widths_still_raise_and_name_the_supported_ones(hidden, heads):
    with pytest.raises(NotImplementedError, match="48, 64, 96 or 128"):
        MaskGitTransformer(**dict(V1, hidden_size=hidden, num_attention_heads=heads))
    with pytest.raises(NotImplementedError, match="48, 64, 96 or 128"):
        MaskGiTUViT_v2(**dict(UVIT, hidden_size=hidden, num_attention_heads=heads))
    with pytest.raises(NotImplementedError, match="48, 64, 96 or 128"):
        MaskGiTUViT_v2(**dict(UVIT, in_channels=hidden, block_out_channels=(hidden,), block_num_heads=heads))


@pytest.mark.parametrize("hd", [96, 128])
def test_head_widths_96_and_128_construct(hd):
    m = MaskGitTransformer(**dict(V1, hidden_size=2 * hd))
    assert m.config.hidden_size // m.config.num_attention_heads == hd
    u = MaskGiTUViT_v2(**dict(UVIT, hidden_size=2 * hd, in_channels=2 * hd, block_out_channels=(2 * hd,)))
    assert u.config.hidden_size // u.config.num_attention_heads == hd


REF_SIDE = r'''
import json, sys, torch
sys.path.insert(0, sys.argv[1])
from oracle.ref_snapshot import import_reference
muse = import_reference()
from muse.modeling_transformer_v2 import MaskGiTUViT_v2
out = {}
for kind, key, cfg in json.load(open(sys.argv[2])):
    cls = muse.MaskGitTransformer if kind == "v1" else MaskGiTUViT_v2
    torch.manual_seed(0)
    m = cls(**cfg)
    out[key] = (list(m.state_dict().items()), {k: v for k, v in m.config.items() if not k.startswith("_")})
torch.save(out, sys.argv[3])
'''


@pytest.mark.skipif(not ref_snapshot.available(), reason="oracle/_ref snapshot of the reference not available")
def test_seeded_construction_matches_the_reference(tmp_path):
    """torch.manual_seed(0) then the constructor: the same tensor names in the same order, shapes, dtypes and values as
    the unmodified reference at head widths 96 and 128, and the same config"""
    jobs = [("v1", f"v1 hd {hd}", cfg) for hd, cfg in V1_WIDTHS.items()]
    jobs += [("v2", f"v2 {k}", dict(cfg, block_out_channels=list(cfg["block_out_channels"])))
             for k, cfg in UVIT_WIDTHS.items()]
    (tmp_path / "jobs.json").write_text(json.dumps(jobs))
    (tmp_path / "ref.py").write_text(REF_SIDE)
    r = subprocess.run([sys.executable, str(tmp_path / "ref.py"), ROOT, str(tmp_path / "jobs.json"), str(tmp_path / "ref.pt")],
                       capture_output=True, text=True, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr[-3000:]
    ref = torch.load(tmp_path / "ref.pt")
    for kind, key, cfg in jobs:
        torch.manual_seed(0)
        m = (MaskGitTransformer if kind == "v1" else MaskGiTUViT_v2)(**cfg)
        ours = list(m.state_dict().items())
        theirs, ref_cfg = ref[key]
        assert [n for n, _ in ours] == [n for n, _ in theirs], key
        for (n, a), (_, b) in zip(ours, theirs):
            assert a.shape == b.shape and a.dtype == b.dtype and torch.equal(a, b), (key, n)
        mine = dict(m.config)
        for k, v in ref_cfg.items():
            if k in mine:
                assert (list(mine[k]) if isinstance(mine[k], tuple) else mine[k]) == \
                    (list(v) if isinstance(v, tuple) else v), (key, k)


def _v1_batch(g):
    tokens = torch.randint(0, 64, (3, 16), generator=g)
    cls = torch.randint(0, 7, (3,), generator=g)
    return T.mask_tokens(tokens, cls, torch.rand(3, generator=g), torch.rand(3, 16, generator=g), 64, 71)


@pytest.mark.parametrize("hd", [128, 96])
def test_transformer_host_wiring_reproduces_the_oracle_in_fp32(monkeypatch, hd):
    """exact mode: logits, loss and every parameter gradient of the scale 1 / sqrt(head_dim) path against the oracle's
    fp32 autograd"""
    cfg = V1_WIDTHS[hd]
    cpu_math_ops.install(monkeypatch, exact=True)
    torch.manual_seed(1)
    m = MaskGitTransformer(**cfg).train()
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    inp, lab = _v1_batch(torch.Generator().manual_seed(2))
    ref_logits, ref_loss, ref_grads = T.forward_backward(sd, cfg, inp, lab, label_smoothing=0.1)
    logits, loss = m(inp, labels=lab, label_smoothing=0.1)
    loss.backward()
    assert _rel(logits, ref_logits) < 2e-5
    assert abs(float(loss.detach()) - float(ref_loss)) < 2e-6 * abs(float(ref_loss)) + 1e-7
    params = dict(m.named_parameters())
    assert set(params) == set(ref_grads)
    for n, gr in ref_grads.items():
        assert _rel(params[n].grad, gr) < 2e-4, (n, _rel(params[n].grad, gr))
    m.eval()
    with torch.no_grad():
        assert _rel(m(inp), ref_logits) < 2e-5


@pytest.mark.parametrize("widths", list(UVIT_WIDTHS))
def test_uvit_host_wiring_reproduces_the_oracle_in_fp32(monkeypatch, widths):
    """head_dim 128 / 96 in the transformer layers and 96 / 128 in the block attentions: no_grad inference, the training
    loss and every gradient against the oracle's fp32 autograd"""
    cfg = UVIT_WIDTHS[widths]
    cpu_math_ops.install(monkeypatch, exact=True)
    torch.manual_seed(3)
    m = MaskGiTUViT_v2(**cfg)
    with torch.no_grad():
        for p in m.parameters():  # adaLN mappers and GRN parameters are zeros at init
            p.add_((0.1 if p.dim() == 1 else 0.02) * torch.randn_like(p))
    g = torch.Generator().manual_seed(4)
    ids, lab = torch.randint(0, 64, (2, 16), generator=g), torch.randint(0, 64, (2, 16), generator=g)
    enc, ce, mc = torch.randn(2, 5, 32, generator=g), torch.randn(2, 16, generator=g), torch.rand(2, 5, generator=g) * 100
    q = {k: v.detach().clone().requires_grad_(True) for k, v in m.state_dict().items()}
    ref_logits, ref_loss = V2.forward(q, dict(m.config), ids, enc, ce, mc, labels=lab, label_smoothing=0.1)
    ref_loss.backward()
    m.eval()
    with torch.no_grad():
        assert _rel(m(ids, enc, ce, mc), ref_logits) < 5e-5
    m.train()
    _, loss = m(ids, enc, ce, mc, labels=lab, label_smoothing=0.1)
    loss.backward()
    assert abs(float(loss.detach()) - float(ref_loss.detach())) < 1e-5 * float(ref_loss.detach())
    for n, p in m.named_parameters():
        assert _rel(p.grad, q[n].grad) < 5e-4, (n, _rel(p.grad, q[n].grad))
