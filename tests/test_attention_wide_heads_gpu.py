"""Attention head widths 96 and 128 on the GPU: the wgmma kernels (two 64-column TMA boxes per tile) against fp64 torch
math for every (batch, head, row), their dropout bits against the Philox mapping, and MaskGitTransformer /
MaskGiTUViT_v2 with these widths against the oracle's fp32 autograd.

The per-row bounds are the HD-64 ones of tests/local_error.py (BOUNDS["attn.*"], ATTN_LSE_ABS), not looser; each
kernel test prints its worst per-row error next to its bound."""
import math

import pytest
import torch

from open_muse_b200 import MaskGiTUViT_v2, ops
from open_muse_b200.modeling_transformer import MaskGitTransformer
from open_muse_b200.optim import FusedAdamW
from oracle import transformer_oracle as T
from oracle import transformer_v2_oracle as V2
from tests.local_error import ATTN_LSE_ABS, BOUNDS, attn_rows, check_local
from tests.test_dropout_cpu import attn_keep, keep_scale, pack_bits, unpack_bits
from tests.test_kernel_local_gpu import _heads, _plant_q, _randn

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16
F64 = torch.float64
P_DROP, SEED, SITE = 0.1, -1234567890123456789, 7


def _rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-20))


def _operands(B, nh, Sq, Skv, hd):
    """Q / K / V as strided column views: self-attention slices one [T, 3H] projection, cross-attention takes Q from its
    own buffer and K / V from one [T_kv, 2H] projection.  Planted rows as in tests/test_kernel_local_gpu.py."""
    H = nh * hd
    scale = 1.0 / math.sqrt(hd)
    cross = Sq != Skv
    if cross:
        qbuf, kvbuf = _randn((B * Sq, H), 1).to(BF).float(), _randn((B * Skv, 2 * H), 2).to(BF).float()
        qcol, kbuf, kcol, vcol = 0, kvbuf, 0, H
    else:
        qbuf = kbuf = _randn((B * Sq, 3 * H), 1).to(BF).float()
        qcol, kcol, vcol = 0, H, 2 * H
    k4 = _heads(kbuf[:, kcol:kcol + H], B, Skv, nh, hd)
    q4 = _heads(qbuf[:, qcol:qcol + H], B, Sq, nh, hd).clone()
    q4 *= torch.tensor([0.25, 1.0, 4.0]).repeat(B * nh)[:B * nh].view(B, nh, 1, 1)
    _plant_q(q4, k4, scale, Sq, Skv)
    qbuf[:, qcol:qcol + H] = q4.permute(0, 2, 1, 3).reshape(B * Sq, H)
    qbuf = qbuf.to(BF).to(DEV)
    kvdev = qbuf if not cross else kvbuf.to(BF).to(DEV)
    return qbuf[:, qcol:qcol + H], kvdev[:, kcol:kcol + H], kvdev[:, vcol:vcol + H], scale


def _attention_case(B, nh, Sq, Skv, hd, drop):
    H = nh * hd
    case = f"(B {B}, nh {nh}, Sq {Sq}, Skv {Skv}, hd {hd}{', dropout' if drop else ''})"
    q, k, v, scale = _operands(B, nh, Sq, Skv, hd)
    do = _randn((B * Sq, H), 3).to(BF).to(DEV)
    dropout = (P_DROP, torch.tensor([SEED], dtype=torch.int64, device=DEV), SITE) if drop else None
    res = ops.attn_fwd(q, k, v, B, nh, Sq, Skv, scale, head_dim=hd, dropout=dropout)
    o, lse = res[0], res[1]
    dq = torch.full((B * Sq, H), float("nan"), dtype=BF, device=DEV)
    dk = torch.full((B * Skv, H), float("nan"), dtype=BF, device=DEV)
    dv = torch.full((B * Skv, H), float("nan"), dtype=BF, device=DEV)
    ops.attn_bwd(q, k, v, o, do, lse, dq, dk, dv, B, nh, Sq, Skv, scale, head_dim=hd,
                 dropout=(P_DROP, res[2]) if drop else None)
    torch.cuda.synchronize()

    qd, kd, vd = (_heads(t.to(F64), B, S, nh, hd).clone().requires_grad_(True) for t, S in ((q, Sq), (k, Skv), (v, Skv)))
    s = (qd @ kd.transpose(-1, -2)) * scale
    p = s.softmax(-1)
    if drop:
        p = p * (unpack_bits(res[2].cpu(), Skv).to(DEV).to(F64) * keep_scale(P_DROP))
    od = p @ vd
    od.backward(_heads(do.to(F64), B, Sq, nh, hd))
    lse_ref = torch.logsumexp(s.detach(), -1)

    tok = lambda t, S: t.detach().permute(0, 2, 1, 3).reshape(B * S, H)  # noqa: E731
    gq, gkv = attn_rows(B, nh, Sq, hd), attn_rows(B, nh, Skv, hd)
    for key, out, ref, grp in (("attn.o", o, tok(od, Sq), gq), ("attn.dq", dq, tok(qd.grad, Sq), gq),
                               ("attn.dk", dk, tok(kd.grad, Skv), gkv), ("attn.dv", dv, tok(vd.grad, Skv), gkv)):
        r = check_local(out, ref, grp, *BOUNDS[key], f"{key} {case}")
        print(f"{key} {case}: worst per-row {r.worst:.3e} (bound {BOUNDS[key][0]:.1e}) at {r.where}, "
              f"elementwise {r.elem:.3e} (bound {BOUNDS[key][1]:.1e})")
    lse_err = float((lse.to(F64) - lse_ref).abs().max())
    print(f"attn.lse {case}: max |lse - lse_ref| {lse_err:.3e} (bound {ATTN_LSE_ABS:.1e})")
    assert lse_err <= ATTN_LSE_ABS, (case, lse_err)
    return res


SHAPES = [
    (2, 3, 257, 257), (2, 3, 65, 65), (2, 3, 385, 385), (3, 2, 130, 5),  # ragged lengths
    (2, 3, 256, 77),  # cross-attention on 77 text states
    (8, 8, 257, 257),  # 320 CTAs per kernel: more than one wave at two (fwd, dQ) or one (dK/dV) CTA per SM on 132 SMs
]


@pytest.mark.parametrize("hd", [128, 96])
@pytest.mark.parametrize("B,nh,Sq,Skv", SHAPES)
def test_wide_head_attention_local(B, nh, Sq, Skv, hd):
    _attention_case(B, nh, Sq, Skv, hd, drop=False)


@pytest.mark.parametrize("hd", [128, 96])
@pytest.mark.parametrize("B,nh,Sq,Skv", [(2, 2, 257, 257), (3, 2, 100, 77)])
def test_wide_head_attention_dropout(B, nh, Sq, Skv, hd):
    """The keep bits are the Philox mapping's for (seed, site, b, h, row, column), whatever the head width; the outputs
    with those bits are held to the same per-row bounds as without dropout"""
    res = _attention_case(B, nh, Sq, Skv, hd, drop=True)
    keep = attn_keep(SEED, SITE, B, nh, Sq, Skv, P_DROP)
    assert torch.equal(res[2].cpu(), pack_bits(keep))
    # the same draw at head width 64 gives the same bits: they do not depend on HD
    q, k, v, _ = _operands(B, nh, Sq, Skv, 64)
    bits64 = ops.attn_fwd(q, k, v, B, nh, Sq, Skv, 0.125, head_dim=64,
                          dropout=(P_DROP, torch.tensor([SEED], dtype=torch.int64, device=DEV), SITE))[2]
    assert torch.equal(bits64, res[2])


# ------------------------------------------------------------------------------------------------------------ models
V1_CFG = dict(vocab_size=2025, max_position_embeddings=257, hidden_size=256, num_hidden_layers=2, num_attention_heads=2,
              intermediate_size=512, codebook_size=1024, num_vq_tokens=256, num_classes=1000, hidden_dropout=0.0,
              attention_dropout=0.0)
UVIT_CFG = dict(hidden_size=256, num_attention_heads=2, in_channels=192, block_out_channels=(192,), block_num_heads=2,
                num_res_blocks=1, num_hidden_layers=2, intermediate_size=512, vocab_size=72, codebook_size=64,
                encoder_hidden_size=32, cond_embed_dim=16, micro_cond_encode_dim=8, micro_cond_embed_dim=40,
                norm_type="rmsnorm", hidden_dropout=0.0, attention_dropout=0.0)


def _v1_batch(B, seed):
    g = torch.Generator().manual_seed(seed)
    tokens = torch.randint(0, 1024, (B, 256), generator=g)
    cls = torch.randint(0, 1000, (B,), generator=g)
    return T.mask_tokens(tokens, cls, torch.rand(B, generator=g), torch.rand(B, 256, generator=g), 1024, 2024)


def _grad_report(errs, cos):
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:6]
    print("worst grad rel-L2 (bound 6e-2, query / key weights excepted):", ", ".join(f"{k}={v:.2e}" for k, v in worst))
    print(f"min grad cosine {min(cos.values()):.5f} (bound 0.998)")
    # DESIGN.md section 2: <= 6e-2 per parameter with cosine >= 0.998; only attention query / key weights may exceed it
    above = {k: v for k, v in errs.items() if v > 6e-2}
    assert all(".query." in k or ".key." in k for k in above) and len(above) <= 2, above
    assert all(cos[k] >= 0.998 for k in errs if k not in above), sorted(cos.items(), key=lambda kv: kv[1])[:5]


def test_maskgit_transformer_head_dim_128_vs_oracle():
    """hidden 256 / 2 heads: logits, loss and every gradient of one bf16 training step against the oracle's fp32 autograd"""
    torch.manual_seed(0)
    m = MaskGitTransformer(**V1_CFG)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    inp, lab = _v1_batch(2, 1)
    ref_logits, ref_loss, ref_grads = T.forward_backward(sd, V1_CFG, inp, lab)
    m.to(DEV).train()
    with torch.autocast("cuda", dtype=BF):
        logits, loss = m(inp.to(DEV), labels=lab.to(DEV))
    loss.backward()
    rel = _rel(logits, ref_logits)
    lrel = abs(float(loss.detach()) - float(ref_loss)) / float(ref_loss)
    print(f"logits rel-L2 {rel:.3e} (bound 1e-2), loss rel {lrel:.3e} (bound 2e-3)")
    assert rel < 1e-2
    assert abs(float(loss) - float(ref_loss)) < 2e-3 * float(ref_loss)
    params = dict(m.named_parameters())
    errs = {n: _rel(params[n].grad, ref_grads[n]) for n in ref_grads}
    cos = {n: float(torch.nn.functional.cosine_similarity(params[n].grad.float().cpu().flatten(), ref_grads[n].flatten(),
                                                          dim=0)) for n in ref_grads}
    _grad_report(errs, cos)
    m.eval()
    with torch.no_grad():
        ids = m.generate2(class_ids=torch.tensor([1, 5], device=DEV), timesteps=4, guidance_scale=2.0,
                          generator=torch.Generator(device=DEV).manual_seed(3))
    assert ids.shape == (2, 256) and int(ids.min()) >= 0 and int(ids.max()) < 1024


def _uvit_inputs(B, S, seed):
    g = torch.Generator().manual_seed(seed)
    ids, lab = torch.randint(0, 64, (B, S), generator=g), torch.randint(0, 64, (B, S), generator=g)
    enc, ce, mc = torch.randn(B, 5, 32, generator=g), torch.randn(B, 16, generator=g), torch.rand(B, 5, generator=g) * 100
    return ids, lab, enc, ce, mc


@pytest.mark.parametrize("downup", [False, True])
def test_uvit_head_dims_128_and_96_vs_oracle(downup):
    """head_dim 128 in the transformer layers (256 / 2) and 96 in the block attentions (192 / 2): logits, loss and every
    gradient against the oracle's fp32 autograd, then generate2 with classifier-free guidance to completion"""
    cfg = dict(UVIT_CFG, force_down_up_sample=downup)
    torch.manual_seed(3)
    m = MaskGiTUViT_v2(**cfg)
    with torch.no_grad():
        for p in m.parameters():  # adaLN mappers and GRN parameters are zeros at init
            p.add_((0.1 if p.dim() == 1 else 0.02) * torch.randn_like(p))
    ids, lab, enc, ce, mc = _uvit_inputs(2, 64, 4)
    q = {k: v.detach().clone().float().requires_grad_(True) for k, v in m.state_dict().items()}
    ref_logits, ref_loss = V2.forward(q, dict(m.config), ids, enc, ce, mc, labels=lab)
    ref_loss.backward()
    m.to(DEV).train()
    with torch.autocast("cuda", dtype=BF):
        logits, loss = m(ids.to(DEV), enc.to(DEV), ce.to(DEV), mc.to(DEV), labels=lab.to(DEV))
    loss.backward()
    rel = _rel(logits, ref_logits)
    lrel = abs(float(loss.detach()) - float(ref_loss)) / float(ref_loss)
    print(f"logits rel-L2 {rel:.3e} (bound 1e-2), loss rel {lrel:.3e} (bound 2e-3)")
    assert rel < 1e-2
    assert abs(float(loss) - float(ref_loss)) < 2e-3 * float(ref_loss)
    errs = {n: _rel(p.grad, q[n].grad) for n, p in m.named_parameters()}
    cos = {n: float(torch.nn.functional.cosine_similarity(p.grad.float().cpu().flatten(), q[n].grad.flatten(), dim=0))
           for n, p in m.named_parameters()}
    _grad_report(errs, cos)
    m.eval()
    with torch.no_grad():
        kw = dict(encoder_hidden_states=enc.to(DEV), cond_embeds=ce.to(DEV), micro_conds=mc.to(DEV),
                  empty_embeds=torch.zeros(1, 5, 32, device=DEV), empty_cond_embeds=torch.zeros(1, 16, device=DEV),
                  temperature=(2.0, 0.0), timesteps=4, seq_len=64, guidance_scale=3.0)
        a = m.generate2(**kw, generator=torch.Generator(device=DEV).manual_seed(5))
        b = m.generate2(**kw, generator=torch.Generator(device=DEV).manual_seed(5))
    assert a.shape == (2, 64) and torch.equal(a, b) and int(a.min()) >= 0 and int(a.max()) < 64


def test_uvit_fp8_inference_at_head_dims_128_and_96():
    """set_gemm_precision("fp8") keeps attention in bf16: with 128- and 96-wide heads the no_grad forward and a guided
    generate2 run, the logits stay near the bf16 ones (the sanity bound of tests/test_fp8_gpu.py's micro fixture), and
    switching back to bf16 gives the bf16 logits bit for bit"""
    torch.manual_seed(3)
    m = MaskGiTUViT_v2(**UVIT_CFG)
    with torch.no_grad():
        for p in m.parameters():
            p.add_((0.1 if p.dim() == 1 else 0.02) * torch.randn_like(p))
    m.to(DEV).eval()
    ids, _, enc, ce, mc = (t.to(DEV) for t in _uvit_inputs(2, 64, 4))
    with torch.no_grad():
        ref = m(ids, enc, ce, mc)
        m.set_gemm_precision("fp8")
        out = m(ids, enc, ce, mc)
        kw = dict(encoder_hidden_states=enc, cond_embeds=ce, micro_conds=mc, empty_embeds=torch.zeros(1, 5, 32, device=DEV),
                  empty_cond_embeds=torch.zeros(1, 16, device=DEV), timesteps=4, seq_len=64, guidance_scale=3.0)
        gen = m.generate2(**kw, generator=torch.Generator(device=DEV).manual_seed(5))
        m.set_gemm_precision("bf16")
        again = m(ids, enc, ce, mc)
    print(f"FP8 vs bf16 logits rel-L2 {_rel(out, ref):.3e} (bound 0.1)")
    assert torch.isfinite(out).all() and _rel(out, ref) < 0.1 and torch.equal(again, ref)
    assert gen.shape == (2, 64) and int(gen.min()) >= 0 and int(gen.max()) < 64


def test_head_dim_128_train_step_gradients_are_bit_reproducible():
    """Three identical forward + backward passes at head_dim 128 give bit-identical logits, loss and gradients"""
    torch.manual_seed(0)
    m = MaskGitTransformer(**V1_CFG).to(DEV).train()
    inp, lab = (t.to(DEV) for t in _v1_batch(24, 5))
    runs = []
    for _ in range(3):
        m.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=BF):
            logits, loss = m(inp, labels=lab)
        loss.backward()
        torch.cuda.synchronize()
        runs.append((logits.clone(), loss.clone(), {n: p.grad.clone() for n, p in m.named_parameters()}))
    for other in runs[1:]:
        assert torch.equal(runs[0][0], other[0]) and torch.equal(runs[0][1], other[1])
        for n, gr in runs[0][2].items():
            assert torch.equal(gr, other[2][n]), n


def test_attention_dropout_masks_replay_in_the_reference_at_head_dim_128():
    """Training with attention and hidden dropout at head_dim 128: the masks recorded with ops.dropout_record, handed to
    the unmodified reference in fp32, give the same logits, loss and gradients (the HD-64 dropout tolerances)"""
    from oracle.ref_snapshot import import_reference
    from tests.test_dropout_cpu import _Replay

    cfg = dict(V1_CFG, hidden_dropout=0.1, attention_dropout=0.1)
    inp, lab = _v1_batch(2, 7)
    torch.manual_seed(3)
    m = MaskGitTransformer(**cfg).to(DEV).train()
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    torch.manual_seed(4)
    with ops.dropout_record() as log:
        logits, loss = m(inp.to(DEV), labels=lab.to(DEV))
    loss.backward()
    masks = {s: b.cpu() for s, b in log}
    ref = import_reference().MaskGitTransformer(**cfg).to(DEV)
    ref.load_state_dict(sd)
    ref.train()
    sc = keep_scale(0.1)
    replay = lambda site, n: _Replay(unpack_bits(masks[site], n).to(DEV), sc)  # noqa: E731
    ref.embed.dropout = replay(0, cfg["hidden_size"])
    for i, layer in enumerate(ref.transformer_layers):
        layer.attention.dropout = replay(1 + 3 * i, inp.shape[1])
        layer.ffn.dropout = replay(3 + 3 * i, cfg["intermediate_size"])
    r_logits, r_loss = ref(inp.to(DEV), labels=lab.to(DEV))
    r_loss.backward()
    print(f"dropout replay: logits rel-L2 {_rel(logits, r_logits):.3e} (bound 1e-2)")
    assert _rel(logits, r_logits) < 1e-2
    assert abs(float(loss) - float(r_loss)) < 2e-3 * abs(float(r_loss))
    above = [(n, _rel(dict(m.named_parameters())[n].grad, p.grad)) for n, p in ref.named_parameters()
             if _rel(dict(m.named_parameters())[n].grad, p.grad) >= 6e-2]
    assert all("attention.query" in n or "attention.key" in n for n, _ in above) and len(above) <= 2, above


# ------------------------------------------------------------------------------------------------ scaled-up models
def test_cc12m_width_transformer_with_8_heads_trains_and_samples():
    """hidden 1024 / 8 heads (head_dim 128), intermediate 4096, RMSNorm, cross-attention on 77 x 768 text states: one
    FusedAdamW step and a guided generate2"""
    cfg = dict(vocab_size=8256, max_position_embeddings=256, hidden_size=1024, num_hidden_layers=2, num_attention_heads=8,
               intermediate_size=4096, add_cross_attention=True, encoder_hidden_size=768, codebook_size=8192,
               num_vq_tokens=256, norm_type="rmsnorm", use_encoder_layernorm=True, use_codebook_size_for_output=True,
               hidden_dropout=0.0, attention_dropout=0.0)
    torch.manual_seed(0)
    m = MaskGitTransformer(**cfg).to(DEV).train()
    g = torch.Generator().manual_seed(1)
    B = 4
    ids = torch.randint(0, 8192, (B, 256), generator=g)
    mask = torch.rand(B, 256, generator=g) < 0.5
    inp, lab = torch.where(mask, 8255, ids).to(DEV), torch.where(mask, ids, -100).to(DEV)
    enc = torch.randn(B, 77, 768, generator=g).to(DEV)
    opt = FusedAdamW(m.parameters(), lr=1e-4, weight_decay=0.01, model=m)
    before = {n: p.detach().clone() for n, p in m.named_parameters()}
    with torch.autocast("cuda", dtype=BF):
        _, loss = m(inp, labels=lab, encoder_hidden_states=enc)
    loss.backward()
    assert all(torch.isfinite(p.grad).all() for p in m.parameters())
    opt.step()
    assert all(not torch.equal(before[n], p.detach()) for n, p in m.named_parameters())
    m.eval()
    with torch.no_grad():
        out = m.generate2(encoder_hidden_states=enc[:2], negative_embeds=torch.zeros(2, 77, 768, device=DEV),
                          timesteps=4, guidance_scale=2.0, generator=torch.Generator(device=DEV).manual_seed(2))
    assert out.shape == (2, 256) and int(out.min()) >= 0 and int(out.max()) < 8192


def test_uvit_class_defaults_with_8_and_6_heads_trains_and_samples():
    """MaskGiTUViT_v2 at its class defaults with num_attention_heads 8 (1024 / 8 = 128) and block_num_heads 6 (768 / 6 =
    128): one FusedAdamW step and a guided generate2"""
    torch.manual_seed(0)
    m = MaskGiTUViT_v2(num_attention_heads=8, block_num_heads=6).to(DEV).train()
    c = m.config
    g = torch.Generator().manual_seed(1)
    B = 2
    ids = torch.randint(0, c.codebook_size, (B, 256), generator=g)
    mask = torch.rand(B, 256, generator=g) < 0.5
    inp, lab = torch.where(mask, c.mask_token_id, ids).to(DEV), torch.where(mask, ids, -100).to(DEV)
    enc = torch.randn(B, 77, c.encoder_hidden_size, generator=g).to(DEV)
    ce = torch.randn(B, c.cond_embed_dim, generator=g).to(DEV)
    mc = torch.tensor([[256.0, 256.0, 0.0, 0.0, 6.0], [512.0, 512.0, 32.0, 16.0, 5.0]], device=DEV)
    opt = FusedAdamW(m.parameters(), lr=1e-4, weight_decay=0.01, model=m)
    with torch.autocast("cuda", dtype=BF):
        _, loss = m(inp, enc, ce, mc, labels=lab)
    loss.backward()
    assert torch.isfinite(loss) and all(torch.isfinite(p.grad).all() for p in m.parameters() if p.grad is not None)
    opt.step()
    m.eval()
    with torch.no_grad():
        out = m.generate2(encoder_hidden_states=enc, cond_embeds=ce, micro_conds=mc,
                          empty_embeds=torch.zeros(1, 77, c.encoder_hidden_size, device=DEV),
                          empty_cond_embeds=torch.zeros(1, c.cond_embed_dim, device=DEV), timesteps=4, guidance_scale=3.0,
                          generator=torch.Generator(device=DEV).manual_seed(2))
    assert out.shape == (B, 256) and int(out.min()) >= 0 and int(out.max()) < c.codebook_size
