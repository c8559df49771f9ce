"""GPU parity of the MaskGiTUViT_v2 inference path: new kernels vs fp32 torch math, the assembled model vs the reference
fixture (micro) and vs the pinned oracle at U-ViT-sized widths, CFG generate2 properties."""
import math
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from open_muse_b200 import MaskGiTUViT_v2, ops  # noqa: E402
from oracle import transformer_v2_oracle as V2  # noqa: E402

DEV = "cuda"


def _rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-20))


@pytest.mark.parametrize("H,rms,with_res,with_mod,a_bf16", [(1024, 1, True, True, True), (768, 0, True, False, True),
                                                           (64, 1, False, True, False), (128, 0, True, True, False)])
def test_add_norm_mod_vs_torch(H, rms, with_res, with_mod, a_bf16):
    g = torch.Generator().manual_seed(H)
    B, S = 3, 20
    a = torch.randn(B * S, H, generator=g)
    a = a.to(torch.bfloat16) if a_bf16 else a
    r = torch.randn(B * S, H, generator=g) if with_res else None
    w = 1 + 0.1 * torch.randn(H, generator=g)
    mod_all = torch.randn(B, 4 * H + 64, generator=g) * 0.3
    mod = mod_all[:, 64:64 + 2 * H] if with_mod else None
    x = a.float() + (r if with_res else 0)
    if rms:
        y = x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + 1e-6) * w
    else:
        y = torch.nn.functional.layer_norm(x, (H,), w, None, 1e-6)
    if with_mod:
        y = (y.view(B, S, H) * (1 + mod[:, None, :H]) + mod[:, None, H:]).view(B * S, H)
    mod_dev = mod_all.to(DEV)[:, 64:64 + 2 * H] if with_mod else None
    r_out, yk = ops.add_norm_mod(a.to(DEV), w.to(DEV), 1e-6, rms, residual=None if r is None else r.to(DEV), mod=mod_dev,
                                 rows_per_sample=S)
    assert torch.allclose(r_out.cpu(), x, atol=1e-6) and _rel(yk, y) < 5e-3
    _, yf = ops.add_norm_mod(a.to(DEV), w.to(DEV), 1e-6, rms, out_dtype=torch.float32, residual=None if r is None else r.to(DEV),
                             mod=mod_dev, rows_per_sample=S, want_residual=False)
    assert _rel(yf, y) < 1e-5


@pytest.mark.parametrize("C,hw,rms", [(768, 16, 1), (64, 4, 0), (1024, 8, 1)])
def test_dwconv_norm_grn_adaln_silu_vs_torch(C, hw, rms):
    g = torch.Generator().manual_seed(C)
    B = 2
    x = torch.randn(B, hw, hw, C, generator=g)
    wd = torch.randn(C, 1, 3, 3, generator=g) * 0.3
    nw = 1 + 0.1 * torch.randn(C, generator=g)
    conv = torch.nn.functional.conv2d(x.permute(0, 3, 1, 2), wd, None, padding=1, groups=C).permute(0, 2, 3, 1)
    conv = conv.to(torch.bfloat16).float()
    ref = conv * torch.rsqrt(conv.pow(2).mean(-1, keepdim=True) + 1e-6) * nw if rms else \
        torch.nn.functional.layer_norm(conv, (C,), nw, None, 1e-6)
    y = ops.dwconv3x3_norm(x.view(-1, C).to(DEV), wd.view(C, 9).t().contiguous().to(DEV), nw.to(DEV), B, hw, hw, 1e-6, rms)
    assert _rel(y, ref.view(-1, C)) < 6e-3
    # GELU + GRN
    z = (torch.randn(B, hw, hw, C, generator=g) * 1.5).to(torch.bfloat16)
    gamma, beta = torch.randn(C, generator=g) * 0.2, torch.randn(C, generator=g) * 0.2
    gg = torch.nn.functional.gelu(z.float()).to(torch.bfloat16).float()
    gx = torch.norm(gg, p=2, dim=(1, 2), keepdim=True)
    nx = gx / (gx.mean(dim=-1, keepdim=True) + 1e-6)
    ref = gamma * (gg * nx) + beta + gg
    out = ops.grn(z.view(-1, C).to(DEV), gamma.to(DEV), beta.to(DEV), B, hw * hw)
    assert _rel(out, ref.view(-1, C)) < 6e-3
    # in-place adaLN and SiLU
    mod = torch.randn(B, 2 * C + 32, generator=g)
    h = torch.randn(B * hw * hw, C, generator=g)
    ref = (h.view(B, -1, C) * (1 + mod[:, None, 32:32 + C]) + mod[:, None, 32 + C:32 + 2 * C]).view(-1, C)
    hk = ops.adaln_apply_(h.to(DEV).clone(), mod.to(DEV)[:, 32:32 + 2 * C], B, hw * hw)
    assert _rel(hk, ref) < 1e-6
    s = ops.silu_bf16(h.to(DEV))
    assert _rel(s, torch.nn.functional.silu(h)) < 5e-3


def _stage_report(m, ref_stages):
    rep = []
    for k, v in m._debug_stages.items():
        if k in ref_stages:
            rep.append(f"{k}={_rel(v, ref_stages[k]):.2e}")
    return " ".join(rep)


def test_micro_uvit_v2_vs_reference_fixture(golden):
    g = golden("micro_uvit_v2.pt")
    m = MaskGiTUViT_v2(**g["config"])
    m.load_state_dict(g["state_dict"])
    m.to(DEV).eval()
    st = {}
    with torch.no_grad():
        V2.forward(g["state_dict"], g["config"], g["input_ids"], g["encoder_hidden_states"], g["cond_embeds"],
                   g["micro_conds"], stages=st)
    m._debug_stages = {}
    args = [g[k].to(DEV) for k in ("input_ids", "encoder_hidden_states", "cond_embeds", "micro_conds")]
    with torch.autocast("cuda", dtype=torch.bfloat16):
        logits, loss = m(*args, labels=g["labels"].to(DEV), label_smoothing=0.1)
    print("stages:", _stage_report(m, st))
    m._debug_stages = None
    assert logits.dtype == torch.bfloat16 and logits.shape == g["logits"].shape
    assert _rel(logits, g["logits"]) < 2e-2, _rel(logits, g["logits"])
    assert abs(float(loss) - float(g["loss"])) / float(g["loss"]) < 2e-3
    _, loss_w = m(*args, labels=g["labels"].to(DEV), loss_weight=g["loss_weight"].to(DEV))
    assert abs(float(loss_w) - float(g["loss_weighted"])) / float(g["loss_weighted"]) < 2e-3
    out = m(*args)
    assert out.dtype == torch.float32 and _rel(out, g["logits"]) < 2e-2


def test_micro_uvit_v2_force_down_up_sample_vs_reference_fixture(golden):
    """force_down_up_sample=True (reference :505-583): the k2s2 conv and the ConvTranspose2d run as patch GEMMs; stages,
    logits, loss and the generate2 trace against the fixture made by the unmodified reference (8x8 tokens, 4x4 inside)."""
    g = golden("micro_uvit_v2_downup.pt")
    m = MaskGiTUViT_v2(**g["config"])
    m.load_state_dict(g["state_dict"])
    m.to(DEV).eval()
    m._debug_stages = {}
    args = [g[k].to(DEV) for k in ("input_ids", "encoder_hidden_states", "cond_embeds", "micro_conds")]
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        logits, loss = m(*args, labels=g["labels"].to(DEV), label_smoothing=0.1)
    st = m._debug_stages
    m._debug_stages = None
    print("stages:", " ".join(f"{k}={_rel(st[k], g['stages'][k]):.2e}" for k in ("downsample", "upsample")))
    assert st["downsample"].shape == g["stages"]["downsample"].shape and st["upsample"].shape == g["stages"]["upsample"].shape
    assert _rel(st["downsample"], g["stages"]["downsample"]) < 1e-2
    assert _rel(st["upsample"], g["stages"]["upsample"]) < 2e-2
    assert logits.shape == g["logits"].shape and _rel(logits, g["logits"]) < 2e-2, _rel(logits, g["logits"])
    assert abs(float(loss) - float(g["loss"])) / float(g["loss"]) < 2e-3
    ids = m.generate2(*args[1:], g["empty_embeds"].to(DEV), g["empty_cond_embeds"].to(DEV), temperature=(2.0, 0.0),
                      timesteps=4, guidance_scale=3.0, seq_len=64, generator=torch.Generator(DEV).manual_seed(g["gen_seed"]))
    assert ids.shape == g["gen_ids"].shape and int(ids.min()) >= 0 and int(ids.max()) < 64


def test_micro_uvit_v2_force_down_up_sample_training_gradients_vs_oracle(golden):
    """Training with force_down_up_sample=True (the 512-px configs, configs/research_run_512_with_downsample*.yaml): the
    strided conv / transposed conv train as patch GEMMs (uvit_v2_train.ResampleFn).  Loss and EVERY gradient -- incl. the
    Conv2d [co, ci, 2, 2] and ConvTranspose2d [ci, co, 2, 2] weights and their Norm2D weights -- against the oracle's fp32
    autograd on the reference fixture weights (the oracle's forward is pinned to the unmodified reference's stages)."""
    g = golden("micro_uvit_v2_downup.pt")
    assert g["config"]["force_down_up_sample"]
    q = {k: v.clone().requires_grad_(True) for k, v in g["state_dict"].items()}
    _, ref_loss = V2.forward(q, g["config"], g["input_ids"], g["encoder_hidden_states"], g["cond_embeds"], g["micro_conds"],
                             labels=g["labels"], label_smoothing=0.1)
    ref_loss.backward()
    m = MaskGiTUViT_v2(**g["config"])
    m.load_state_dict(g["state_dict"])
    m.to(DEV).train()
    args = [g[k].to(DEV) for k in ("input_ids", "encoder_hidden_states", "cond_embeds", "micro_conds")]
    with torch.autocast("cuda", dtype=torch.bfloat16):
        logits, loss = m(*args, labels=g["labels"].to(DEV), label_smoothing=0.1)
    loss.backward()
    assert logits.shape == g["logits"].shape and _rel(logits, g["logits"]) < 2e-2
    assert abs(float(loss) - float(ref_loss)) / float(ref_loss) < 2e-3
    errs = {}
    for n, p in m.named_parameters():
        assert p.grad is not None and p.grad.shape == p.shape, n
        errs[n] = _rel(p.grad, q[n].grad)
    resample = {k: v for k, v in errs.items() if "sample" in k}
    print("resampling grads rel-L2:", ", ".join(f"{k}={v:.2e}" for k, v in resample.items()))
    assert len(resample) >= 2 and max(resample.values()) < 6e-2, resample
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:8]
    print("worst grad rel-L2:", ", ".join(f"{k}={v:.2e}" for k, v in worst))
    bad = {k: v for k, v in errs.items() if v > 8e-2 and not (".query." in k or ".key." in k)}
    assert not bad, bad


def test_uvit_v2_default_widths_vs_oracle():
    """U-ViT widths of the cc12m configs (hidden 1024 / 16 heads, blocks 768 / 12 heads, kv_mapper, 256 tokens, 77 text
    states) with a shortened stack, random re-draw of the zero-initialised tensors; fp32 oracle on the CPU."""
    cfg = dict(num_hidden_layers=2, num_res_blocks=1, vocab_size=1032, codebook_size=1024, intermediate_size=2816)
    torch.manual_seed(0)
    m = MaskGiTUViT_v2(**cfg)
    gen = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for k, x in m.state_dict().items():
            if "adaLN_modulation.mapper" in k or k.endswith("gamma") or k.endswith("beta") or k == "mlm_layer.conv1.weight":
                x.copy_(torch.randn(x.shape, generator=gen) * 0.03)
    B = 2
    ids = torch.randint(0, 1024, (B, 256), generator=gen)
    ids[torch.rand(B, 256, generator=gen) < 0.5] = 1031
    enc = torch.randn(B, 77, 768, generator=gen)
    ce = torch.randn(B, 768, generator=gen)
    mc = torch.tensor([[256.0, 256.0, 0.0, 0.0, 6.0], [512.0, 512.0, 32.0, 16.0, 5.0]])
    st = {}
    with torch.no_grad():
        ref = V2.forward({k: v.float() for k, v in m.state_dict().items()}, cfg, ids, enc, ce, mc, stages=st)
    m.to(DEV).eval()
    m._debug_stages = {}
    with torch.autocast("cuda", dtype=torch.bfloat16):
        logits = m(ids.to(DEV), enc.to(DEV), ce.to(DEV), mc.to(DEV))
    print("stages:", _stage_report(m, st))
    assert _rel(logits, ref) < 2e-2, _rel(logits, ref)
    agree = float((logits.float().cpu().argmax(-1) == ref.argmax(-1)).float().mean())
    assert agree > 0.9, agree


def test_uvit_v2_generate2_cfg_properties(golden):
    g = golden("micro_uvit_v2.pt")
    m = MaskGiTUViT_v2(**g["config"])
    m.load_state_dict(g["state_dict"])
    m.to(DEV).eval()
    kw = dict(encoder_hidden_states=g["encoder_hidden_states"].to(DEV), cond_embeds=g["cond_embeds"].to(DEV),
              micro_conds=g["micro_conds"][:1].to(DEV), empty_embeds=g["empty_embeds"].to(DEV),
              empty_cond_embeds=g["empty_cond_embeds"].to(DEV), temperature=(2.0, 0.0), timesteps=4, seq_len=16)
    a = m.generate2(**kw, guidance_scale=3.0, generator=torch.Generator(device=DEV).manual_seed(5))
    b = m.generate2(**kw, guidance_scale=3.0, generator=torch.Generator(device=DEV).manual_seed(5))
    assert a.shape == (3, 16) and a.dtype == torch.int64 and torch.equal(a, b)
    assert int(a.min()) >= 0 and int(a.max()) < 64  # no mask tokens left, codebook range
    ids, inter = m.generate2(**kw, guidance_scale=3.0, guidance_schedule="linear", return_intermediate=True,
                             generator=torch.Generator(device=DEV).manual_seed(5))
    # the intermediates are the RAW per-step samples (the reference's semantics, pinned on the CPU by
    # tests/test_uvit_numeric_cpu.py::test_uvit_generate2_intermediates_are_the_raw_samples_of_the_reference)
    assert len(inter) == 4 and all(t.shape == ids.shape and t.dtype == torch.int64 for t in inter)
    assert all(int(t.min()) >= 0 and int(t.max()) < 64 for t in inter)
    # the CUDA-graph replay of the step forward is bit-identical to launching the kernels one by one
    e = m.generate2(**kw, guidance_scale=3.0, use_cuda_graph=False, generator=torch.Generator(device=DEV).manual_seed(5))
    assert torch.equal(a, e) and m._graph is not None
    # partially given tokens are kept
    start = torch.full((3, 16), 71, dtype=torch.long, device=DEV)
    start[:, :5] = torch.arange(5, device=DEV)
    c = m.generate2(**kw, guidance_scale=2.0, input_ids=start, generator=torch.Generator(device=DEV).manual_seed(6))
    assert torch.equal(c[:, :5], start[:, :5]) and int(c.max()) < 64


def test_pipeline_with_uvit_v2_and_checkpoint_roundtrip(tmp_path, golden):
    """PipelineMuse(text-conditioned U-ViT + MaskGitVQGAN detokeniser) from precomputed text embeddings, and the
    <dir>/{vae,transformer} layout through save_pretrained / from_pretrained (class name dispatch)."""
    from open_muse_b200 import MaskGitVQGAN, PipelineMuse

    g = golden("micro_uvit_v2.pt")
    tr = MaskGiTUViT_v2(**g["config"])
    tr.load_state_dict(g["state_dict"])
    torch.manual_seed(0)
    vae = MaskGitVQGAN(resolution=8, hidden_channels=32, channel_mult=(1, 2), num_res_blocks=1, z_channels=16,
                       num_embeddings=64, quantized_embed_dim=16)
    pipe = PipelineMuse(vae=vae, transformer=tr, is_class_conditioned=False).to(DEV)
    kw = dict(prompt_embeds=g["encoder_hidden_states"][:2], pooled_embeds=g["cond_embeds"][:2],
              negative_prompt_embeds=g["empty_embeds"].expand(2, -1, -1), negative_pooled_embeds=g["empty_cond_embeds"].expand(2, -1),
              timesteps=3, guidance_scale=2.0, num_images_per_prompt=2, output_type="pt")
    a = pipe(**kw, generator=torch.Generator(device=DEV).manual_seed(1))
    assert a.shape == (4, 3, 32, 32) and bool(torch.isfinite(a).all())  # 256 tokens = 16x16 latent, f = 2
    pipe.save_pretrained(tmp_path)
    assert sorted(os.listdir(tmp_path)) == ["transformer", "vae"]
    pipe2 = PipelineMuse.from_pretrained(str(tmp_path), is_class_conditioned=True).to(DEV)
    pipe2.is_class_conditioned = False
    assert isinstance(pipe2.transformer, MaskGiTUViT_v2)
    b = pipe2(**kw, generator=torch.Generator(device=DEV).manual_seed(1))
    assert torch.equal(a, b)


@pytest.mark.parametrize("C,hw,rms", [(768, 16, 1), (64, 4, 0)])
def test_uvit_backward_kernels_vs_autograd(C, hw, rms):
    """add_norm_mod / dwconv+norm / GELU+GRN / adaLN / SiLU backward kernels against torch autograd of the fp32 math."""
    g = torch.Generator().manual_seed(C + hw)
    B, S = 2, hw * hw
    T = B * S
    dev = lambda t: t.to(DEV)
    # ---- add_norm_mod
    a = torch.randn(T, C, generator=g).requires_grad_(True)
    r = torch.randn(T, C, generator=g).requires_grad_(True)
    w = (1 + 0.1 * torch.randn(C, generator=g)).requires_grad_(True)
    mod = (torch.randn(B, 2 * C, generator=g) * 0.3).requires_grad_(True)
    x = a + r
    n = x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + 1e-6) * w if rms else torch.nn.functional.layer_norm(x, (C,), w, None, 1e-6)
    y = (n.view(B, S, C) * (1 + mod[:, None, :C]) + mod[:, None, C:]).view(T, C)
    dy, dro = torch.randn(T, C, generator=g), torch.randn(T, C, generator=g)
    (y * dy).sum().backward(retain_graph=True)
    (x * dro).sum().backward()
    mod_d, dmod, dw = dev(mod.detach()), torch.zeros(B, 2 * C, device=DEV), torch.zeros(C, device=DEV)
    da, dr = ops.add_norm_mod_bwd(dev(dy), dev(dro), dev(x.detach()), dev(w.detach()), 1e-6, rms, torch.float32, mod=mod_d,
                                  rows_per_sample=S, dw=dw, dmod=dmod)
    assert _rel(da, a.grad) < 1e-4 and _rel(dr, r.grad) < 1e-4 and _rel(dw, w.grad) < 1e-4 and _rel(dmod, mod.grad) < 1e-4
    # ---- depthwise conv + norm
    xin = torch.randn(B, hw, hw, C, generator=g).requires_grad_(True)
    wd = (torch.randn(C, 1, 3, 3, generator=g) * 0.3).requires_grad_(True)
    nw = (1 + 0.1 * torch.randn(C, generator=g)).requires_grad_(True)
    conv = torch.nn.functional.conv2d(xin.permute(0, 3, 1, 2), wd, None, padding=1, groups=C).permute(0, 2, 3, 1)
    out = conv * torch.rsqrt(conv.pow(2).mean(-1, keepdim=True) + 1e-6) * nw if rms else torch.nn.functional.layer_norm(conv, (C,), nw, None, 1e-6)
    dyc = torch.randn(B, hw, hw, C, generator=g).to(torch.bfloat16)
    (out * dyc.float()).sum().backward()
    wk = dev(wd.detach().view(C, 9).t().contiguous())
    yk, convk = ops.dwconv3x3_norm(dev(xin.detach().view(T, C)), wk, dev(nw.detach()), B, hw, hw, 1e-6, rms, save_conv=True)
    dwk, dnw = torch.zeros(9, C, device=DEV), torch.zeros(C, device=DEV)
    dres = torch.randn(T, C, generator=g)
    dx = ops.dwconv3x3_norm_bwd(dev(dyc.view(T, C)), convk, dev(xin.detach().view(T, C)), wk, dev(nw.detach()), dev(dres), dwk,
                                dnw, B, hw, hw, 1e-6, rms)
    assert _rel(dx.cpu() - dres, xin.grad.view(T, C)) < 1e-2
    assert _rel(dwk.t().reshape(C, 1, 3, 3), wd.grad) < 1e-2 and _rel(dnw, nw.grad) < 1e-2
    # ---- GELU + GRN
    z = (torch.randn(B, hw, hw, C, generator=g) * 1.5).to(torch.bfloat16)
    zf = z.float().requires_grad_(True)
    gamma = (torch.randn(C, generator=g) * 0.2).requires_grad_(True)
    beta = (torch.randn(C, generator=g) * 0.2).requires_grad_(True)
    gg = torch.nn.functional.gelu(zf)
    gx = torch.norm(gg, p=2, dim=(1, 2), keepdim=True)
    og = gamma * (gg * (gx / (gx.mean(dim=-1, keepdim=True) + 1e-6))) + beta + gg
    dog = torch.randn(B, hw, hw, C, generator=g).to(torch.bfloat16)
    (og * dog.float()).sum().backward()
    _, stats = ops.grn(dev(z.view(T, C)), dev(gamma.detach()), dev(beta.detach()), B, S, save_stats=True)
    dgam, dbet = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    dz = ops.grn_bwd(dev(z.view(T, C)), dev(dog.view(T, C)), stats, dev(gamma.detach()), dgam, dbet, B, S)
    assert _rel(dz, zf.grad.view(T, C)) < 1.5e-2 and _rel(dgam, gamma.grad) < 1e-2 and _rel(dbet, beta.grad) < 1e-2
    # ---- adaLN apply and SiLU
    h = torch.randn(T, C, generator=g).requires_grad_(True)
    m2 = (torch.randn(B, 2 * C, generator=g) * 0.5).requires_grad_(True)
    o2 = (h.view(B, S, C) * (1 + m2[:, None, :C]) + m2[:, None, C:]).view(T, C)
    do2 = torch.randn(T, C, generator=g)
    (o2 * do2).sum().backward()
    dm2 = torch.zeros(B, 2 * C, device=DEV)
    dh = ops.adaln_bwd(dev(do2), dev(h.detach()), dev(m2.detach()), dm2, B, S)
    assert _rel(dh, h.grad) < 1e-5 and _rel(dm2, m2.grad) < 1e-4
    sx = torch.randn(T, C, generator=g).requires_grad_(True)
    dsy = torch.randn(T, C, generator=g).to(torch.bfloat16)
    (torch.nn.functional.silu(sx) * dsy.float()).sum().backward()
    acc = torch.ones(T, C, device=DEV)
    ops.silu_bwd(dev(dsy), dev(sx.detach()), out=acc)
    assert _rel(acc.cpu() - 1, sx.grad) < 1e-4
    assert _rel(ops.silu_bwd(dev(dsy), dev(sx.detach().to(torch.bfloat16))), sx.grad) < 1.5e-2


def test_micro_uvit_v2_training_gradients_vs_oracle(golden):
    """One training forward/backward of MaskGiTUViT_v2 (hand-written backward through every block) against the oracle's fp32
    autograd on the reference fixture weights; then a few optimizer steps must reduce the loss."""
    g = golden("micro_uvit_v2.pt")
    q = {k: v.clone().requires_grad_(True) for k, v in g["state_dict"].items()}
    _, ref_loss = V2.forward(q, g["config"], g["input_ids"], g["encoder_hidden_states"], g["cond_embeds"], g["micro_conds"],
                             labels=g["labels"], label_smoothing=0.1)
    ref_loss.backward()
    m = MaskGiTUViT_v2(**g["config"])
    m.load_state_dict(g["state_dict"])
    m.to(DEV).train()
    args = [g[k].to(DEV) for k in ("input_ids", "encoder_hidden_states", "cond_embeds", "micro_conds")]
    with torch.autocast("cuda", dtype=torch.bfloat16):
        logits, loss = m(*args, labels=g["labels"].to(DEV), label_smoothing=0.1)
    loss.backward()
    assert abs(float(loss) - float(ref_loss)) / float(ref_loss) < 2e-3
    errs = {}
    for n, p in m.named_parameters():
        assert p.grad is not None, n
        errs[n] = _rel(p.grad, q[n].grad)
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:8]
    print("worst grad rel-L2:", ", ".join(f"{k}={v:.2e}" for k, v in worst))
    bad = {k: v for k, v in errs.items() if v > 8e-2 and not (".query." in k or ".key." in k)}
    assert not bad, bad
    cos = {n: float(torch.nn.functional.cosine_similarity(p.grad.float().cpu().flatten(), q[n].grad.flatten(), dim=0))
           for n, p in m.named_parameters()}
    assert min(cos.values()) > 0.95, sorted(cos.items(), key=lambda kv: kv[1])[:5]
    opt = torch.optim.AdamW(m.parameters(), lr=2e-3)
    opt.zero_grad(set_to_none=True)
    losses = []
    for _ in range(6):
        with torch.autocast("cuda", dtype=torch.bfloat16):
            _, l = m(*args, labels=g["labels"].to(DEV))
        l.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
        losses.append(float(l))
    assert losses[-1] < losses[0] - 0.05, losses


def test_uvit_v2_default_widths_training_gradients_vs_oracle():
    """Training backward at the U-ViT widths (hidden 1024 / 16 heads, blocks 768 / 12 heads + kv_mapper, 256 tokens, 77 text
    states): exercises the wgmma attention backward, the 4-chunk norm kernels and the wide GRN against fp32 autograd."""
    cfg = dict(num_hidden_layers=2, num_res_blocks=1, vocab_size=1032, codebook_size=1024, intermediate_size=2816)
    torch.manual_seed(0)
    m = MaskGiTUViT_v2(**cfg)
    gen = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for k, x in m.state_dict().items():
            if "adaLN_modulation.mapper" in k or k.endswith("gamma") or k.endswith("beta") or k == "mlm_layer.conv1.weight":
                x.copy_(torch.randn(x.shape, generator=gen) * 0.03)
    B = 2
    ids = torch.randint(0, 1024, (B, 256), generator=gen)
    mask = torch.rand(B, 256, generator=gen) < 0.5
    inp, lab = torch.where(mask, 1031, ids), torch.where(mask, ids, -100)
    enc = torch.randn(B, 77, 768, generator=gen)
    ce = torch.randn(B, 768, generator=gen)
    mc = torch.tensor([[256.0, 256.0, 0.0, 0.0, 6.0], [512.0, 512.0, 32.0, 16.0, 5.0]])
    q = {k: v.detach().clone().float().requires_grad_(True) for k, v in m.state_dict().items()}
    _, ref_loss = V2.forward(q, cfg, inp, enc, ce, mc, labels=lab)
    ref_loss.backward()
    m.to(DEV).train()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        _, loss = m(inp.to(DEV), enc.to(DEV), ce.to(DEV), mc.to(DEV), labels=lab.to(DEV))
    loss.backward()
    assert abs(float(loss) - float(ref_loss)) / float(ref_loss) < 2e-3
    errs = {n: _rel(p.grad, q[n].grad) for n, p in m.named_parameters()}
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:6]
    print("worst grad rel-L2:", ", ".join(f"{k}={v:.2e}" for k, v in worst))
    bad = {k: v for k, v in errs.items() if v > 8e-2 and not (".query." in k or ".key." in k)}
    assert not bad, bad


def test_micro_uvit_v2_loss_weight_training(golden):
    """per-token loss_weight (train_muse.py:216-224 -> modeling_transformer_v2.py:305-317) in training mode: weighted loss
    value vs the reference fixture, gradients vs the oracle's autograd."""
    g = golden("micro_uvit_v2.pt")
    q = {k: v.clone().requires_grad_(True) for k, v in g["state_dict"].items()}
    _, ref = V2.forward(q, g["config"], g["input_ids"], g["encoder_hidden_states"], g["cond_embeds"], g["micro_conds"],
                        labels=g["labels"], loss_weight=g["loss_weight"])
    ref.backward()
    m = MaskGiTUViT_v2(**g["config"])
    m.load_state_dict(g["state_dict"])
    m.to(DEV).train()
    args = [g[k].to(DEV) for k in ("input_ids", "encoder_hidden_states", "cond_embeds", "micro_conds")]
    with torch.autocast("cuda", dtype=torch.bfloat16):
        _, loss = m(*args, labels=g["labels"].to(DEV), loss_weight=g["loss_weight"].to(DEV))
    loss.backward()
    assert abs(float(loss) - float(g["loss_weighted"])) / float(g["loss_weighted"]) < 2e-3
    for n in ("mlm_layer.conv2.weight", "transformer_layers.1.ffn.wo.weight", "embed.embeddings.weight", "encoder_proj.weight"):
        assert _rel(dict(m.named_parameters())[n].grad, q[n].grad) < 5e-2, n
