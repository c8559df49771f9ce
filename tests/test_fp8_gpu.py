"""FP8 inference of MaskGiTUViT_v2 on the H100: the e4m3 GEMM against fp64, the three e4m3 producers against an fp64
restatement, the model in FP8 mode against its bf16 mode, and a small trained model's masked-token loss in both modes.

GEMM bounds.  The H100's e4m3 MMA does not sum its products in fp32: measured here, it keeps about 13-14 bits relative to
the largest product of each k32 instruction, which no fp32 promotion outside the instruction can restore (DESIGN.md
section 4: with each 128-wide k-block promoted, 1.4 % of the outputs of random operands lie more than one bf16 ulp from the
fp64 product, 6-8 % without promotion).  So the GEMM is held to two bounds: on small-integer operands, where every sum is
exact in any accumulator, the output equals the fp64 product rounded to bf16 (this pins every row, column and k-block
of the tiling); on random operands, every row's rel-L2 error stays within 6e-3 (twice the worst measured) and the
per-element error in bf16 ulps -- of max(|ref|, rms(row) / 256), so that outputs cancelling to zero are measured against
their row's size -- is reported."""
import math
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from open_muse_b200 import MaskGiTUViT_v2, ops  # noqa: E402
from open_muse_b200.optim import FusedAdamW  # noqa: E402
from tests import local_error as LE  # noqa: E402

DEV = "cuda"
E4M3 = torch.float8_e4m3fn


def _rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-20))


def _quant(x):
    """per-row e4m3 restatement of the producers: s = amax / 448 (1 for a zero row), q = e4m3(x / s)"""
    amax = x.abs().amax(dim=1)
    s = torch.where(amax > 0, (amax.float() / 448.0), torch.ones_like(amax.float()))
    return (x.double() / s.double()[:, None]).clamp(-448, 448).to(E4M3), s


def _bf16_ulp(v):
    v = v.abs().clamp_min(1e-30)
    return torch.exp2(torch.floor(torch.log2(v)) - 7)


def gemm_ulps(out, ref):
    """|out - ref| in bf16 ulps of max(|ref|, rms(row) / 256), per element (module docstring)"""
    ref = ref.double()
    floor = ref.pow(2).mean(dim=1, keepdim=True).sqrt() / 256
    return (out.double() - ref).abs() / _bf16_ulp(torch.maximum(ref.abs(), floor))


def run_gemm(M, N, K, seed, integers=False):
    """(kernel output bf16 [M, N], fp64 reference of the dequantized operands); pad columns of A and B hold e4m3 NaN
    bytes and the output buffer is NaN-filled around [M, N] (canaries).  integers: operands in {-3..3} with unit scales."""
    g = torch.Generator().manual_seed(seed)
    ld = (K + 15) // 16 * 16
    if integers:
        qa, sa = torch.randint(-3, 4, (M, K), generator=g).float().to(E4M3), torch.ones(M)
        qb, sb = torch.randint(-3, 4, (N, K), generator=g).float().to(E4M3), torch.ones(N)
    else:
        a32 = torch.randn(M, K, generator=g) * torch.exp(torch.randn(M, 1, generator=g))
        b32 = torch.randn(N, K, generator=g) * 0.02 * torch.exp(0.5 * torch.randn(N, 1, generator=g))
        qa, sa = _quant(a32)
        qb, sb = _quant(b32)
    A = torch.full((M, ld), 0x7F, dtype=torch.uint8)
    B = torch.full((N, ld), 0x7F, dtype=torch.uint8)
    A[:, :K] = qa.view(torch.uint8)
    B[:, :K] = qb.view(torch.uint8)
    ldc = N + 8
    C = torch.full((M + 3, ldc), float("nan"), dtype=torch.bfloat16, device=DEV)
    fa = ops.F8(A.to(DEV).view(E4M3), sa.to(DEV))
    fb = ops.F8(B.to(DEV).view(E4M3), sb.to(DEV))
    ops.gemm_fp8(fa, fb, C, M, N, K, ld, ld, ldc)
    torch.cuda.synchronize()
    Cc = C.cpu()
    assert torch.isnan(Cc[M:]).all() and torch.isnan(Cc[:M, N:]).all(), "rows past M or columns past N were written"
    ref = (qa.double() * sa.double()[:, None]) @ (qb.double() * sb.double()[:, None]).t()
    return Cc[:M, :N], ref


GEMM_SHAPES = [(200, 72, 136), (200, 2816, 4096), (2056, 2816, 768), (2056, 72, 2816), (4096, 5632, 2816),
               (4096, 1024, 4096), (2056, 5632, 136)]


@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
def test_gemm_fp8_exact_on_integer_operands(M, N, K):
    out, ref = run_gemm(M, N, K, seed=M + N + K, integers=True)
    want = ref.float().to(torch.bfloat16)
    bad = out != want
    assert not bad.any(), f"gemm_fp8 {M}x{N}x{K}: {int(bad.sum())} outputs differ, first at {bad.nonzero()[0].tolist()}"


@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
def test_gemm_fp8_vs_fp64(M, N, K):
    out, ref = run_gemm(M, N, K, seed=M * 7 + N * 3 + K)
    assert torch.isfinite(out).all()
    u = gemm_ulps(out, ref)
    loc = LE.check_local(out, ref, LE.rows(M), bound=6e-3, elem_bound=1e-1, what=f"gemm_fp8 {M}x{N}x{K}")
    print(f"gemm_fp8 M={M} N={N} K={K}: worst {float(u.max()):.1f} bf16 ulps at row {int(u.amax(1).argmax())}, "
          f"{float((u > 1).double().mean()):.2%} of the outputs past one ulp; worst row rel-L2 {loc.worst:.2e} at "
          f"{loc.where}")


def test_gemm_fp8_rejects_bad_layouts():
    f = ops.F8(torch.zeros(8, 64, dtype=E4M3, device=DEV), torch.ones(8, device=DEV))
    with pytest.raises(Exception, match="multiples of 8"):
        ops.gemm_fp8(f, f, torch.empty(8, 12, dtype=torch.bfloat16, device=DEV), 8, 6, 64, 64, 64, 12)


# ------------------------------------------------------------------------------------------------ producers
def _check_e4m3(f8, y64, what):
    """f8: the kernel's F8; y64: fp64 restatement of the value it quantizes [rows, K].  A value may be one e4m3 ulp off
    only where y64 / s lies within 1e-6 (relative, at least 1e-6 absolute in the scaled units) of a rounding midpoint."""
    q = f8.q.cpu().double()
    s = f8.s.cpu()
    amax = y64.abs().amax(dim=1)
    want_s = torch.where(amax > 0, (amax / 448.0).float(), torch.ones_like(amax.float()))
    assert torch.allclose(s, want_s, rtol=2e-6, atol=0), f"{what}: scales differ from amax / 448"
    v = y64 / s.double()[:, None]
    ref = v.clamp(-448, 448).to(E4M3).double()  # satfinite: torch's cast would turn 448 * (1 + 2^-24) into NaN
    bad = q != ref
    if bad.any():
        mid = (q + ref) / 2
        near = (v - mid).abs() <= 1e-6 * v.abs().clamp_min(1.0)
        ulp = (q - ref).abs() <= torch.exp2(torch.floor(torch.log2(torch.maximum(q.abs(), ref.abs()).clamp_min(2 ** -9))) - 3)
        off = bad & ~(near & ulp)
        assert not off.any(), f"{what}: {int(off.sum())} e4m3 values off (first at {off.nonzero()[0].tolist()})"
    print(f"{what}: {int(bad.sum())} of {bad.numel()} values one ulp off at a rounding midpoint")


def _rows_with_edges(rows, H, g, dtype=torch.float32):
    x = torch.randn(rows, H, generator=g)
    x[1] = 0  # an all-zero row
    x[2, 5] = 300.0  # a single large outlier
    return x.to(dtype)


@pytest.mark.parametrize("H,rms,with_mod", [(1024, 1, True), (768, 0, False), (128, 1, True)])
def test_add_norm_mod_e4m3(H, rms, with_mod):
    g = torch.Generator().manual_seed(H)
    B, S = 3, 20
    a = _rows_with_edges(B * S, H, g, torch.bfloat16)
    w = 1 + 0.1 * torch.randn(H, generator=g)
    mod = torch.randn(B, 2 * H, generator=g) * 0.3 if with_mod else None
    _, y = ops.add_norm_mod(a.to(DEV), w.to(DEV), 1e-6, rms, out_dtype=ops.FP8, mod=None if mod is None else mod.to(DEV),
                            rows_per_sample=S, want_residual=False)
    x = a.double()
    if rms:
        n = x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + 1e-6)
    else:
        n = (x - x.mean(-1, keepdim=True)) * torch.rsqrt(x.var(-1, unbiased=False, keepdim=True) + 1e-6)
    y64 = n * w.double()
    if with_mod:
        y64 = (y64.view(B, S, H) * (1 + mod.double()[:, None, :H]) + mod.double()[:, None, H:]).view(B * S, H)
    _check_e4m3(y, y64, f"add_norm_mod e4m3 H={H}")


@pytest.mark.parametrize("C,hw,rms", [(768, 16, 1), (1024, 8, 0)])
def test_dwconv3x3_norm_e4m3(C, hw, rms):
    g = torch.Generator().manual_seed(C + hw)
    B = 2
    x = torch.randn(B, hw, hw, C, generator=g)
    x[0, :3, :3] = 0  # pixel (0, 1, 1) sees only zeros: an all-zero row
    x[1, 4, 4, 7] = 500.0  # one large outlier
    wd = torch.randn(C, 1, 3, 3, generator=g) * 0.3
    nw = 1 + 0.1 * torch.randn(C, generator=g)
    y, conv = ops.dwconv3x3_norm(x.view(-1, C).to(DEV), wd.view(C, 9).t().contiguous().to(DEV), nw.to(DEV), B, hw, hw,
                                 1e-6, rms, save_conv=True, out_dtype=ops.FP8)
    # the norm is restated from the kernel's own bf16 conv output (the conv itself is checked by test_uvit_v2_gpu.py)
    conv = conv.cpu().double()
    if rms:
        n = conv * torch.rsqrt(conv.pow(2).mean(-1, keepdim=True) + 1e-6)
    else:
        n = (conv - conv.mean(-1, keepdim=True)) * torch.rsqrt(conv.var(-1, unbiased=False, keepdim=True) + 1e-6)
    _check_e4m3(y, n * nw.double(), f"dwconv3x3_norm e4m3 C={C}")


@pytest.mark.parametrize("I", [2816, 128])
def test_glu_e4m3(I):
    g = torch.Generator().manual_seed(I)
    rows = 300
    ab = torch.randn(rows, 2 * I, generator=g) * 1.5
    ab[1] = 0
    ab[2, I + 3] = 400.0
    ab = ab.to(torch.bfloat16)
    out = ops.glu_fwd(ab.to(DEV), out_dtype=ops.FP8)
    a, b = ab[:, :I].double(), ab[:, I:].double()
    ge = a * 0.5 * (1 + torch.erf(a / math.sqrt(2)))
    gb = ge.float().to(torch.bfloat16).double()
    # the kernel's GELU is exact to its erf approximation (|err| <= 1.5e-7 on the CDF); where that moves the bf16 rounding
    # of gelu(a), the fp64 value of that element is taken from the kernel's side of the rounding
    y = gb * b
    f = out.q.cpu().double() * out.s.cpu().double()[:, None]
    lo = (ge - 1.5e-7 * a.abs()).float().to(torch.bfloat16).double()
    hi = (ge + 1.5e-7 * a.abs()).float().to(torch.bfloat16).double()
    amb = lo != hi
    alt = torch.where(gb == lo, hi, lo) * b
    y = torch.where(amb & ((f - alt).abs() < (f - y).abs()), alt, y)
    _check_e4m3(out, y, f"glu e4m3 I={I}")


def test_quantize_rows_e4m3():
    g = torch.Generator().manual_seed(3)
    w = (torch.randn(300, 2816, generator=g) * 0.02)
    w[1] = 0
    w[2, 9] = 5.0
    wb = w.to(torch.bfloat16)
    f = ops.quantize_rows_e4m3(wb.to(DEV))
    _check_e4m3(f, wb.double(), "quantize_rows_e4m3")


# ------------------------------------------------------------------------------------------------ model
def _model(g=None, **cfg):
    if g is not None:
        m = MaskGiTUViT_v2(**g["config"])
        m.load_state_dict(g["state_dict"])
    else:
        torch.manual_seed(0)
        with torch.device(DEV):
            m = MaskGiTUViT_v2(**cfg)
    return m.to(DEV).eval()


def _inputs(m, B, S, seed):
    c = m.config
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, c.vocab_size, (B, S), generator=g)
    ids[:, ::3] = c.mask_token_id
    ehs = torch.randn(B, 77, c.encoder_hidden_size, generator=g)
    cond = torch.randn(B, c.cond_embed_dim, generator=g)
    micro = torch.tensor([[512.0, 512.0, 0.0, 0.0, 6.0]]).repeat(B, 1)
    return [t.to(DEV) for t in (ids, ehs, cond, micro)]


def _fp8_vs_bf16(m, args, what):
    with torch.no_grad():
        ref = m(*args)
        m.set_gemm_precision("fp8")
        out = m(*args)
        m.set_gemm_precision("bf16")
        again = m(*args)
    rel = _rel(out, ref)
    print(f"{what}: FP8 vs bf16 logits rel-L2 {rel:.3e}")
    assert torch.isfinite(out).all() and torch.equal(again, ref)
    return rel


def test_micro_fixture_fp8_logits(golden):
    g = golden("micro_uvit_v2.pt")
    m = _model(g)
    args = [g[k].to(DEV) for k in ("input_ids", "encoder_hidden_states", "cond_embeds", "micro_conds")]
    assert _fp8_vs_bf16(m, args, "micro_uvit_v2") < 0.1  # 0.024 measured


@pytest.mark.parametrize("down_up", [False, True])
def test_class_defaults_fp8_logits_cfg_batch(down_up):
    m = _model(force_down_up_sample=down_up)
    for p in m.parameters():  # away from the zero-initialised adaLN mappers / mlm conv1, so every site carries signal
        p.data.add_(torch.randn_like(p) * 0.02)
    S = 1024 if down_up else 256
    args = _inputs(m, 16, S, seed=1)  # B = 8 with CFG doubles to 16 rows of samples
    # measured on an H100 80GB HBM3 (700 W): 0.142 (256 tokens) and 0.158 (force_down_up_sample); a sanity bound, the
    # accuracy that matters is the quality proxy below
    assert _fp8_vs_bf16(m, args, f"class defaults, force_down_up_sample={down_up}, B=16 x {S} tokens") < 0.3


def test_fp8_is_inference_only(golden):
    g = golden("micro_uvit_v2.pt")
    m = _model(g).set_gemm_precision("fp8")
    args = [g[k].to(DEV) for k in ("input_ids", "encoder_hidden_states", "cond_embeds", "micro_conds")]
    with pytest.raises(RuntimeError, match="inference only"):
        m(*args)  # grad enabled
    m.train()
    with torch.no_grad(), pytest.raises(RuntimeError, match="inference only"):
        m(*args)


def test_fp8_generate2_reproducible_and_graph_equals_eager(golden):
    g = golden("micro_uvit_v2.pt")
    m = _model(g).set_gemm_precision("fp8")
    kw = dict(encoder_hidden_states=g["encoder_hidden_states"].to(DEV), cond_embeds=g["cond_embeds"].to(DEV),
              micro_conds=g["micro_conds"][:1].to(DEV), empty_embeds=g["empty_embeds"].to(DEV),
              empty_cond_embeds=g["empty_cond_embeds"].to(DEV), temperature=(2.0, 0.0), timesteps=6, seq_len=16,
              guidance_scale=3.0)
    gen = lambda: torch.Generator(device=DEV).manual_seed(11)  # noqa: E731
    a = m.generate2(**kw, generator=gen())
    b = m.generate2(**kw, generator=gen())
    e = m.generate2(**kw, use_cuda_graph=False, generator=gen())
    assert torch.equal(a, b) and torch.equal(a, e) and m._graph is not None
    assert int(a.min()) >= 0 and int(a.max()) < 64
    m.set_gemm_precision("bf16")
    bf = m.generate2(**kw, generator=gen())
    print(f"generate2 ids equal to bf16 mode: {float((bf == a).float().mean()):.3f}")


# ------------------------------------------------------------------------------------------------ quality proxy
QUALITY = dict(hidden_size=128, num_attention_heads=2, in_channels=64, block_out_channels=(64,), block_num_heads=1,
               num_res_blocks=1, num_hidden_layers=2, intermediate_size=256, vocab_size=72, codebook_size=64,
               encoder_hidden_size=32, cond_embed_dim=16, micro_cond_encode_dim=8, micro_cond_embed_dim=40)


def _task_batch(B, g, cls_emb):
    """class c's 16x16 template is token c * 8 + (x + 2 y) % 8, shifted by a random (dx, dy); 20 % of the tokens are
    replaced by uniform noise (so the loss floor is well above zero).  Returns ids, labels of a 50 % masking, the class
    conditioning and text states."""
    c = torch.randint(0, 8, (B,), generator=g)
    dx, dy = torch.randint(0, 8, (B,), generator=g), torch.randint(0, 8, (B,), generator=g)
    yy, xx = torch.meshgrid(torch.arange(16), torch.arange(16), indexing="ij")
    tok = c[:, None, None] * 8 + ((xx[None] + dx[:, None, None]) + 2 * (yy[None] + dy[:, None, None])) % 8
    tok = tok.reshape(B, 256)
    noise = torch.rand(B, 256, generator=g) < 0.2
    tok = torch.where(noise, torch.randint(0, 64, (B, 256), generator=g), tok)
    masked = torch.rand(B, 256, generator=g) < 0.5
    ids = torch.where(masked, torch.full_like(tok, 71), tok)
    labels = torch.where(masked, tok, torch.full_like(tok, -100))
    cond = cls_emb[c]
    ehs = cls_emb[c][:, None, :].repeat(1, 4, 2)
    micro = torch.zeros(B, 5)
    return [t.to(DEV) for t in (ids, ehs, cond, micro)], labels.to(DEV)


def test_quality_proxy_trained_uvit_fp8_ce_within_2_percent():
    torch.manual_seed(0)
    m = MaskGiTUViT_v2(**QUALITY).to(DEV).train()
    g = torch.Generator().manual_seed(0)
    cls_emb = torch.randn(8, 16, generator=g)
    opt = FusedAdamW(m.parameters(), lr=2e-3, weight_decay=0.0, model=m)
    for _ in range(400):
        args, labels = _task_batch(32, g, cls_emb)
        _, loss = m(*args, labels=labels)
        loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
    m.eval()
    held, held_labels = _task_batch(256, torch.Generator().manual_seed(123), cls_emb)
    with torch.no_grad():
        _, ce_bf16 = m(*held, labels=held_labels)
        m.set_gemm_precision("fp8")
        _, ce_fp8 = m(*held, labels=held_labels)
    assert any(isinstance(v, ops.F8) for layer in m._weights()["layers"] for v in layer.values())  # FP8 operands were used
    ce_bf16, ce_fp8 = float(ce_bf16), float(ce_fp8)
    assert ce_fp8 != ce_bf16
    gap = abs(ce_fp8 - ce_bf16) / ce_bf16
    print(f"quality proxy: masked CE bf16 {ce_bf16:.4f} (0.5 ln V = {0.5 * math.log(64):.4f}), FP8 {ce_fp8:.4f}, "
          f"relative gap {gap:.4%}")
    assert ce_bf16 < 0.5 * math.log(64)
    assert gap < 0.02
