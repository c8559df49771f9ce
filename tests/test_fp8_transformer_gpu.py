"""FP8 inference of MaskGitTransformer on the H100: the FP8 GEMM with the fused residual against integers, against
muse_gemm_fp8 plus the residual and against fp64; the e4m3 forms of the norm passes against fp64; the model in FP8 mode
against its bf16 mode; and a small trained class-conditional model's masked-token loss in both modes.

Every kernel launch here runs past the first wave of CTAs: the GEMM shapes have more output tiles than the H100 has SMs,
and the norm passes more rows than their resident warps cover.  The GEMM bounds are those of tests/test_fp8_gpu.py."""
import gc
import json
import math
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from open_muse_b200 import EMAModel, FusedAdamW, FusedAdamW8bit, FusedLion, MaskGitTransformer, ops  # noqa: E402
from tests import local_error as LE  # noqa: E402
from tests.test_fp8_gpu import _quant, _rel, gemm_ulps  # noqa: E402

DEV = "cuda"
E4M3 = torch.float8_e4m3fn
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(autouse=True)
def _release_models():
    """a model and its operand cache refer to each other, and a generate2 model holds CUDA graphs: collect them when each
    test ends, so that no later test's memory measurement sees them freed mid-way"""
    yield
    gc.collect()
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ FP8 GEMM + residual
def _operands(M, N, K, seed, integers):
    """e4m3 operands with NaN pad bytes past K (canaries), their scales, an fp32 residual, and the fp64 product"""
    g = torch.Generator().manual_seed(seed)
    ld = (K + 15) // 16 * 16
    if integers:
        qa, sa = torch.randint(-3, 4, (M, K), generator=g).float().to(E4M3), torch.ones(M)
        qb, sb = torch.randint(-3, 4, (N, K), generator=g).float().to(E4M3), torch.ones(N)
        res = torch.randint(-1000, 1000, (M, N), generator=g).float()
    else:
        qa, sa = _quant(torch.randn(M, K, generator=g) * torch.exp(torch.randn(M, 1, generator=g)))
        qb, sb = _quant(torch.randn(N, K, generator=g) * 0.02 * torch.exp(0.5 * torch.randn(N, 1, generator=g)))
        res = torch.randn(M, N, generator=g)
    A = torch.full((M, ld), 0x7F, dtype=torch.uint8)
    B = torch.full((N, ld), 0x7F, dtype=torch.uint8)
    A[:, :K] = qa.view(torch.uint8)
    B[:, :K] = qb.view(torch.uint8)
    fa = ops.F8(A.to(DEV).view(E4M3), sa.to(DEV))
    fb = ops.F8(B.to(DEV).view(E4M3), sb.to(DEV))
    prod = (qa.double() * sa.double()[:, None]) @ (qb.double() * sb.double()[:, None]).t()
    return fa, fb, res, prod, ld


def run_gemm_res(M, N, K, seed, integers=False):
    """(kernel output fp32 [M, N], residual, fp64 product, operands); the output buffer is NaN-filled around [M, N]"""
    fa, fb, res, prod, ld = _operands(M, N, K, seed, integers)
    ldc = N + 8
    R = torch.zeros(M, ldc, device=DEV)
    R[:, :N] = res.to(DEV)
    C = torch.full((M + 3, ldc), float("nan"), device=DEV)
    ops.gemm_fp8_res(fa, fb, R, C, M, N, K, ld, ld, ldc)
    torch.cuda.synchronize()
    Cc = C.cpu()
    assert torch.isnan(Cc[M:]).all() and torch.isnan(Cc[:M, N:]).all(), "rows past M or columns past N were written"
    return Cc[:M, :N], res, prod, (fa, fb, ld)


# M x N tiles of 128 x 128: 16 x 9 = 144 and 33 x 8 = 264 output tiles, more than the 132 CTAs of one wave
GEMM_SHAPES = [(2000, 1096, 64), (2000, 1096, 136), (4200, 1000, 1024), (2056, 1032, 4096)]


@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
def test_gemm_fp8_res_exact_on_integer_operands(M, N, K):
    out, res, prod, _ = run_gemm_res(M, N, K, seed=M + N + K, integers=True)
    want = res + prod.float().to(torch.bfloat16).float()
    bad = out != want
    assert not bad.any(), f"gemm_fp8_res {M}x{N}x{K}: {int(bad.sum())} outputs differ, first at {bad.nonzero()[0].tolist()}"


@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
def test_gemm_fp8_res_is_gemm_fp8_plus_the_residual_and_near_fp64(M, N, K):
    out, res, prod, (fa, fb, ld) = run_gemm_res(M, N, K, seed=M * 7 + N * 3 + K)
    plain = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
    ops.gemm_fp8(fa, fb, plain, M, N, K, ld, ld, N)
    assert torch.equal(out, res + plain.cpu().float())  # the same accumulation and rounding, then the residual add
    u = gemm_ulps(out - res, prod)
    loc = LE.check_local(out - res, prod, LE.rows(M), bound=6e-3, elem_bound=1e-1, what=f"gemm_fp8_res {M}x{N}x{K}")
    print(f"gemm_fp8_res M={M} N={N} K={K}: worst {float(u.max()):.1f} bf16 ulps, worst row rel-L2 {loc.worst:.2e} at "
          f"{loc.where}")


def test_linear_fwd_routes_f8_with_residual_to_the_fused_epilogue():
    fa, fb, res, prod, ld = _operands(300, 256, 128, 5, integers=True)
    x = ops.F8(fa.q[:, :128].contiguous(), fa.s)
    w = ops.F8(fb.q[:, :128].contiguous(), fb.s)
    y = ops.linear_fwd(x, w, res=res.to(DEV), out_dtype=torch.float32)
    assert y.dtype == torch.float32
    assert torch.equal(y.cpu(), res + prod.float().to(torch.bfloat16).float())
    with pytest.raises(TypeError):
        ops.linear_fwd(x, w, out_dtype=torch.float32)


# ------------------------------------------------------------------------------------------------ e4m3 norm forms
def _check_e4m3(f8, y64, what, tol=2e-5):
    """f8: the kernel's F8; y64: fp64 restatement of the row values it quantizes.  The scales must be amax / 448; a value
    may be one e4m3 ulp off only where y64 / s lies within tol * max(|y64 / s|, 16) of a rounding midpoint.  tol covers the
    fp32 error of a normalised row (its mean, variance and rsqrtf), which is relative to the row's size rather than the
    element's (hence the floor of 16 in the scaled units, where the row's largest value is 448): over the millions of values
    per test here, a few fall that close to a midpoint, on either side."""
    q = f8.q.cpu().double()
    s = f8.s.cpu()
    amax = y64.abs().amax(dim=1)
    want_s = torch.where(amax > 0, (amax / 448.0).float(), torch.ones_like(amax.float()))
    assert torch.allclose(s, want_s, rtol=2e-6, atol=0), f"{what}: scales differ from amax / 448"
    v = y64 / s.double()[:, None]
    ref = v.clamp(-448, 448).to(E4M3).double()  # satfinite: torch's cast would turn 448 * (1 + 2^-24) into NaN
    bad = q != ref
    worst = 0.0
    if bad.any():
        mid = (q + ref) / 2
        dist = (v - mid).abs() / v.abs().clamp_min(16.0)
        # one e4m3 step: 2^(e - 3) in binade e, and 2^-9 throughout the subnormals (|v| < 2^-6)
        step = torch.exp2(torch.floor(torch.log2(torch.maximum(q.abs(), ref.abs()).clamp_min(2 ** -6))) - 3)
        ulp = (q - ref).abs() <= step
        off = bad & ~((dist <= tol) & ulp)
        assert not off.any(), f"{what}: {int(off.sum())} e4m3 values off (first at {off.nonzero()[0].tolist()})"
        worst = float(dist[bad].max())
    print(f"{what}: {int(bad.sum())} of {bad.numel()} values one ulp off at a rounding midpoint (farthest {worst:.1e})")


ROWS = 9000  # 2250 CTAs of 4 rows: more than the 2112 (132 SMs x 16) resident at once


def _norm64(x, w, eps, rms):
    x = x.double()
    if rms:
        n = x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps)
    else:
        n = (x - x.mean(-1, keepdim=True)) * torch.rsqrt(x.var(-1, unbiased=False, keepdim=True) + eps)
    return n * w.double()


def _rows(rows, H, g, dtype):
    x = torch.randn(rows, H, generator=g) * 2 + 0.5
    x[1] = 0  # an all-zero row
    x[2, 5] = 300.0  # a single large outlier
    return x.to(dtype)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("rms", [0, 1])
@pytest.mark.parametrize("H", [512, 768, 1024])
def test_norm_fwd_e4m3(H, rms, dtype):
    g = torch.Generator().manual_seed(H + rms)
    x = _rows(ROWS, H, g, dtype)
    w = 1 + 0.1 * torch.randn(H, generator=g)
    res = torch.randn(ROWS, H, generator=g) if dtype == torch.float32 and rms else None
    kw = dict(rms=rms, res=None if res is None else res.to(DEV))
    y, st = ops.norm_fwd(x.to(DEV), w.to(DEV), 1e-6, ops.FP8, **kw)
    yb, stb = ops.norm_fwd(x.to(DEV), w.to(DEV), 1e-6, torch.bfloat16, **kw)
    assert torch.equal(st, stb)  # the statistics are the bf16 form's
    y64 = _norm64(x, w, 1e-6, rms) if res is None else _norm64(x, w, 1e-6, rms) + res.double()
    if res is None:
        y64[1] = 0  # (an all-zero row normalises to zero: no NaN from the fp64 restatement)
    _check_e4m3(y, y64, f"norm_fwd e4m3 H={H} rms={rms} x {dtype}" + (" + res" if res is not None else ""))


@pytest.mark.parametrize("I", [2048, 3072, 4096])
def test_glu_norm_fwd_e4m3(I):
    g = torch.Generator().manual_seed(I)
    rows = 3300  # 413 CTAs of 8 rows: past the 264 (132 SMs x 2) resident at I <= 2048 and the 132 above
    ab = torch.randn(rows, 2 * I, generator=g) * 1.5
    ab[1] = 0
    ab[2, I + 3] = 400.0
    ab = ab.to(torch.bfloat16).to(DEV)
    w = (1 + 0.1 * torch.randn(I, generator=g)).to(DEV)
    y, st = ops.norm_fwd(ab, w, 1e-6, ops.FP8, act=2, rms=0)
    yb, stb = ops.norm_fwd(ab, w, 1e-6, torch.bfloat16, act=2, rms=0)
    assert torch.equal(st, stb)
    # the value the pass normalises, restated: v = bf16(bf16(gelu(a)) * b) (the product of two bf16 values is exact in fp32)
    a, b = ab[:, :I].cpu().double(), ab[:, I:].cpu().double()
    ge = a * 0.5 * (1 + torch.erf(a / math.sqrt(2)))
    v = (ge.float().to(torch.bfloat16).double() * b).float().to(torch.bfloat16).double()
    # the kernel's GELU (common.cuh gelu_eval) is a * cdf with the 1.5e-7 erf approximation of Abramowitz-Stegun 7.1.26,
    # evaluated in fp32 with an approximate reciprocal and exponential: |err| <= 5e-7 |a| bounds both.  Where that can move
    # the bf16 rounding of gelu(a), the fp64 value cannot say which side the kernel takes: there (about 1.5 % of the
    # elements) v is taken from the bf16 GLU pass, which must equal the restatement at every other element
    lo = (ge - 5e-7 * a.abs()).float().to(torch.bfloat16)
    hi = (ge + 5e-7 * a.abs()).float().to(torch.bfloat16)
    amb = lo != hi
    v_pass = ops.glu_fwd(ab).cpu().double()
    assert torch.equal(v_pass[~amb], v[~amb])
    v = torch.where(amb, v_pass, v)
    mean, rstd = st.cpu().double()
    m64 = v.mean(-1)
    r64 = torch.rsqrt(v.var(-1, unbiased=False) + 1e-6)
    assert torch.allclose(mean, m64, rtol=1e-4, atol=1e-6) and torch.allclose(rstd, r64, rtol=1e-4, atol=0)
    y64 = _norm64(v, w.cpu(), 1e-6, 0)
    print(f"GLU + mid-norm I={I}: {int(amb.sum())} elements with an ambiguous bf16 gelu(a); worst statistics rel. error "
          f"{float(((rstd - r64).abs() / r64).max()):.1e}")
    _check_e4m3(y, y64, f"GLU + mid-norm e4m3 I={I}")


@pytest.mark.parametrize("H", [512, 768, 1024])
def test_norm2_fwd_e4m3(H):
    g = torch.Generator().manual_seed(H)
    a = _rows(ROWS, H, g, torch.bfloat16).to(DEV)
    res = torch.randn(ROWS, H, generator=g).to(DEV)
    w1, w2 = (1 + 0.1 * torch.randn(2, H, generator=g)).to(DEV)
    x2, h2, st = ops.norm2_fwd(a, res, w1, w2, 1e-6, rms1=1, rms2=0, h2_dtype=ops.FP8)
    x2b, h2b, stb = ops.norm2_fwd(a, res, w1, w2, 1e-6, rms1=1, rms2=0)
    assert torch.equal(x2, x2b) and torch.equal(st, stb)  # x2 and the statistics are bit-equal to the bf16 form's
    _check_e4m3(h2, _norm64(x2.cpu(), w2.cpu(), 1e-6, 0), f"norm2 e4m3 H={H}")


# ------------------------------------------------------------------------------------------------ model
V1_MICRO = ["micro_transformer.pt", "micro_t2i_transformer.pt", "micro_t2i_proj_transformer.pt"]


def _model(g):
    if "state_dict" in g:
        m = MaskGitTransformer(**g["config"])
        m.load_state_dict(g["state_dict"])
    else:
        torch.manual_seed(g["seed"])
        m = MaskGitTransformer(**g["config"])
    return m.to(DEV).eval()


def _inputs(g):
    if "batch" in g:
        return dict(input_ids=g["batch"]["input_ids"].to(DEV))
    return dict(input_ids=g["input_ids"].to(DEV), encoder_hidden_states=g["encoder_hidden_states"].to(DEV))


def _fp8_vs_bf16(m, kw, what):
    with torch.no_grad():
        ref = m.set_gemm_precision("bf16")(**kw)
        out = m.set_gemm_precision("fp8")(**kw)
        again = m.set_gemm_precision("bf16")(**kw)
    assert torch.equal(ref, again)  # bf16 logits are bit-identical after the round trip
    rel = _rel(out, ref)
    print(f"{what}: FP8 vs bf16 logits rel-L2 {rel:.3e}")
    return rel


@pytest.mark.parametrize("name", V1_MICRO)
def test_micro_fixture_fp8_logits(golden, name):
    g = golden(name)
    assert _fp8_vs_bf16(_model(g), _inputs(g), name) < 0.05


def test_fp8_logits_reported_at_hd48_and_base_widths(golden):
    """no gate: the values are reported (DESIGN.md section 5)"""
    g = golden("hd48_transformer.pt")
    rel = _fp8_vs_bf16(_model(g), _inputs(g), "hd48 (768 / 16 heads, I 3072), 2 layers")
    assert math.isfinite(rel)
    cfg = json.load(open(os.path.join(HERE, "golden", "configs.json")))["imagenet.yaml"]["transformer"]
    torch.manual_seed(0)
    m = MaskGitTransformer(**cfg).to(DEV).eval()
    ids = torch.randint(0, 1024, (8, 257), generator=torch.Generator().manual_seed(1))
    ids[:, 0] = 1024 + 7
    ids[:, 1::2] = cfg["vocab_size"] - 1
    rel = _fp8_vs_bf16(m, dict(input_ids=ids.to(DEV)), "imagenet.yaml widths (24 x 768, I 3072), random init, B=8")
    assert math.isfinite(rel)


def test_fp8_forward_refuses_training_use(golden):
    g = golden("micro_transformer.pt")
    m = _model(g).set_gemm_precision("fp8")
    with pytest.raises(RuntimeError, match="inference only"):
        m(**_inputs(g), labels=g["batch"]["labels"].to(DEV))
    m.train()
    with torch.no_grad(), pytest.raises(RuntimeError, match="inference only"):
        m(**_inputs(g))


def _generate(m, kw, graph, gen=None):
    gen = (torch.Generator(device=DEV) if gen is None else gen).manual_seed(11)
    kw = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in kw.items()}  # class_ids is offset in place
    return m.generate2(**kw, generator=gen, use_cuda_graph=graph)


@pytest.mark.parametrize("name", ["micro_transformer.pt", "micro_t2i_transformer.pt"])
def test_fp8_generate2_graph_equals_eager_and_is_reproducible(golden, name):
    g = golden(name)
    m = _model(g).set_gemm_precision("fp8")
    if "batch" in g:
        kw = dict(class_ids=g["batch"]["class_ids"].to(DEV), timesteps=6)
    else:
        ehs = g["encoder_hidden_states"].to(DEV)
        kw = dict(encoder_hidden_states=ehs, negative_embeds=torch.randn_like(ehs) * 0.1, guidance_scale=3.0, timesteps=6)
    a, b, e = _generate(m, kw, True), _generate(m, kw, True), _generate(m, kw, False)
    assert torch.equal(a, b) and torch.equal(a, e)
    assert int(a.min()) >= 0 and int(a.max()) < m.config.codebook_size
    bf = _generate(m.set_gemm_precision("bf16"), kw, True)
    print(f"{name}: generate2 ids equal to bf16 mode: {float((bf == a).float().mean()):.3f}")


@pytest.mark.parametrize("first,other", [("bf16", "fp8"), ("fp8", "bf16")])
def test_generate2_graphs_stay_valid_across_precision_switches(golden, first, other):
    """first -> other -> first: each graphed generate2 equals the eager one, and the third call replays the graph the
    first one captured.  After each call NaN-filled tensors of the packed buffers' sizes are allocated, so a graph whose
    weight buffers had been freed and handed out again would read NaN weights."""
    g = golden("micro_t2i_transformer.pt")
    ehs = g["encoder_hidden_states"].to(DEV)
    kw = dict(encoder_hidden_states=ehs, negative_embeds=torch.randn_like(ehs) * 0.1, guidance_scale=3.0, timesteps=6)
    m = _model(g)
    gen = torch.Generator(device=DEV)  # one generator object: it is part of the graph cache key
    junk = []

    def run(prec):
        m.set_gemm_precision(prec)
        graphed, eager = _generate(m, kw, True, gen), _generate(m, kw, False, gen)
        pk = m._packed
        junk.append(torch.full_like(pk.flat, float("nan")))
        junk.extend(torch.full_like(f8.q, float("nan")) for _, f8 in pk.f8_pairs)
        return graphed, eager

    (a, ea), (b, eb), (c, ec) = run(first), run(other), run(first)
    assert torch.equal(a, ea) and torch.equal(b, eb) and torch.equal(c, ec)
    assert torch.equal(a, c)
    assert len(m._gen_graphs) == 2  # one graph per precision: the third call replayed the first one's


@pytest.mark.parametrize("opt_cls", [FusedAdamW, FusedLion, FusedAdamW8bit])
def test_fp8_operands_follow_fused_optimizer_steps(golden, opt_cls):
    g = golden("micro_t2i_proj_transformer.pt")
    m = _model(g)
    kw = _inputs(g)
    with torch.no_grad():
        m.set_gemm_precision("fp8")(**kw)
    ema = EMAModel(m.parameters(), decay=0.5)
    opt = opt_cls(m.parameters(), lr=1e-3, ema=ema, model=m)
    for _ in range(2):
        m.set_gemm_precision("bf16").train()
        _, loss = m(**kw, labels=g["labels"].to(DEV))
        loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
        m.set_gemm_precision("fp8").eval()
        with torch.no_grad():
            out = m(**kw)
        assert torch.isfinite(out).all()
        assert m._packed.quantized
        for src, f8 in m._packed.quantized:
            want = ops.quantize_rows_e4m3(src)
            assert torch.equal(f8.q.view(torch.uint8), want.q.view(torch.uint8)) and torch.equal(f8.s, want.s)


# ------------------------------------------------------------------------------------------------ quality proxy
QUALITY = dict(vocab_size=64 + 1 + 8, hidden_size=128, num_hidden_layers=2, num_attention_heads=2, intermediate_size=512,
               max_position_embeddings=257, codebook_size=64, num_vq_tokens=256, num_classes=8, hidden_dropout=0.0,
               attention_dropout=0.0)


def _task_batch(B, g):
    """class c's 16x16 template is token c * 8 + (x + 2 y) % 8; 20 % of the tokens are replaced by uniform noise (so the
    loss floor, about 1.3 nats, is well above zero).  Returns the class id + 50 %-masked ids and labels."""
    c = torch.randint(0, 8, (B,), generator=g)
    yy, xx = torch.meshgrid(torch.arange(16), torch.arange(16), indexing="ij")
    tok = c[:, None, None] * 8 + (xx[None] + 2 * yy[None]) % 8
    tok = tok.reshape(B, 256)
    noise = torch.rand(B, 256, generator=g) < 0.2
    tok = torch.where(noise, torch.randint(0, 64, (B, 256), generator=g), tok)
    masked = torch.rand(B, 256, generator=g) < 0.5
    ids = torch.where(masked, torch.full_like(tok, 72), tok)  # vocab = codebook + classes + mask: mask id 72
    labels = torch.where(masked, tok, torch.full_like(tok, -100))
    ids = torch.cat([(c + 64)[:, None], ids], dim=1)  # class tokens follow the codebook
    labels = torch.cat([torch.full((B, 1), -100), labels], dim=1)
    return ids.to(DEV), labels.to(DEV)


def test_quality_proxy_trained_transformer_fp8_ce_within_2_percent():
    torch.manual_seed(0)
    m = MaskGitTransformer(**QUALITY).to(DEV).train()
    g = torch.Generator().manual_seed(0)
    opt = FusedAdamW(m.parameters(), lr=2e-3, weight_decay=0.0, model=m)
    for _ in range(600):
        ids, labels = _task_batch(32, g)
        _, loss = m(ids, labels=labels)
        loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
    m.eval()
    ids, labels = _task_batch(256, torch.Generator().manual_seed(123))
    with torch.no_grad():
        _, ce_bf16 = m(ids, labels=labels)
        m.set_gemm_precision("fp8")
        _, ce_fp8 = m(ids, labels=labels)
    assert m._packed.quantized  # FP8 operands were used
    ce_bf16, ce_fp8 = float(ce_bf16), float(ce_fp8)
    assert ce_fp8 != ce_bf16
    gap = abs(ce_fp8 - ce_bf16) / ce_bf16
    print(f"quality proxy: masked CE bf16 {ce_bf16:.4f} (0.5 ln V = {0.5 * math.log(64):.4f}), FP8 {ce_fp8:.4f}, "
          f"relative gap {gap:.4%}")
    assert ce_bf16 < 0.5 * math.log(64)
    assert gap < 0.02
