"""``MaskGiTUViT_v2(use_fused_mlp=True)`` on the H100: the tanh-GELU pass (muse_gelu_tanh_fwd / _bwd) against fp64, its e4m3
form, past the first wave of CTAs; and the micro model against the unmodified
reference's fixture (tests/golden/micro_uvit_v2_fused_mlp.pt) in training, with gradient checkpointing, as a CUDA graph,
after fused optimizer steps and in FP8 mode."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from open_muse_b200 import FusedAdamW, FusedAdamW8bit, FusedLion, MaskGiTUViT_v2, ops  # noqa: E402
from tests.golden import make_golden_fused_mlp as GF  # noqa: E402

DEV = "cuda"
E4M3 = torch.float8_e4m3fn
ARGS = ("input_ids", "encoder_hidden_states", "cond_embeds", "micro_conds")
FIXTURE = "micro_uvit_v2_fused_mlp.pt"
SHAPES = [(32 * 256, 8), (32 * 256, 2816), (3 * 257, 4096), (3 * 257, 2816)]  # rows past the first wave of CTAs


def _rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-20))


def gelu_tanh64(x):
    x = x.double()
    return 0.5 * x * (1 + torch.tanh((2 / torch.pi) ** 0.5 * (x + 0.044715 * x ** 3)))


def gelu_tanh_grad64(x):
    x = x.double()
    t = torch.tanh((2 / torch.pi) ** 0.5 * (x + 0.044715 * x ** 3))
    return 0.5 * (1 + t) + 0.5 * x * (1 - t * t) * (2 / torch.pi) ** 0.5 * (1 + 3 * 0.044715 * x * x)


def _bf16_ulp(v):
    return torch.exp2(torch.floor(torch.log2(v.abs().clamp_min(1e-30))) - 7)


def _pre(rows, I, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, I, generator=g) * 3.0
    x[0, :] = 0
    x[-1, : min(I, 8)] = torch.tensor([-12.0, -5.0, -1e-3, 1e-3, 0.5, 5.0, 12.0, 30.0])[: min(I, 8)]
    return x.to(torch.bfloat16)


# ------------------------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize("rows,I", SHAPES)
def test_gelu_tanh_fwd_within_one_bf16_ulp_of_fp64(rows, I):
    """every element within one bf16 ulp of the fp64 value.  Where gelu_tanh(x) cancels towards 0 (x << 0) the fp32
    1 + tanh(.) of the formula carries an absolute error of about |x| 2^-24, as torch's own kernel does: the ulp is taken
    at max(|ref|, |x| 2^-16)."""
    x = _pre(rows, I, rows + I)
    out = ops.gelu_tanh_fwd(x.to(DEV))
    torch.cuda.synchronize()
    assert out.dtype == torch.bfloat16 and out.shape == (rows, I)
    ref = gelu_tanh64(x)
    err = (out.cpu().double() - ref).abs()
    ulp = _bf16_ulp(torch.maximum(ref.abs(), x.double().abs() * 2 ** -16))
    bad = err > ulp
    assert not bad.any(), f"{int(bad.sum())} elements, first at {bad.nonzero()[0].tolist()}"
    # torch's CUDA gelu(approximate="tanh") on the same bf16 input: the same formula, so mostly the same bf16 values
    same = float((out == torch.nn.functional.gelu(x.to(DEV), approximate="tanh")).float().mean())
    print(f"gelu_tanh_fwd rows={rows} I={I}: max err / ulp {float((err / ulp).max()):.3f}, equal to torch {same:.5f}")


@pytest.mark.parametrize("rows,I", SHAPES)
def test_gelu_tanh_bwd_rows_within_the_bf16_rounding_bound(rows, I):
    x = _pre(rows, I, 7 * rows + I)
    g = torch.Generator().manual_seed(I)
    dout = (torch.randn(rows, I, generator=g) * torch.exp(torch.randn(rows, 1, generator=g))).to(torch.bfloat16)
    dpre = ops.gelu_tanh_bwd(x.to(DEV), dout.to(DEV))
    torch.cuda.synchronize()
    assert dpre.dtype == torch.bfloat16 and dpre.shape == (rows, I)
    ref = dout.double() * gelu_tanh_grad64(x)
    d = dpre.cpu().double()
    err = (d - ref).norm(dim=1)
    bound = 2 ** -8 * ref.norm(dim=1) + 1e-30  # one bf16 rounding (2^-9 relative) plus the fp32 evaluation, with margin
    assert (err <= bound).all(), f"rows {(err > bound).nonzero().flatten()[:5].tolist()}"
    print(f"gelu_tanh_bwd rows={rows} I={I}: worst row rel {float((err / ref.norm(dim=1).clamp_min(1e-30)).max()):.2e}")


@pytest.mark.parametrize("rows,I", [(3 * 257, 4096), (32 * 256, 2816), (300, 8)])
def test_gelu_tanh_e4m3(rows, I):
    """scales and codes as tests/test_fp8_gpu.py checks the GLU: s = amax / 448 (1 for a zero row), q = e4m3(y / s).  The
    kernel quantizes its fp32 gelu_tanh, whose 1 + tanh(.) carries an absolute error of a few 2^-24 (where it cancels, for
    x < 0, that is a large relative error), so y / s is known to within tol = (|x| + |y|) 2^-22 / s plus 1e-6 relative; a
    code may be the rounding of any value in that band, which differs from the rounding of y / s only near a midpoint."""
    x = _pre(rows, I, I + 3)
    x[1] = 0  # an all-zero row
    x[2, 3 % I] = 400.0  # a single large outlier
    out = ops.gelu_tanh_fwd(x.to(DEV), out_dtype=ops.FP8)
    torch.cuda.synchronize()
    assert isinstance(out, ops.F8) and out.q.shape == (rows, I) and out.s.shape == (rows,)
    y = gelu_tanh64(x)
    s = out.s.cpu()
    amax = y.abs().amax(dim=1)
    assert torch.allclose(s, torch.where(amax > 0, (amax / 448.0).float(), torch.ones_like(s)), rtol=2e-6, atol=0)
    v = y / s.double()[:, None]
    tol = (x.double().abs() + y.abs()) * 2 ** -22 / s.double()[:, None] + 1e-6 * v.abs().clamp_min(1.0)
    e4 = lambda t: t.clamp(-448, 448).to(E4M3).double()  # noqa: E731  (satfinite, as the kernel stores)
    q = out.q.cpu().double()
    ok = (q >= e4(v - tol)) & (q <= e4(v + tol))  # rounding is monotone: the codes of the band lie between these two
    assert ok.all(), f"{int((~ok).sum())} codes off, first at {(~ok).nonzero()[0].tolist()}"
    print(f"gelu_tanh e4m3 rows={rows} I={I}: {int((q != e4(v)).sum())} of {q.numel()} codes at a rounding midpoint")


def test_gelu_tanh_e4m3_rejects_rows_wider_than_4096():
    with pytest.raises(Exception, match="I <= 4096"):
        ops.gelu_tanh_fwd(torch.zeros(4, 4104, dtype=torch.bfloat16, device=DEV), out_dtype=ops.FP8)


# ------------------------------------------------------------------------------------------------------------- model
def _model(g, **over):
    """the fixture's model: its weights rebuilt from the fixture's seeds (tests/test_fused_mlp_cpu.py pins them)"""
    return GF.seeded_model(MaskGiTUViT_v2, **over)[0].to(DEV)


def _args(g):
    return [g[k].to(DEV) for k in ARGS]


def _train(m, g, ckpt=False, **kw):
    m.train()
    if ckpt:
        m.enable_gradient_checkpointing()
    m.zero_grad(set_to_none=True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        logits, loss = m(*_args(g), labels=g["labels"].to(DEV), **kw)
    loss.backward()
    torch.cuda.synchronize()
    return logits.detach().clone(), loss.detach().clone()


@pytest.mark.parametrize("weighted", [False, True])
def test_micro_fused_mlp_vs_reference_fixture(golden, weighted):
    """tolerances of tests/test_uvit_v2_gpu.py: logits 2e-2, loss 2e-3, every gradient rel-L2 8e-2 (query / key excepted)
    and cosine > 0.95, i.e. rel-L2 below 0.3 for all.  The fixture keeps each gradient's signature, so the rel-L2 is the
    estimate of make_golden_fused_mlp.signature_error"""
    g = golden(FIXTURE)
    m = _model(g)
    kw = dict(loss_weight=g["loss_weight"].to(DEV)) if weighted else dict(label_smoothing=0.1)
    logits, loss = _train(m, g, **kw)
    want_loss, want = (g["loss_weighted"], g["grads_weighted"]) if weighted else (g["loss"], g["grads"])
    if not weighted:
        assert _rel(logits, g["logits"]) < 2e-2, _rel(logits, g["logits"])
    assert abs(float(loss) - float(want_loss)) / float(want_loss) < 2e-3
    assert [n for n, _ in m.named_parameters()] == list(want)
    errs = {n: GF.signature_error(p.grad, want[n]) for n, p in m.named_parameters()}
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:6]
    print("worst grad rel-L2 (estimated):", ", ".join(f"{k}={v:.2e}" for k, v in worst))
    bad = {k: v for k, v in errs.items() if v > 8e-2 and not (".query." in k or ".key." in k)}
    assert not bad, bad
    assert max(errs.values()) < 0.3, worst
    if not weighted:  # the no_grad path, the one generate2 runs
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            assert _rel(m.eval()(*_args(g)), g["logits"]) < 2e-2


@pytest.mark.parametrize("p", [0.0, 0.1])
def test_gradient_checkpointing_is_bit_identical(golden, p):
    g = golden(FIXTURE)
    runs = []
    for ckpt in (False, True):
        torch.manual_seed(11)
        runs.append(_train(_model(g, hidden_dropout=p, attention_dropout=p), g, ckpt=ckpt, label_smoothing=0.1))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


@pytest.mark.parametrize("fp8", [False, True])
def test_generate2_cuda_graph_equals_eager(golden, fp8):
    g = golden(FIXTURE)
    m = _model(g).eval()
    if fp8:
        m.set_gemm_precision("fp8")
    kw = dict(encoder_hidden_states=g["encoder_hidden_states"].to(DEV), cond_embeds=g["cond_embeds"].to(DEV),
              micro_conds=g["micro_conds"][:1].to(DEV), empty_embeds=g["empty_embeds"].to(DEV),
              empty_cond_embeds=g["empty_cond_embeds"].to(DEV), temperature=(2.0, 0.0), timesteps=6, seq_len=16,
              guidance_scale=3.0)
    gen = lambda: torch.Generator(device=DEV).manual_seed(11)  # noqa: E731
    a = m.generate2(**kw, generator=gen())
    e = m.generate2(**kw, use_cuda_graph=False, generator=gen())
    assert torch.equal(a, e) and m._graph is not None
    assert int(a.min()) >= 0 and int(a.max()) < 64
    # release the captured graph here: the model sits in a reference cycle (its operand cache points back at it), and a
    # cyclic collection that frees a graph while a later test is capturing its own would invalidate that capture
    m._graph = None


def _walk(d):
    for v in (d.values() if isinstance(d, dict) else d):
        if isinstance(v, (dict, list)):
            yield from _walk(v)
        elif isinstance(v, torch.Tensor):
            yield v


@pytest.mark.parametrize("opt_cls", [FusedAdamW, FusedLion, FusedAdamW8bit])
def test_fused_optimizer_steps_write_the_fused_mlp_operands(golden, opt_cls):
    """model=: the optimizer writes the bf16 operands ("wi" = wi_0 alone) itself; they equal a fresh rebuild"""
    g = golden(FIXTURE)
    m = _model(g)
    opt = opt_cls(m.parameters(), lr=1e-3, weight_decay=0.01, model=m)
    for _ in range(2):
        _train(m, g, label_smoothing=0.1)
        opt.step()
    torch.cuda.synchronize()
    key = m._cache_key
    W = m._weights()
    assert m._cache_key == key  # no rebuild: the step moved the key
    fresh, _, _, _ = m._build_weights()
    assert W["layers"][0]["wi"].shape == m.transformer_layers[0].ffn.wi_0.weight.shape
    got, want = list(_walk(W)), list(_walk(fresh))
    assert len(got) == len(want)
    for a, b in zip(got, want):
        assert torch.equal(a, b)


def test_fp8_mode(golden):
    g = golden(FIXTURE)
    m = _model(g).eval()
    args = _args(g)
    with torch.no_grad():
        ref = m(*args)
        out = m.set_gemm_precision("fp8")(*args)
    assert any(isinstance(v, ops.F8) for layer in m._weights()["layers"] for v in layer.values())
    rel = _rel(out, ref)
    print(f"micro fused-MLP fixture: FP8 vs bf16 logits rel-L2 {rel:.3e} (GLU micro fixture: 0.024)")
    assert torch.isfinite(out).all() and rel < 0.024
    m.train()
    with pytest.raises(RuntimeError, match="inference only"):
        m(*args, labels=g["labels"].to(DEV))
