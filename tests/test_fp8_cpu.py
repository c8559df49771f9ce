"""The FP8 GEMM precision of MaskGiTUViT_v2 without a GPU: the host code runs on the torch restatements of
tests/cpu_math_ops.py, extended here by the e4m3 forms of the producers, the FP8 GEMM and the weight quantizer.

  * bf16 mode (the default, and after a round trip through FP8) makes the same ops calls and gives the same logits;
  * FP8 mode routes exactly the transformer layers' [q;k;v], cross-attention q, [wi_0;wi_1] and wo GEMMs and the blocks'
    channelwise[0] and attention q GEMMs, each fed by the pass that produces its activation;
  * FP8 mode refuses training-mode and grad-enabled forwards;
  * the weight operands are the per-row e4m3 quantization of the bf16 operands (against torch.float8_e4m3fn), and stay
    so after fused-optimizer steps with model=, EMA swaps, load_state_dict and in-place edits;
  * the ctypes table lists the new entry points (tests/test_boundary_cpu.py checks it against the header)."""
import pytest
import torch

from open_muse_b200 import EMAModel, FusedAdamW, FusedLion, MaskGiTUViT_v2, ops
from open_muse_b200 import _lib
from tests import cpu_math_ops
from tests import test_lion_cpu

ARGS = ("input_ids", "encoder_hidden_states", "cond_embeds", "micro_conds")
E4M3 = torch.float8_e4m3fn


def quant(x):
    """per-row e4m3: s = amax / 448 (1 for an all-zero row), q = e4m3_rn_satfinite(x / s)"""
    x = x.float()
    amax = x.abs().amax(dim=1)
    s = torch.where(amax > 0, amax / 448.0, torch.ones_like(amax))
    return ops.F8((x / s[:, None]).clamp(-448, 448).to(E4M3), s)


def deq(f):
    return f.q.float() * f.s[:, None]


def install(mp, log=None):
    """cpu_math_ops (exact mode) plus the e4m3 forms; log (list) receives (op, e4m3 output?, F8 weight name or None)"""
    cpu_math_ops.install(mp, exact=True)
    base = {k: getattr(ops, k) for k in ("linear_fwd", "add_norm_mod", "dwconv3x3_norm", "glu_fwd")}

    def rec(op, f8, w=None):
        if log is not None:
            log.append((op, f8, w))

    def linear_fwd(x, w, out_dtype=None, res=None, n_valid=None):
        if isinstance(x, ops.F8):
            assert isinstance(w, ops.F8) and res is None and out_dtype in (None, torch.bfloat16)
            rec("linear_fwd", True, id(w))
            return (deq(x) @ deq(w).t()).to(torch.bfloat16)
        assert not isinstance(w, ops.F8)
        rec("linear_fwd", False)
        return base["linear_fwd"](x, w, out_dtype=out_dtype, res=res, n_valid=n_valid)

    def add_norm_mod(a, w, eps, rms, out_dtype=None, **kw):
        if out_dtype == ops.FP8:
            r, y = base["add_norm_mod"](a, w, eps, rms, out_dtype=torch.float32, **kw)
            rec("add_norm_mod", True)
            return r, quant(y)
        rec("add_norm_mod", False)
        return base["add_norm_mod"](a, w, eps, rms, **({} if out_dtype is None else {"out_dtype": out_dtype}), **kw)

    def dwconv3x3_norm(x, wk, norm_w, B, hh, ww, eps, rms, save_conv=False, **kw):
        if kw.get("out_dtype") == ops.FP8:
            assert not save_conv
            rec("dwconv3x3_norm", True)
            return quant(base["dwconv3x3_norm"](x, wk, norm_w, B, hh, ww, eps, rms))
        assert not kw
        rec("dwconv3x3_norm", False)
        return base["dwconv3x3_norm"](x, wk, norm_w, B, hh, ww, eps, rms, save_conv=save_conv)

    def glu_fwd(ab, **kw):
        if kw.get("out_dtype") == ops.FP8:
            rec("glu_fwd", True)
            return quant(base["glu_fwd"](ab))
        assert not kw
        rec("glu_fwd", False)
        return base["glu_fwd"](ab)

    def quantize_rows_e4m3(x, out=None):
        f = quant(x)
        if out is None:
            return f
        out.q.copy_(f.q), out.s.copy_(f.s)
        return out

    for name, fn in dict(linear_fwd=linear_fwd, add_norm_mod=add_norm_mod, dwconv3x3_norm=dwconv3x3_norm, glu_fwd=glu_fwd,
                         quantize_rows_e4m3=quantize_rows_e4m3).items():
        mp.setattr(ops, name, fn)


def _model(g, mp):
    m = MaskGiTUViT_v2(**g["config"])
    m.load_state_dict(g["state_dict"])
    mp.setattr(MaskGiTUViT_v2, "device", property(lambda self: torch.device("cpu")), raising=False)
    return m.eval()


def _fp8_sites(m):
    """name of every F8 weight of the FP8-mode operand dict, by object id"""
    W = m._weights()
    out = {}
    for j, w in enumerate(W["down"] + W["up"]):
        out[id(w["cw0"])] = f"block{j}.cw0"
        out[id(w["a1"]["q"])] = f"block{j}.attention.q"
        out[id(w["a2"]["q"])] = f"block{j}.crossattention.q"
    for i, w in enumerate(W["layers"]):
        out[id(w["sa"]["qkv"])] = f"layer{i}.qkv"
        out[id(w["ca"]["q"])] = f"layer{i}.crossattention.q"
        out[id(w["wi"])] = f"layer{i}.wi"
        out[id(w["wo"])] = f"layer{i}.wo"
    assert all(isinstance(v, ops.F8) for v in _walk(W) if id(v) in out)
    return out


def _walk(d):
    for v in (d.values() if isinstance(d, dict) else d):
        if isinstance(v, (dict, list)):
            yield from _walk(v)
        else:
            yield v


@pytest.mark.parametrize("name", ["micro_uvit_v2.pt", "micro_uvit_v2_downup.pt"])
def test_bf16_mode_calls_and_logits_unchanged_by_a_round_trip(golden, monkeypatch, name):
    g = golden(name)
    log_a, log_b = [], []
    install(monkeypatch, log_a)
    a = _model(g, monkeypatch)
    args = [g[k] for k in ARGS]
    with torch.no_grad():
        la = a(*args)
    install(monkeypatch, log_b)
    b = _model(g, monkeypatch)
    with torch.no_grad():
        b.set_gemm_precision("fp8")
        b(*args)
        log_b.clear()
        b.set_gemm_precision("bf16")
        lb = b(*args)
    assert log_a == log_b and not any(f8 for _, f8, _ in log_a)
    assert torch.equal(la, lb)
    assert not any(isinstance(v, ops.F8) for v in _walk(b._weights()))


@pytest.mark.parametrize("name", ["micro_uvit_v2.pt", "micro_uvit_v2_downup.pt"])
def test_fp8_mode_routes_exactly_the_listed_sites(golden, monkeypatch, name):
    g = golden(name)
    log = []
    install(monkeypatch, log)
    m = _model(g, monkeypatch).set_gemm_precision("fp8")
    args = [g[k] for k in ARGS]
    with torch.no_grad():
        ref = m.set_gemm_precision("bf16")(*args)
        log.clear()
        out = m.set_gemm_precision("fp8")(*args)
    sites = _fp8_sites(m)
    used = [sites[w] for op, f8, w in log if op == "linear_fwd" and f8]
    assert sorted(used) == sorted(sites.values())  # each FP8 site once per forward, and nothing else
    producers = sorted(op for op, f8, _ in log if f8 and op != "linear_fwd")
    L, R = len(m.transformer_layers), len(m.down_blocks[0].res_blocks) * 2
    assert producers == sorted(["add_norm_mod"] * (3 * L + 2 * R) + ["glu_fwd"] * L + ["dwconv3x3_norm"] * R)
    rel = float((out - ref).norm() / ref.norm())
    assert 0 < rel < 0.1, rel


def test_fp8_mode_is_inference_only(golden, monkeypatch):
    g = golden("micro_uvit_v2.pt")
    install(monkeypatch)
    m = _model(g, monkeypatch).set_gemm_precision("fp8")
    args = [g[k] for k in ARGS]
    with pytest.raises(RuntimeError, match="inference only"):
        m(*args, labels=g["labels"])
    m.train()
    with torch.no_grad(), pytest.raises(RuntimeError, match="inference only"):
        m(*args)
    with pytest.raises(RuntimeError, match="inference only"):
        m.generate2(encoder_hidden_states=g["encoder_hidden_states"], cond_embeds=g["cond_embeds"],
                    micro_conds=g["micro_conds"][:1], empty_embeds=g["empty_embeds"], empty_cond_embeds=g["empty_cond_embeds"])
    with pytest.raises(ValueError):
        m.set_gemm_precision("fp16")
    odd = MaskGiTUViT_v2(**dict(g["config"], intermediate_size=136))  # 8 mod 16: fine in bf16, not for e4m3 rows
    with pytest.raises(ValueError, match="multiples of 16"):
        odd.set_gemm_precision("fp8")
    assert odd.gemm_precision == "bf16"
    assert "gemm_precision" not in m.config


def test_weight_quantization_is_per_row_e4m3_of_the_bf16_operands(golden, monkeypatch):
    g = golden("micro_uvit_v2.pt")
    install(monkeypatch)
    m = _model(g, monkeypatch).set_gemm_precision("fp8")
    W = m._weights()
    l0 = m.transformer_layers[0]
    qkv = torch.cat([l0.attention.query.weight, l0.attention.key.weight, l0.attention.value.weight]).detach()
    f = W["layers"][0]["sa"]["qkv"]
    amax = qkv.abs().amax(1)
    assert torch.equal(f.s, amax / 448)
    assert torch.equal(f.q.view(torch.uint8), (qkv / f.s[:, None]).to(E4M3).view(torch.uint8))
    assert f.q.dtype == E4M3 and f.q.shape == qkv.shape
    # satfinite and the all-zero row
    z = torch.zeros(3, 16)
    z[1, 2] = 1.0
    q = quant(z)
    assert torch.equal(q.s, torch.tensor([1.0, 1.0 / 448, 1.0])) and float(q.q.float()[1, 2]) == 448.0


def _coherent(m):
    """every F8 weight equals the quantization of the bf16 operand it was built from, and of a freshly built cache"""
    m._weights()
    fresh, _, _, _ = m._build_weights()
    for src, f8 in m._packed.quantized:
        want = quant(src)
        assert torch.equal(f8.q.view(torch.uint8), want.q.view(torch.uint8)) and torch.equal(f8.s, want.s)
    got = [v for v in _walk(m._weights()) if isinstance(v, ops.F8)]
    ref = [v for v in _walk(fresh) if isinstance(v, ops.F8)]
    assert len(got) == len(ref) > 0
    for a, b in zip(got, ref):
        assert torch.equal(a.q.view(torch.uint8), b.q.view(torch.uint8)) and torch.equal(a.s, b.s)


@pytest.mark.parametrize("opt_cls", [FusedAdamW, FusedLion])
def test_fp8_copies_follow_optimizer_steps_ema_and_loads(golden, monkeypatch, opt_cls):
    g = golden("micro_uvit_v2.pt")
    install(monkeypatch)
    m = _model(g, monkeypatch)
    args = [g[k] for k in ARGS]
    with torch.no_grad():
        m.set_gemm_precision("fp8")(*args)  # the FP8 cache exists before the step
    m.set_gemm_precision("bf16").train()
    _, loss = m(*args, labels=g["labels"])
    loss.backward()
    ema = EMAModel(m.parameters(), decay=0.5)
    opt = opt_cls(m.parameters(), lr=1e-2, ema=ema, model=m)
    m.set_gemm_precision("fp8").eval()
    before = [v.q.clone() for v in _walk(m._weights()) if isinstance(v, ops.F8)]
    test_lion_cpu.install(monkeypatch)  # the fused step's library call, restated
    opt.step()
    install(monkeypatch)
    key = m._cache_key
    after = [v.q for v in _walk(m._weights()) if isinstance(v, ops.F8)]
    assert m._cache_key == key  # the step moved the key itself: no rebuild ...
    assert any(not torch.equal(a.view(torch.uint8), b.view(torch.uint8)) for a, b in zip(after, before))
    _coherent(m)  # ... and re-quantized every FP8 copy
    with torch.no_grad():
        base = m(*args)
        for s in ema.shadow_params:  # shadows that differ from the parameters whatever the step's decay
            s.mul_(0.9)
        ema.store(m.parameters())
        ema.copy_to(m.parameters())
        _coherent(m)
        assert not torch.equal(m(*args), base)
        ema.restore(m.parameters())
        assert torch.equal(m(*args), base)
        m.transformer_layers[0].ffn.wo.weight.mul_(1.5)
        _coherent(m)
        m.load_state_dict(g["state_dict"])
        _coherent(m)


def test_ctypes_table_lists_the_fp8_entry_points():
    assert _lib.ABI_VERSION == 11
    for name in ("muse_gemm_fp8", "muse_quantize_rows_e4m3"):
        assert name in _lib.SIGNATURES
