"""The FP8 GEMM precision of MaskGitTransformer without a GPU: the host code runs on the torch restatements of
tests/cpu_math_ops.py, extended here by the e4m3 forms of the norm passes, the GLU pass, the FP8 GEMM with and without
its fused residual, and the weight quantizer.

  * bf16 mode (the default, and after a round trip through FP8) makes the same ops calls and gives the same logits;
  * FP8 mode routes exactly each layer's [q;k;v], cross-attention q, [wi_0;wi_1] and wo GEMMs, each fed by the pass the
    table of DESIGN.md section 5 names (the fused norm2 pass and the separate norm pass both), wo with its residual;
  * FP8 mode refuses training-mode and grad-enabled forwards, and widths the e4m3 passes do not cover;
  * the weight operands are the per-row e4m3 quantization of the bf16 operands (against torch.float8_e4m3fn), keep their
    addresses, and stay so after fused-optimizer steps with model=, EMA swaps, load_state_dict and in-place edits;
  * the ctypes table lists the new entry points, and the norm and GEMM kernels of the bf16 paths compile to the same SASS
    as before the e4m3 forms were added.

The e4m3 contracts restated here: a producer stores q = e4m3_rn_satfinite(y / s) with s = amax(|y[r]|) / 448 (1 for an
all-zero row), y the fp32 value its bf16 form rounds; muse_gemm_fp8_res stores res + bf16(acc * sa[m] * sb[n])."""
import os
import subprocess

import pytest
import torch

from open_muse_b200 import EMAModel, FusedAdamW, FusedAdamW8bit, FusedLion, MaskGitTransformer, ops
from open_muse_b200 import _lib
from tests import cpu_math_ops
from tests import test_adamw8bit_cpu
from tests import test_lion_cpu
from tests.test_fused_mlp_cpu import _demangled_sass, obj_tools

E4M3 = torch.float8_e4m3fn
FIXTURES = ["micro_transformer.pt", "micro_t2i_transformer.pt", "micro_t2i_proj_transformer.pt", "hd48_transformer.pt"]


def quant(x):
    """per-row e4m3: s = amax / 448 (1 for an all-zero row), q = e4m3_rn_satfinite(x / s)"""
    x = x.float()
    amax = x.abs().amax(dim=1)
    s = torch.where(amax > 0, amax / 448.0, torch.ones_like(amax))
    return ops.F8((x / s[:, None]).clamp(-448, 448).to(E4M3), s)


def deq(f):
    return f.q.float() * f.s[:, None]


def install(mp, log=None):
    """cpu_math_ops (exact mode) plus the e4m3 forms.  log (list) receives one entry per ops call: (name, keyword names,
    e4m3 output?) for the producers and bf16 GEMMs, ("fp8_gemm", F8 weight id, producer of the activation, residual?) for
    the FP8 GEMMs."""
    cpu_math_ops.install(mp, exact=True)
    producer = {}  # id of an e4m3 activation -> the pass that wrote it

    def rec(*entry):
        if log is not None:
            log.append(entry)

    def logged(name):
        base = getattr(ops, name)

        def fn(*a, **kw):
            rec(name, tuple(sorted(kw)), False)
            return base(*a, **kw)
        mp.setattr(ops, name, fn)

    for name in ("linear_fwd", "gemm", "norm_fwd", "norm2_fwd", "glu_fwd", "attn_fwd", "embed_fwd", "cast_bf16", "pack_bf16"):
        logged(name)
    base = {k: getattr(ops, k) for k in ("linear_fwd", "norm_fwd", "norm2_fwd", "glu_fwd")}

    def produced(f8, what):
        producer[id(f8)] = what
        rec(what, (), True)
        return f8

    def linear_fwd(x, w, out_dtype=torch.bfloat16, res=None, n_valid=None):
        if isinstance(x, ops.F8):
            assert isinstance(w, ops.F8) and n_valid is None
            rec("fp8_gemm", id(w), producer.pop(id(x)), res is not None)
            y = (deq(x) @ deq(w).t()).to(torch.bfloat16)
            return y if res is None else res + y.float()
        assert not isinstance(w, ops.F8)
        return base["linear_fwd"](x, w, out_dtype=out_dtype, res=res, n_valid=n_valid)

    def norm_fwd(x, w, eps, out_dtype, act=0, **kw):
        if out_dtype == ops.FP8:
            assert "dropout" not in kw and act in (0, 2)
            y, st = cpu_math_ops.norm_fwd(x, w, eps, torch.float32, act=act, **kw)
            return produced(quant(y), f"norm_fwd act {act}"), st
        return base["norm_fwd"](x, w, eps, out_dtype, act=act, **kw)

    def norm2_fwd(*a, h2_dtype=None, **kw):
        if h2_dtype == ops.FP8:
            x2, h2, st = cpu_math_ops.norm2_fwd(*a, **kw)
            return x2, produced(quant(h2), "norm2_fwd"), st
        assert h2_dtype is None
        return base["norm2_fwd"](*a, **kw)

    def glu_fwd(ab, out_dtype=None, **kw):
        if out_dtype == ops.FP8:
            assert not kw
            return produced(quant(cpu_math_ops.glu_fwd(ab)), "glu_fwd")
        assert out_dtype is None
        return base["glu_fwd"](ab, **kw)

    def quantize_rows_e4m3(x, out=None):
        f = quant(x)
        if out is None:
            return f
        out.q.copy_(f.q), out.s.copy_(f.s)
        return out

    for name, fn in dict(linear_fwd=linear_fwd, norm_fwd=norm_fwd, norm2_fwd=norm2_fwd, glu_fwd=glu_fwd,
                         quantize_rows_e4m3=quantize_rows_e4m3).items():
        mp.setattr(ops, name, fn)


def _model(g, mp):
    if "state_dict" in g:
        m = MaskGitTransformer(**g["config"])
        m.load_state_dict(g["state_dict"])
    else:  # hd48: the weights follow from the seed
        torch.manual_seed(g["seed"])
        m = MaskGitTransformer(**g["config"])
    mp.setattr(MaskGitTransformer, "device", property(lambda self: torch.device("cpu")), raising=False)
    return m.eval()


def _inputs(g):
    if "batch" in g:
        return dict(input_ids=g["batch"]["input_ids"])
    return dict(input_ids=g["input_ids"], encoder_hidden_states=g["encoder_hidden_states"])


def _labels(g):
    return g["batch"]["labels"] if "batch" in g else g["labels"]


def _sites(m):
    """the F8 weight of each FP8 site, by object id -> (layer, site)"""
    out = {}
    for i, d in enumerate(m._packed.layers):
        for name, w in d.items():
            if isinstance(w, ops.F8):
                out[id(w)] = (i, name)
    return out


@pytest.mark.parametrize("name", FIXTURES)
def test_bf16_mode_calls_and_logits_unchanged_by_a_round_trip(golden, monkeypatch, name):
    g = golden(name)
    log_a, log_b = [], []
    install(monkeypatch, log_a)
    a = _model(g, monkeypatch)
    with torch.no_grad():
        la = a(**_inputs(g))
    install(monkeypatch, log_b)
    b = _model(g, monkeypatch)
    with torch.no_grad():
        b(**_inputs(g))
        flat = b._packed.flat.data_ptr()
        b.set_gemm_precision("fp8")
        b(**_inputs(g))
        f8 = [(w.q.data_ptr(), w.s.data_ptr()) for _, w in b._packed.quantized]
        log_b.clear()
        assert b.set_gemm_precision("bf16") is b and b.gemm_precision == "bf16"
        lb = b(**_inputs(g))
        log_bf16 = list(log_b)
        # the buffers depend on the parameters' storage only: no switch re-allocates them (captured graphs stay valid)
        assert b._packed.flat.data_ptr() == flat
        b.set_gemm_precision("fp8")
        b(**_inputs(g))
        assert b._packed.flat.data_ptr() == flat and f8 == [(w.q.data_ptr(), w.s.data_ptr()) for _, w in b._packed.quantized]
        assert torch.equal(b.set_gemm_precision("bf16")(**_inputs(g)), lb)
    assert log_a == log_bf16 and not any(e[0] == "fp8_gemm" or e[2] is True for e in log_a)
    assert torch.equal(la, lb)
    assert not b._packed.quantized and not _sites(b)


@pytest.mark.parametrize("name", FIXTURES)
def test_fp8_mode_routes_exactly_the_listed_sites(golden, monkeypatch, name):
    g = golden(name)
    log = []
    install(monkeypatch, log)
    m = _model(g, monkeypatch)
    c = m.config
    with torch.no_grad():
        ref = m(**_inputs(g))
        log.clear()
        out = m.set_gemm_precision("fp8")(**_inputs(g))
    sites = _sites(m)
    want_sites = {"qkv", "wi", "wo"} | ({"cq"} if c.add_cross_attention else set())
    assert sorted(sites.values()) == sorted((i, s) for i in range(c.num_hidden_layers) for s in want_sites)
    fused = c.use_normformer and not c.add_cross_attention  # post-attention norm + FFN pre-norm in one pass
    want = {"qkv": ("norm_fwd act 0", False), "cq": ("norm_fwd act 0", False),
            "wi": ("norm2_fwd" if fused else "norm_fwd act 0", False),
            "wo": ("norm_fwd act 2" if c.use_normformer else "glu_fwd", True)}
    used = [(sites[w], prod, res) for kind, w, prod, res in (e for e in log if e[0] == "fp8_gemm")]
    # each FP8 site once per forward, fed by its producer, and nothing else
    assert sorted(u[0] for u in used) == sorted(sites.values())
    for (i, site), prod, res in used:
        assert (prod, res) == want[site], (i, site, prod, res)
    n_e4m3 = sum(1 for e in log if e[0] != "fp8_gemm" and e[2] is True)
    assert n_e4m3 == len(sites)  # every e4m3 activation is consumed by an FP8 GEMM
    rel = float((out - ref).norm() / ref.norm())
    assert 0 < rel < 0.1, rel


def test_fp8_mode_is_inference_only_and_checks_widths(golden, monkeypatch):
    g = golden("micro_transformer.pt")
    install(monkeypatch)
    m = _model(g, monkeypatch).set_gemm_precision("fp8")
    with pytest.raises(RuntimeError, match="inference only"):
        m(**_inputs(g), labels=_labels(g))
    m.train()
    with torch.no_grad(), pytest.raises(RuntimeError, match="inference only"):
        m(**_inputs(g))
    with pytest.raises(RuntimeError, match="inference only"):
        m.generate2(class_ids=g["batch"]["class_ids"].clone(), timesteps=2, use_cuda_graph=False)
    with pytest.raises(ValueError):
        m.set_gemm_precision("fp16")
    assert m.gemm_precision == "fp8" and "gemm_precision" not in m.config
    small = dict(g["config"], num_hidden_layers=0)
    # (hidden_size is a multiple of 16 whenever its head width is one of the supported 48, 64, 96 or 128)
    for widths, match in (({"intermediate_size": 136}, "multiples of 16"),
                          ({"hidden_size": 1280, "num_attention_heads": 20, "intermediate_size": 5120}, "<= 1024"),
                          ({"hidden_size": 1024, "num_attention_heads": 16, "intermediate_size": 4112}, "<= 4096")):
        odd = MaskGitTransformer(**dict(small, **widths))
        with pytest.raises(ValueError, match=match):
            odd.set_gemm_precision("fp8")
        assert odd.gemm_precision == "bf16"


def test_every_reference_v1_config_takes_fp8(golden):
    """the configs the reference scripts build as a MaskGitTransformer pass the width checks; the *_larger U-ViT widths,
    instantiated as v1, do not (they keep working in bf16)"""
    import json

    configs = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "configs.json")))
    takes = {}
    for name, c in configs.items():
        t = c["transformer"]
        m = MaskGitTransformer(**dict(t, num_hidden_layers=0, vocab_size=16, codebook_size=8, num_classes=None,
                                      add_cross_attention=False, use_conv_in_out=False, embedding_size=None))
        try:
            m.set_gemm_precision("fp8")
            takes[name] = True
        except ValueError:
            takes[name] = False
        if c["script_class"] == "MaskGitTransformer":
            assert takes[name], name
    assert {n for n, ok in takes.items() if not ok} >= {n for n in configs if "larger" in n}
    assert any(c["script_class"] == "MaskGitTransformer" for c in configs.values())


def test_weight_operands_are_per_row_e4m3_of_the_bf16_operands(golden, monkeypatch):
    g = golden("micro_t2i_transformer.pt")
    install(monkeypatch)
    m = _model(g, monkeypatch).set_gemm_precision("fp8")
    with torch.no_grad():
        m(**_inputs(g))
    l0 = m.transformer_layers[0]
    qkv = torch.cat([l0.attention.query.weight, l0.attention.key.weight, l0.attention.value.weight]).detach()
    f = m._packed.layers[0]["qkv"]
    amax = qkv.abs().amax(1)
    assert torch.equal(f.s, amax / 448)
    assert torch.equal(f.q.view(torch.uint8), (qkv / f.s[:, None]).to(E4M3).view(torch.uint8))
    assert f.q.dtype == E4M3 and f.q.shape == qkv.shape
    # satfinite and the all-zero row
    z = torch.zeros(3, 16)
    z[1, 2] = 1.0
    q = quant(z)
    assert torch.equal(q.s, torch.tensor([1.0, 1.0 / 448, 1.0])) and float(q.q.float()[1, 2]) == 448.0


def _addresses(m):
    return [(w.q.data_ptr(), w.s.data_ptr()) for _, w in m._packed.quantized]


def _coherent(m, addresses):
    """every F8 weight equals the quantization of the bf16 operand it stands for, at the address it had"""
    m._packed.refresh()
    assert _addresses(m) == addresses
    for src, f8 in m._packed.quantized:
        want = quant(src)
        assert torch.equal(f8.q.view(torch.uint8), want.q.view(torch.uint8)) and torch.equal(f8.s, want.s)
    assert len(m._packed.quantized) == len(_sites(m)) > 0


@pytest.mark.parametrize("opt_cls", [FusedAdamW, FusedLion, FusedAdamW8bit])
def test_fp8_copies_follow_optimizer_steps_ema_and_loads(golden, monkeypatch, opt_cls):
    g = golden("micro_t2i_proj_transformer.pt")
    install(monkeypatch)
    m = _model(g, monkeypatch)
    with torch.no_grad():
        m.set_gemm_precision("fp8")(**_inputs(g))  # the FP8 cache exists before the step
    addresses = _addresses(m)
    _coherent(m, addresses)
    m.set_gemm_precision("bf16").train()
    _, loss = m(**_inputs(g), labels=_labels(g))
    loss.backward()
    ema = EMAModel(m.parameters(), decay=0.5)
    opt = opt_cls(m.parameters(), lr=1e-2, ema=ema, model=m)
    m.set_gemm_precision("fp8").eval()
    m._packed.refresh()
    addresses = _addresses(m)
    before = [w.q.clone() for _, w in m._packed.quantized]
    (test_adamw8bit_cpu if opt_cls is FusedAdamW8bit else test_lion_cpu).install(monkeypatch)  # the fused step, restated
    opt.step()
    install(monkeypatch)
    key = m._packed.key
    m._packed.refresh()
    assert m._packed.key == key  # the step moved the key itself: no rebuild ...
    assert any(not torch.equal(a.view(torch.uint8), w.q.view(torch.uint8)) for a, (_, w) in zip(before, m._packed.quantized))
    _coherent(m, addresses)  # ... and re-quantized every FP8 copy in place
    with torch.no_grad():
        base = m(**_inputs(g))
        for s in ema.shadow_params:  # shadows that differ from the parameters whatever the step's decay
            s.mul_(0.9)
        ema.store(m.parameters())
        ema.copy_to(m.parameters())
        _coherent(m, addresses)
        assert not torch.equal(m(**_inputs(g)), base)
        ema.restore(m.parameters())
        _coherent(m, addresses)
        assert torch.equal(m(**_inputs(g)), base)
        m.transformer_layers[0].ffn.wo.weight.mul_(1.5)
        _coherent(m, addresses)
        m.load_state_dict(g["state_dict"])
        _coherent(m, addresses)


def test_ctypes_table_lists_the_fp8_transformer_entry_points():
    assert _lib.ABI_VERSION == 11
    for name in ("muse_gemm_fp8_res", "muse_norm_fwd_e4m3", "muse_norm2_fwd_e4m3"):
        assert name in _lib.SIGNATURES


# ------------------------------------------------------------------ SASS of the norm and GEMM kernels with an e4m3 form
# sha1 of each kernel's instruction list (cuobjdump -sass, addresses and encodings stripped) as nvcc 12.9 built
# csrc/norm.cu and csrc/gemm_wgmma.cu with build.NVCC_FLAGS before the F8 flag and the FP8 residual epilogue were added,
# under the names the kernels have now: the bf16 instantiations must still compile to exactly these instructions.
_GEMM = "void muse::<unnamed>::gemm_wgmma_kernel<(int){}, (bool){}, (bool){}, (int){}>(CUtensorMap_st, CUtensorMap_st, " \
        "CUtensorMap_st, CUtensorMap_st, muse::<unnamed>::GemmParams)"
NORM_SASS_SHA1 = {
    "glu_norm_fwd_kernel<(int)1, (bool)0, (bool)0, __nv_bfloat16>": "21ec17c612080c4d320da6cfcd3da20e45228c15",
    "glu_norm_fwd_kernel<(int)1, (bool)1, (bool)0, __nv_bfloat16>": "b7d8997902b4555b6181aac5de690077e6f5eef3",
    "glu_norm_fwd_kernel<(int)16, (bool)0, (bool)0, __nv_bfloat16>": "10355dd3665c29f26baddf3f1f14cc2796df1a8d",
    "glu_norm_fwd_kernel<(int)16, (bool)1, (bool)0, __nv_bfloat16>": "abb2d1c98301645811fb63e81d729729df8137dc",
    "glu_norm_fwd_kernel<(int)2, (bool)0, (bool)0, __nv_bfloat16>": "195d9dc6051653d97b5e3eb644f74eb89316cab8",
    "glu_norm_fwd_kernel<(int)2, (bool)1, (bool)0, __nv_bfloat16>": "33ce9e9a373a6dcc323641d8a30a2d0d711ab5d5",
    "glu_norm_fwd_kernel<(int)4, (bool)0, (bool)0, __nv_bfloat16>": "e6563cfe16a76217971f4c6c3df76b7cc042eb71",
    "glu_norm_fwd_kernel<(int)4, (bool)1, (bool)0, __nv_bfloat16>": "941ee8fbf673d9b3999edea1351c88318d345e26",
    "glu_norm_fwd_kernel<(int)8, (bool)0, (bool)0, __nv_bfloat16>": "ae07dc4088adb24bd74e061dbfd9ee420f25fb0f",
    "glu_norm_fwd_kernel<(int)8, (bool)1, (bool)0, __nv_bfloat16>": "89047417436da8cceb1ade61c4e64bf38682e6ac",
    "norm2_fwd_warp_kernel<(int)1, (bool)0, __nv_bfloat16>": "08744c22fe02f9c0d6a6b8446aeeb5dd71f8be22",
    "norm2_fwd_warp_kernel<(int)2, (bool)0, __nv_bfloat16>": "79ff42f109ac28f9ba561340277c88085e93e56b",
    "norm2_fwd_warp_kernel<(int)4, (bool)0, __nv_bfloat16>": "32cb88cff808b36bdf28fa62510ab76e8b52cfc9",
    "norm_fwd_warp_kernel<__nv_bfloat16, __nv_bfloat16, (int)1, (bool)0>": "2b100c0e6d205584fc0e224f315271c4093aa013",
    "norm_fwd_warp_kernel<__nv_bfloat16, __nv_bfloat16, (int)2, (bool)0>": "443e40d42a5e77ffd22ed1c7ecd7ff832968d444",
    "norm_fwd_warp_kernel<__nv_bfloat16, __nv_bfloat16, (int)4, (bool)0>": "d45232302e976f2185ee45fe32477da213902080",
    "norm_fwd_warp_kernel<__nv_bfloat16, float, (int)1, (bool)0>": "2b083b203d34b9490047694f514f18afd1dcb026",
    "norm_fwd_warp_kernel<__nv_bfloat16, float, (int)2, (bool)0>": "7aa24a34699753f92ea9dd54e1a664972d5fde1a",
    "norm_fwd_warp_kernel<__nv_bfloat16, float, (int)4, (bool)0>": "e2bf0194c4a8c6d969a45b549b5095d2386caed5",
    "norm_fwd_warp_kernel<float, __nv_bfloat16, (int)1, (bool)0>": "81e3ba2ccf7f8a0e2ca09b7fa49c002865554321",
    "norm_fwd_warp_kernel<float, __nv_bfloat16, (int)2, (bool)0>": "882fda24fdab52bfae17d6e473b9fa3765a41b21",
    "norm_fwd_warp_kernel<float, __nv_bfloat16, (int)4, (bool)0>": "ea6c21a1af44992e43d1087437d147a826acfa9e",
    "norm_fwd_warp_kernel<float, float, (int)1, (bool)0>": "21889f04776f64684cbe14a15676854f1fbba9c3",
    "norm_fwd_warp_kernel<float, float, (int)2, (bool)0>": "cae7f69347b833527f80a73bf1d14ba076657717",
    "norm_fwd_warp_kernel<float, float, (int)4, (bool)0>": "977ffee2c476b829a6159df584fec3846eec780c",
}
GEMM_SASS_SHA1 = {
    "muse::<unnamed>::splitk_reduce_kernel(const float *, float *, int, int, int, int, int, int, int)": "d5a1faf9b526c38fdbca01199e1da1356855990b",
    _GEMM.format(128, 0, 0, 0): "a19b6dc7f7319914c45451eafc07d1c9c41548b1",
    _GEMM.format(128, 0, 0, 1): "4de200444ec5f526b7a8f2fa46c5b45e34117d1a",
    _GEMM.format(128, 0, 0, 2): "b3f98b5d3e7f46008c0a87a442b42c3835f52a1a",
    _GEMM.format(128, 0, 0, 3): "430ceeac3cec0f38cf452334c76eab6c8b45e3d5",
    _GEMM.format(128, 0, 0, 4): "b810279371f42e8d69a3166e2691fcc726ac36da",
    _GEMM.format(128, 0, 0, 5): "60c96c018d023c056abaf7aaae923749e306daad",
    _GEMM.format(128, 0, 1, 0): "bfa0299b7b4a005585117c2d5ff6d819c8fdc51e",
    _GEMM.format(128, 0, 1, 1): "bb204f798c15d84fbba78c6fb617a9130a8893ac",
    _GEMM.format(128, 0, 1, 2): "513c75c0219c9e094a33e838958ba74150f5751d",
    _GEMM.format(128, 0, 1, 3): "eac72c27275c3eeb97d7b9068ed5bb2b3457c1c4",
    _GEMM.format(128, 0, 1, 4): "109a5a31474688ad0bafa91efae14a5f3cb79d7f",
    _GEMM.format(128, 1, 0, 0): "5ff5112235b29b486d8e1aeace008e1ff2137a03",
    _GEMM.format(128, 1, 0, 1): "23cf89d20610a1283caba29831016370f76c7d2e",
    _GEMM.format(128, 1, 0, 2): "6dfa8b8e3321f8df1cb11fd1ca188018d145bf5a",
    _GEMM.format(128, 1, 0, 3): "9c9cd839351a44015b75ed2fa0fae0dab6ab499f",
    _GEMM.format(128, 1, 0, 4): "f34fc0e872011c99010ba2cdc1ac231079912f3c",
    _GEMM.format(128, 1, 1, 0): "a723b1492e51669b9b9fdb738be071f6ef40cccb",
    _GEMM.format(128, 1, 1, 1): "af682c9948811ecad460fc4007a9f5ed3533b84f",
    _GEMM.format(128, 1, 1, 2): "0532f9825865a564016c0acd5fd49acfeb61543a",
    _GEMM.format(128, 1, 1, 3): "83b78e4feb773b8eaa35ed50e4a55a85cb950185",
    _GEMM.format(128, 1, 1, 4): "b4f033f337e2c09b48f31d1dc933191d400b333c",
    _GEMM.format(256, 0, 0, 0): "e4d26637f8f285e560c06fac9162d38496e55952",
    _GEMM.format(256, 0, 0, 1): "c3ecf4dd44219ed9ee6a03349ea0f26eb02cd494",
    _GEMM.format(256, 0, 0, 2): "5118580896293da5fc5e14c88c58e69b4c6e8b14",
    _GEMM.format(256, 0, 0, 3): "3590b0f244eadc6c7a30f0cf2a60461ce3280976",
    _GEMM.format(256, 0, 0, 4): "0de2d7fd6db55a99dff8f9478c432a58f7f6fe27",
    _GEMM.format(256, 0, 1, 0): "59ad512c640ce23e4e5cd35a6aa1f8ce3c863ca4",
    _GEMM.format(256, 0, 1, 1): "21e3b4395e534ce704c3146c39d5d9aaa87b4f54",
    _GEMM.format(256, 0, 1, 2): "100d336f3f73628ca43fcfb940bf8a02aed80e08",
    _GEMM.format(256, 0, 1, 3): "fde2ff5df1de692de77a340357d523b32501fd0f",
    _GEMM.format(256, 0, 1, 4): "489d83eb20b9452db417d055e525219c81cac50d",
    _GEMM.format(256, 1, 0, 0): "9fe731ec3a64cfd6fc3bbaf7089f773a8ecc54c1",
    _GEMM.format(256, 1, 0, 1): "c3e3ec4e782a74c134480b5ac8ece92bc3b19b6f",
    _GEMM.format(256, 1, 0, 2): "edd19ca88e4218facd4364aa933f26e788968566",
    _GEMM.format(256, 1, 0, 3): "5aaf1bb9371ccec808f66041811ea1d26f56cb9d",
    _GEMM.format(256, 1, 0, 4): "7b53773107850b83584cc28a0fcb78ae88026d67",
    _GEMM.format(256, 1, 1, 0): "ba4a85d204a41860671db79eb0bc5da6ab8bce91",
    _GEMM.format(256, 1, 1, 1): "6c8e0baf552a8bbe0369e8007e5627f66cc284e7",
    _GEMM.format(256, 1, 1, 2): "bd0f6459be2e9622b3eb522a745254ee5cdcec00",
    _GEMM.format(256, 1, 1, 3): "6c1a14db827944be0764bf3b9bc7e366df5aa3d1",
    _GEMM.format(256, 1, 1, 4): "d78307de08a1caa7518ca5f2fa0c4c208b25ea9b",
}


def _check_sass(tmp_path, src, recorded):
    from open_muse_b200 import build as b

    nvcc = obj_tools()
    if not all(os.path.exists(os.path.join(os.path.dirname(nvcc), t)) for t in ("cuobjdump", "cu++filt")):
        pytest.skip("cuobjdump / cu++filt not installed next to nvcc")
    if "release 12.9" not in subprocess.run([nvcc, "--version"], capture_output=True, text=True).stdout:
        pytest.skip("the recorded SASS is nvcc 12.9's")
    obj = str(tmp_path / (src + ".o"))
    subprocess.run([nvcc, *b.NVCC_FLAGS, "-c", str(b.CSRC / (src + ".cu")), "-o", obj], check=True)
    got = _demangled_sass(obj)
    for name, sha in recorded.items():
        assert got.get(name) == sha, name
    return got


def test_norm_kernels_compile_to_the_same_sass_as_before_the_e4m3_forms(tmp_path):
    got = _check_sass(tmp_path, "norm", NORM_SASS_SHA1)
    assert "norm_fwd_warp_kernel<float, unsigned char, (int)4, (bool)1>" in got
    assert "glu_norm_fwd_kernel<(int)16, (bool)0, (bool)1, unsigned char>" in got
    assert "norm2_fwd_warp_kernel<(int)4, (bool)1, unsigned char>" in got


def test_gemm_kernels_compile_to_the_same_sass_as_before_the_fp8_residual_epilogue(tmp_path):
    got = _check_sass(tmp_path, "gemm_wgmma", GEMM_SASS_SHA1)
    assert _GEMM.format(128, 0, 0, 6) in got
