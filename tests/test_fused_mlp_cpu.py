"""``MaskGiTUViT_v2(use_fused_mlp=True)`` -- FusedGeLUFeedForward, wo(gelu_tanh(wi_0(x))) -- without a GPU.

The product's host code runs on the kernels' torch restatements (tests/cpu_math_ops.py, exact-fp32 mode) plus the two
restatements of the new tanh-GELU pass below, and is compared with tests/golden/micro_uvit_v2_fused_mlp.pt, which the
UNMODIFIED reference wrote through the stand-in of make_golden_fused_mlp.fused_mlp_standin (flash_attn's heuristic=-1
branch).  The fixture keeps signatures rather than tensors (make_golden_fused_mlp.py): the weights are rebuilt from its
seeds, and each gradient is compared through its norm and four seeded projections.
Also: checkpoints in both directions, dropout (the reference never applies FusedGeLUFeedForward.dropout), the FP8
producer routing, and that the GLU kernels compiled to the same SASS as before they were templated."""
import os
import re
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from open_muse_b200 import MaskGiTUViT_v2, ops
from oracle import ref_snapshot
from tests import cpu_math_ops
from tests import test_fp8_cpu as FP8
from tests import test_uvit_dropout_cpu as UD
from tests.golden import make_golden_fused_mlp as GF
from tests.golden.make_golden_fused_mlp import fused_mlp_standin

ARGS = ("input_ids", "encoder_hidden_states", "cond_embeds", "micro_conds")
FIXTURE = "micro_uvit_v2_fused_mlp.pt"
needs_ref = pytest.mark.skipif(not ref_snapshot.available(), reason="oracle/_ref snapshot of the reference not available")


# ------------------------------------------------------------------------------ restatements of muse_gelu_tanh_fwd/bwd
def gelu_tanh_fwd(pre, out_dtype=None):
    assert out_dtype is None
    return F.gelu(pre.float(), approximate="tanh").to(cpu_math_ops._bf())


def gelu_tanh_bwd(pre, dout):
    x = pre.detach().float().requires_grad_(True)
    with torch.enable_grad():
        y = F.gelu(x, approximate="tanh")
    return torch.autograd.grad(y, x, dout.float())[0].to(pre.dtype)


def install(mp, dropout=False):
    (UD.install if dropout else lambda m: cpu_math_ops.install(m, exact=True))(mp)
    mp.setattr(ops, "gelu_tanh_fwd", gelu_tanh_fwd)
    mp.setattr(ops, "gelu_tanh_bwd", gelu_tanh_bwd)


def _rel(a, b):
    a, b = a.detach().float(), b.detach().float()
    return float((a - b).norm() / b.norm().clamp_min(1e-20))


def _state_dict():
    """the fixture's weights, rebuilt from its seeds (test_seeded_construction_matches_the_reference pins them)"""
    return {k: x.detach().clone() for k, x in GF.seeded_model(MaskGiTUViT_v2)[0].state_dict().items()}


def _model(g, mp, train, **over):
    m = MaskGiTUViT_v2(**dict(g["config"], **over))
    m.load_state_dict(_state_dict())
    mp.setattr(MaskGiTUViT_v2, "device", property(lambda self: torch.device("cpu")), raising=False)
    return m.train(train)


# ------------------------------------------------------------------------------------------------------------- tests
def test_seeded_construction_matches_the_reference(golden):
    """the seeded initial weights and the re-drawn ones equal the reference's, tensor by tensor (fp64 sum and norm)"""
    g = golden(FIXTURE)
    m, init_sig, redrawn, _ = GF.seeded_model(MaskGiTUViT_v2)
    sd = m.state_dict()
    assert list(sd) == list(g["state_signature"]) == list(init_sig) == list(g["init_signature"])
    assert not any("wi_1" in k for k in sd)
    assert redrawn == g["redrawn"]
    for k, x in sd.items():
        assert init_sig[k] == g["init_signature"][k], k
        assert GF.tensor_signature(x) == g["state_signature"][k], k
    assert type(m.transformer_layers[0].ffn).__name__ == "FusedGeLUFeedForward"
    assert [n for n, _ in m.transformer_layers[0].ffn.named_children()] == [
        "pre_mlp_layer_norm", "adaLN_modulation", "wi_0", "dropout", "wo"]
    with pytest.raises(NotImplementedError, match="use_bias"):
        MaskGiTUViT_v2(**dict(g["config"], use_bias=True))


@pytest.mark.parametrize("weighted", [False, True])
def test_training_forward_backward_reproduces_the_reference(golden, monkeypatch, weighted):
    g = golden(FIXTURE)
    install(monkeypatch)
    m = _model(g, monkeypatch, train=True)
    kw = dict(loss_weight=g["loss_weight"]) if weighted else dict(label_smoothing=0.1)
    logits, loss = m(*[g[k] for k in ARGS], labels=g["labels"], **kw)
    loss.backward()
    want_loss, want_grads = (g["loss_weighted"], g["grads_weighted"]) if weighted else (g["loss"], g["grads"])
    if not weighted:
        assert _rel(logits, g["logits"]) < 5e-5
    assert abs(float(loss.detach()) - float(want_loss)) < 1e-5 * abs(float(want_loss))
    names = [n for n, _ in m.named_parameters()]
    assert names == list(want_grads)
    for n, p in m.named_parameters():
        assert p.grad is not None
        e = GF.signature_error(p.grad, want_grads[n])
        assert e < 5e-4, (n, e)


def test_inference_forward_and_generate2_reproduce_the_reference(golden, monkeypatch):
    g = golden(FIXTURE)
    install(monkeypatch)
    m = _model(g, monkeypatch, train=False)
    with torch.no_grad():
        logits, loss = m(*[g[k] for k in ARGS], labels=g["labels"], label_smoothing=0.1)
        assert _rel(logits, g["logits"]) < 5e-5
        assert abs(float(loss) - float(g["loss"])) < 1e-5 * abs(float(g["loss"]))
        ids = m.generate2(encoder_hidden_states=g["encoder_hidden_states"], cond_embeds=g["cond_embeds"],
                          micro_conds=g["micro_conds"][:1], empty_embeds=g["empty_embeds"],
                          empty_cond_embeds=g["empty_cond_embeds"], timesteps=4, temperature=(2.0, 0.0), guidance_scale=3.0,
                          generator=torch.Generator().manual_seed(g["gen_seed"]), seq_len=16, use_cuda_graph=False)
    assert torch.equal(ids, g["gen_ids"])


def _reference():
    # see tests/test_uvit_dropout_cpu.py::_replayed_reference for why a partial ``accelerate`` stand-in is dropped first
    if "accelerate" in sys.modules and "accelerate.utils" not in sys.modules:
        del sys.modules["accelerate"]
    muse = ref_snapshot.import_reference()
    import muse.modeling_transformer_v2  # noqa: F401  (the module fused_mlp_standin patches)

    return muse


@needs_ref
def test_checkpoints_cross_to_the_reference_and_back(golden, tmp_path):
    g = golden(FIXTURE)
    muse = _reference()
    sd = _state_dict()
    m = MaskGiTUViT_v2(**g["config"])
    m.load_state_dict(sd)
    m.save_pretrained(tmp_path / "ours")
    with fused_mlp_standin():
        r = muse.modeling_transformer_v2.MaskGiTUViT_v2.from_pretrained(tmp_path / "ours", low_cpu_mem_usage=False)
        assert r.config.use_fused_mlp and list(r.state_dict()) == list(sd)
        for k, x in r.state_dict().items():
            assert torch.equal(x, sd[k]), k
        with torch.no_grad():  # the loaded reference computes the fixture's logits
            assert _rel(r.eval()(*[g[k] for k in ARGS]), g["logits"]) < 1e-6
        r.save_pretrained(tmp_path / "theirs")
    back = MaskGiTUViT_v2.from_pretrained(tmp_path / "theirs")
    assert back.config.use_fused_mlp and list(back.state_dict()) == list(sd)
    for k, x in back.state_dict().items():
        assert torch.equal(x, sd[k]), k


@needs_ref
def test_dropout_draws_no_ffn_site_and_matches_the_reference_given_the_same_masks(golden):
    g = golden(FIXTURE)
    cfg = dict(g["config"], hidden_dropout=0.1, attention_dropout=0.1)
    with pytest.MonkeyPatch.context() as mp:
        install(mp, dropout=True)
        m = _model(g, mp, train=True, hidden_dropout=0.1, attention_dropout=0.1)
        torch.manual_seed(3)
        with ops.dropout_record() as log:
            logits, loss = m(*[g[k] for k in ARGS], labels=g["labels"], label_smoothing=0.1)
        loss.backward()
        grads = {n: p.grad.clone() for n, p in m.named_parameters()}
    R, L = cfg["num_res_blocks"], cfg["num_hidden_layers"]
    ffn_sites = {3 * (R + i) + 2 for i in range(L)}
    sites = [s for s, _ in log]
    assert sites == [s for s in UD.expected_sites(cfg, 0.1, 0.1) if s not in ffn_sites]  # numbering unchanged
    B, S = g["input_ids"].shape
    Skv = g["encoder_hidden_states"].shape[1]
    _reference()
    with fused_mlp_standin():
        ref = UD._replayed_reference(cfg, _state_dict(), dict(log), S, Skv, 0.1, 0.1)
        r_logits, r_loss = ref(*[g[k] for k in ARGS], labels=g["labels"], label_smoothing=0.1)
        r_loss.backward()
    assert _rel(logits, r_logits) < 5e-5
    assert abs(float(loss.detach()) - float(r_loss.detach())) < 1e-5 * abs(float(r_loss.detach()))
    for n, p in ref.named_parameters():
        assert _rel(grads[n], p.grad) < 5e-4, (n, _rel(grads[n], p.grad))
    assert _rel(logits, g["logits"]) > 1e-3  # the ResBlock and attention masks did act


def test_fp8_mode_feeds_wo_from_the_gelu_pass(golden, monkeypatch):
    g = golden(FIXTURE)
    log = []
    FP8.install(monkeypatch, log)

    def f8_gelu(pre, out_dtype=None):
        if out_dtype == ops.FP8:
            log.append(("gelu_tanh_fwd", True, None))
            return FP8.quant(gelu_tanh_fwd(pre))
        log.append(("gelu_tanh_fwd", False, None))
        return gelu_tanh_fwd(pre)

    monkeypatch.setattr(ops, "gelu_tanh_fwd", f8_gelu)
    m = _model(g, monkeypatch, train=False)
    args = [g[k] for k in ARGS]
    with torch.no_grad():
        ref = m(*args)
        log.clear()
        out = m.set_gemm_precision("fp8")(*args)
    sites = FP8._fp8_sites(m)
    W = m._weights()
    assert all(w["wi"].shape[0] == g["config"]["intermediate_size"] for w in W["layers"])  # wi_0 alone, no gate
    used = [sites[w] for op, f8, w in log if op == "linear_fwd" and f8]
    assert sorted(used) == sorted(sites.values())
    producers = sorted(op for op, f8, _ in log if f8 and op != "linear_fwd")
    L, R = len(m.transformer_layers), len(m.down_blocks[0].res_blocks) * 2
    assert producers == sorted(["add_norm_mod"] * (3 * L + 2 * R) + ["gelu_tanh_fwd"] * L + ["dwconv3x3_norm"] * R)
    assert not any(op == "glu_fwd" for op, _, _ in log)
    rel = float((out - ref).norm() / ref.norm())
    assert 0 < rel < 0.1, rel
    m.train()
    with pytest.raises(RuntimeError, match="inference only"):
        m(*args, labels=g["labels"])


# ---------------------------------------------------------------------------------- SASS of the templated GLU kernels
# sha1 of each GLU kernel's instruction list (cuobjdump -sass, addresses and encodings stripped) as nvcc 12.9 built
# csrc/elementwise.cu with build.NVCC_FLAGS before the GLU and tanh-GELU passes became one template: the GLU
# instantiations of the template must still compile to exactly these instructions.
GLU_SASS_SHA1 = {
    "ffn_act_fwd_kernel<(bool)1, (bool)0>": "d54793eec9e210049724e97797e4596f16b86252",
    "ffn_act_fwd_kernel<(bool)1, (bool)1>": "92c4130669af58b69254944914a2c5da9919d83d",
    "ffn_act_bwd_kernel<(bool)1, (bool)0>": "36eb48a726173bd4e1e5a146a22b0054d8fe5d82",
    "ffn_act_bwd_kernel<(bool)1, (bool)1>": "38fb3d53a5a25cc9dfc62066229d7d24d48b5e21",
    **{f"ffn_act_fwd_e4m3_kernel<(bool)1, (int){ch}>": sha for ch, sha in (
        (1, "1e6e46026ced40722de8db52fb25b7aee7303f13"),
        (2, "98ac7846dafa59dddce30aae477c7f947ac0028c"),
        (4, "33e0fda2efa6c89efa9b8670a02e4f69c27d86e5"),
        (8, "ec1c4500c512c88caf49051be294ff446723e25d"),
        (12, "68a50f8952fa54860024a73c0e52f44d5f7f6688"),
        (16, "191c9f25a03e9724f80997ea2c1f2c8e7488eece"))},
}


def obj_tools():
    """nvcc's path; cuobjdump and cu++filt sit next to it"""
    from open_muse_b200 import build as b

    return b._nvcc()


def _demangled_sass(obj):
    """kernel name (demangled, namespaces dropped) -> sha1 of its instruction list"""
    import hashlib

    bindir = os.path.dirname(obj_tools())
    text = subprocess.run([os.path.join(bindir, "cuobjdump"), "-sass", obj], capture_output=True, text=True, check=True).stdout
    out, name, ins = {}, None, []
    for line in text.splitlines() + ["Function : <end>"]:
        m = re.search(r"Function : (\S+)", line)
        if m:
            if name is not None:
                out[name] = hashlib.sha1("\n".join(ins).encode()).hexdigest()
            name, ins = m.group(1), []
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s*(.*?)\s*;?\s*/\*", line)
        if m and name is not None:
            ins.append(m.group(1))
    names = subprocess.run([os.path.join(bindir, "cu++filt")], input="\n".join(out), capture_output=True, text=True, check=True).stdout.split("\n")
    short = [re.sub(r"^.*::(\w+<.*?>)\(const .*$", r"\1", n) for n in names]
    return {s: out[k] for s, k in zip(short, out)}


def test_glu_kernels_compile_to_the_same_sass_as_before_the_templating(tmp_path):
    from open_muse_b200 import build as b

    nvcc = obj_tools()
    if not all(os.path.exists(os.path.join(os.path.dirname(nvcc), t)) for t in ("cuobjdump", "cu++filt")):
        pytest.skip("cuobjdump / cu++filt not installed next to nvcc")
    if "release 12.9" not in subprocess.run([nvcc, "--version"], capture_output=True, text=True).stdout:
        pytest.skip("the recorded SASS is nvcc 12.9's")
    obj = str(tmp_path / "elementwise.o")
    subprocess.run([nvcc, *b.NVCC_FLAGS, "-c", str(b.CSRC / "elementwise.cu"), "-o", obj], check=True)
    got = _demangled_sass(obj)
    for name, sha in GLU_SASS_SHA1.items():
        assert got.get(name) == sha, name
    assert "ffn_act_fwd_kernel<(bool)0, (bool)0>" in got and "ffn_act_bwd_kernel<(bool)0, (bool)0>" in got
