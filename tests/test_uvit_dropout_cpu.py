"""Dropout of MaskGiTUViT_v2 (hidden_dropout / attention_dropout in training mode) without a GPU.

The product's host code runs in exact mode (tests/cpu_math_ops.py) with the dropout-aware stand-ins of
tests/test_dropout_cpu.py plus GRN stand-ins that draw the ResBlock's masks from the same restatement of the generator.
It is compared with the UNMODIFIED reference whose nn.Dropout modules -- ResBlock.channelwise[3], every Attention.dropout
and GLUFeedForward.dropout -- are replaced by modules that apply the recorded masks."""
import sys

import pytest
import torch

from open_muse_b200 import MaskGiTUViT_v2, ops
from tests import cpu_math_ops
from tests import test_dropout_cpu as D
from tests.test_dropout_cpu import _Replay, _op_trace, _rel, keep_scale, unpack_bits

ARGS = ("input_ids", "encoder_hidden_states", "cond_embeds", "micro_conds")


# ------------------------------------------------------------------------------------------- dropout-aware stand-ins
def _grn(x, gamma, beta, B, HW, save_stats=False, dropout=None):
    if dropout is None:
        return cpu_math_ops.grn(x, gamma, beta, B, HW, save_stats)
    out, sumsq, nx = cpu_math_ops._grn(x, gamma, beta, B, HW)
    out, bits = D._dropout_fwd(out.contiguous(), *dropout)  # the fp32 GRN output is dropped, then rounded once
    return out.to(x.dtype), torch.stack([sumsq, nx]), bits


def _grn_bwd(x, dout, stats, gamma, dgamma, dbeta, B, HW, dropout=None):
    if dropout is not None:
        dout = D._dropout_bwd(dout.float(), dropout[1], dropout[0])
    return cpu_math_ops.grn_bwd(x, dout, stats, gamma, dgamma, dbeta, B, HW)


def install(mp):
    D.install(mp)
    mp.setattr(ops, "grn", _grn)
    mp.setattr(ops, "grn_bwd", _grn_bwd)


# --------------------------------------------------------------------------------------------------------- helpers
def _model(g, mp, p_hidden, p_attn, train=True):
    install(mp)
    m = MaskGiTUViT_v2(**dict(g["config"], hidden_dropout=p_hidden, attention_dropout=p_attn))
    m.load_state_dict(g["state_dict"])
    mp.setattr(MaskGiTUViT_v2, "device", property(lambda self: torch.device("cpu")), raising=False)
    return m.train(train)


def expected_sites(cfg, p_hidden, p_attn):
    """unit j = down pairs, layers, up pairs; site 3 j + kind (pair: ResBlock, attention, crossattention; layer:
    attention, crossattention, FFN); a rate of 0 leaves its sites out"""
    R, L = cfg["num_res_blocks"], cfg["num_hidden_layers"]
    out = []
    for j in range(2 * R + L):
        layer = R <= j < R + L
        rates = (p_attn, p_attn, p_hidden) if layer else (p_hidden, p_attn, p_attn)
        out += [3 * j + k for k, p in enumerate(rates) if p > 0]
    return out


def _columns(cfg, S, Skv):
    """site -> number of mask columns (the rows follow from the masked tensor's shape)"""
    R, L = cfg["num_res_blocks"], cfg["num_hidden_layers"]
    C4 = 4 * cfg["block_out_channels"][0]
    S_in = S // 4 if cfg.get("force_down_up_sample") else S
    cols = {}
    for j in range(2 * R + L):
        layer = R <= j < R + L
        for k, n in enumerate((S_in, Skv, cfg["intermediate_size"]) if layer else (C4, Skv, Skv)):
            cols[3 * j + k] = n
    return cols


def _replayed_reference(cfg, sd, masks, S, Skv, p_hidden, p_attn, device="cpu"):
    """the unmodified reference in fp32 and training mode on ``device``, every nn.Dropout of an active site replaced by
    its recorded mask (masks: site -> bits on the CPU)"""
    from oracle.ref_snapshot import import_reference

    # a test that ran a training script earlier in the session can leave a stand-in ``accelerate`` module behind without
    # its ``accelerate.utils`` entry, which the reference imports: let import_reference install its own pair again
    if "accelerate" in sys.modules and "accelerate.utils" not in sys.modules:
        del sys.modules["accelerate"]
    ref = import_reference().MaskGiTUViT(**cfg)  # the reference's alias of MaskGiTUViT_v2
    ref.load_state_dict(sd)
    ref.to(device).train()
    cols = _columns(cfg, S, Skv)
    R, L = cfg["num_res_blocks"], cfg["num_hidden_layers"]

    def put(obj, attr, site, p):
        if site in masks:
            setattr(obj, attr, _Replay(unpack_bits(masks[site], cols[site]).to(device), keep_scale(p)))

    stages = [(ref.down_blocks[0], 0), (ref.up_blocks[0], R + L)]
    for stage, j0 in stages:
        for i, (rb, ab) in enumerate(zip(stage.res_blocks, stage.attention_blocks)):
            j = j0 + i
            assert isinstance(rb.channelwise[3], torch.nn.Dropout)
            put(rb.channelwise, "3", 3 * j, p_hidden)
            put(ab.attention, "dropout", 3 * j + 1, p_attn)
            put(ab.crossattention, "dropout", 3 * j + 2, p_attn)
    for i, layer in enumerate(ref.transformer_layers):
        j = R + i
        put(layer.attention, "dropout", 3 * j, p_attn)
        put(layer.crossattention, "dropout", 3 * j + 1, p_attn)
        put(layer.ffn, "dropout", 3 * j + 2, p_hidden)
    return ref


def _kept(masks, cols):
    k = torch.cat([unpack_bits(b, cols[s]).flatten() for s, b in masks.items()])
    return float(k.float().mean())


# --------------------------------------------------------------------------------------------------------- tests
CASES = [("micro_uvit_v2.pt", False), ("micro_uvit_v2.pt", True), ("micro_uvit_v2_downup.pt", False)]


@pytest.mark.parametrize("name,weighted", CASES)
def test_training_with_dropout_reproduces_the_reference_given_the_same_masks(golden, name, weighted):
    g = golden(name)
    kw = dict(labels=g["labels"], label_smoothing=0.1)
    if weighted:
        kw["loss_weight"] = g["loss_weight"]
    with pytest.MonkeyPatch.context() as mp:
        m = _model(g, mp, 0.1, 0.1)
        torch.manual_seed(3)
        with ops.dropout_record() as log:
            logits, loss = m(*[g[k] for k in ARGS], **kw)
        loss.backward()
        grads = {n: p.grad.clone() for n, p in m.named_parameters()}
    cfg = dict(g["config"], hidden_dropout=0.1, attention_dropout=0.1)
    assert [s for s, _ in log] == expected_sites(cfg, 0.1, 0.1) == list(range(3 * (2 * cfg["num_res_blocks"] +
                                                                                 cfg["num_hidden_layers"])))
    masks = dict(log)
    B, S = g["input_ids"].shape
    Skv = g["encoder_hidden_states"].shape[1]
    assert 0.75 < _kept(masks, _columns(cfg, S, Skv)) < 0.97  # the masks are not trivially all-kept or all-dropped

    ref = _replayed_reference(cfg, g["state_dict"], masks, S, Skv, 0.1, 0.1)
    r_logits, r_loss = ref(*[g[k] for k in ARGS], **kw)
    r_loss.backward()
    assert _rel(logits, r_logits) < 5e-5
    assert abs(float(loss.detach()) - float(r_loss.detach())) < 1e-5 * abs(float(r_loss.detach()))
    for n, p in ref.named_parameters():
        assert _rel(grads[n], p.grad) < 5e-4, (n, _rel(grads[n], p.grad))
    with torch.no_grad():  # and the masks did something: without them the reference computes other logits
        ref.eval()
        assert _rel(logits, ref(*[g[k] for k in ARGS])) > 1e-3


@pytest.mark.parametrize("p_hidden,p_attn", [(0.1, 0.0), (0.0, 0.1)])
def test_each_rate_gates_only_its_own_sites(golden, p_hidden, p_attn):
    g = golden("micro_uvit_v2.pt")
    with pytest.MonkeyPatch.context() as mp:
        m = _model(g, mp, p_hidden, p_attn)
        torch.manual_seed(5)
        with ops.dropout_record() as log:
            logits, loss = m(*[g[k] for k in ARGS], labels=g["labels"])
        loss.backward()
        grads = {n: p.grad.clone() for n, p in m.named_parameters()}
    cfg = dict(g["config"], hidden_dropout=p_hidden, attention_dropout=p_attn)
    sites = [s for s, _ in log]
    assert sites == expected_sites(cfg, p_hidden, p_attn) == ([0, 5, 8, 9] if p_attn == 0 else [1, 2, 3, 4, 6, 7, 10, 11])
    B, S = g["input_ids"].shape
    Skv = g["encoder_hidden_states"].shape[1]
    ref = _replayed_reference(cfg, g["state_dict"], dict(log), S, Skv, p_hidden, p_attn)
    r_logits, r_loss = ref(*[g[k] for k in ARGS], labels=g["labels"])
    r_loss.backward()
    assert _rel(logits, r_logits) < 5e-5
    for n, p in ref.named_parameters():
        assert _rel(grads[n], p.grad) < 5e-4, (n, _rel(grads[n], p.grad))


def test_training_mode_forward_under_no_grad_applies_the_masks(golden):
    """model.train() + torch.no_grad(): nn.Dropout is active in the reference, so the inference path drops too"""
    g = golden("micro_uvit_v2_downup.pt")
    args = [g[k] for k in ARGS]
    with pytest.MonkeyPatch.context() as mp:
        m = _model(g, mp, 0.1, 0.1)
        torch.manual_seed(7)
        with torch.no_grad(), ops.dropout_record() as log:
            logits, loss = m(*args, labels=g["labels"], label_smoothing=0.1)
        torch.manual_seed(7)  # the same seed through the autograd path: the same masks and logits
        with ops.dropout_record() as log2:
            logits2, _ = m(*args, labels=g["labels"], label_smoothing=0.1)
    cfg = dict(g["config"], hidden_dropout=0.1, attention_dropout=0.1)
    assert [s for s, _ in log] == expected_sites(cfg, 0.1, 0.1)
    assert all(torch.equal(a, b) for (_, a), (_, b) in zip(log, log2))
    assert _rel(logits, logits2) < 1e-6
    B, S = g["input_ids"].shape
    Skv = g["encoder_hidden_states"].shape[1]
    ref = _replayed_reference(cfg, g["state_dict"], dict(log), S, Skv, 0.1, 0.1)
    with torch.no_grad():
        r_logits, r_loss = ref(*args, labels=g["labels"], label_smoothing=0.1)
        assert _rel(logits, r_logits) < 5e-5
        assert abs(float(loss) - float(r_loss)) < 1e-5 * abs(float(r_loss))
        ref.eval()
        assert _rel(logits, ref(*args)) > 1e-3


def _fwd(g):
    return dict(**{k: g[k] for k in ARGS}, labels=g["labels"], label_smoothing=0.1)


@pytest.mark.parametrize("name", ["micro_uvit_v2.pt", "micro_uvit_v2_downup.pt"])
def test_inactive_dropout_leaves_the_op_sequence_alone(golden, name):
    """rate 0.0 in training mode and rate 0.1 in eval mode pass no dropout keyword: the same op calls, with the same
    keywords, as a model whose rates are 0.0, through the autograd path (forward and backward) and under no_grad"""
    g = golden(name)
    traces = {}
    for tag, p, train in (("zero-train", 0.0, True), ("drop-eval", 0.1, False), ("zero-eval", 0.0, False)):
        for grad in (True, False):
            with pytest.MonkeyPatch.context() as mp:
                m = _model(g, mp, p, p, train)
                with torch.set_grad_enabled(grad):
                    traces[tag, grad] = _op_trace(mp, m, _fwd(g), backward=grad)
    for calls in traces.values():
        assert not any("dropout" in n or "dropout" in k for n, k in calls)
    for grad in (True, False):
        assert traces["drop-eval", grad] == traces["zero-eval", grad] == traces["zero-train", grad]
    with pytest.MonkeyPatch.context() as mp:
        m = _model(g, mp, 0.1, 0.1)
        drop_train = _op_trace(mp, m, _fwd(g), backward=True)
    # with dropout on, the only difference is the dropout keyword of the ops that apply or undo a mask
    strip = [(n, tuple(x for x in k if x != "dropout")) for n, k in drop_train]
    assert strip == traces["zero-train", True]
    with_kw = {n for n, k in drop_train if "dropout" in k}
    assert with_kw == {"grn", "grn_bwd", "attn_fwd", "attn_bwd", "glu_fwd", "glu_bwd"}


def test_generate2_in_training_mode_with_dropout_raises(golden, monkeypatch):
    g = golden("micro_uvit_v2.pt")
    m = _model(g, monkeypatch, 0.1, 0.0)
    with pytest.raises(RuntimeError, match="eval"):
        m.generate2(encoder_hidden_states=g["encoder_hidden_states"], cond_embeds=g["cond_embeds"],
                    micro_conds=g["micro_conds"][:1], empty_embeds=g["empty_embeds"],
                    empty_cond_embeds=g["empty_cond_embeds"], timesteps=2, use_cuda_graph=False)
