"""Gradient checkpointing without a GPU: the product's host code runs with the exact torch restatements of the kernels
(tests/cpu_math_ops.py, with the dropout-aware stand-ins of tests/test_dropout_cpu.py / test_uvit_dropout_cpu.py), once
with ``enable_gradient_checkpointing()`` and once without.  A checkpointed unit keeps only its inputs and re-runs its
forward in its backward, so the loss and every parameter gradient must be EQUAL, not just close -- with dropout too, since
the keep bits follow from the device-side seed and the site ids.  The recompute is observed through the op sequence: every
attention forward runs a second time during the backward, and never without checkpointing."""
import json
import os
import subprocess
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from open_muse_b200 import MaskGitTransformer, MaskGiTUViT_v2, ops
from oracle import ref_snapshot
from tests import test_dropout_cpu as D
from tests import test_uvit_dropout_cpu as UD

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
V1_FIXTURES = ["micro_transformer.pt", "micro_t2i_transformer.pt", "micro_t2i_proj_transformer.pt"]
UVIT_FIXTURES = ["micro_uvit_v2.pt", "micro_uvit_v2_downup.pt"]
UVIT_ARGS = ("input_ids", "encoder_hidden_states", "cond_embeds", "micro_conds")


def _v1_inputs(g):
    if "batch" in g:
        return dict(input_ids=g["batch"]["input_ids"], labels=g["batch"]["labels"], label_smoothing=g.get("label_smoothing", 0.0))
    return dict(input_ids=g["input_ids"], labels=g["labels"], encoder_hidden_states=g["encoder_hidden_states"])


def _uvit_inputs(g):
    return dict(zip(UVIT_ARGS, [g[k] for k in UVIT_ARGS]), labels=g["labels"], label_smoothing=0.1)


def _count_during_backward(m, fwd, name):
    """runs forward + backward; returns (loss, grads, calls of ops.<name> in the forward, in the backward)"""
    calls, phase = {"fwd": 0, "bwd": 0}, ["fwd"]
    fn = getattr(ops, name)

    def wrap(*a, **k):
        calls[phase[0]] += 1
        return fn(*a, **k)

    with pytest.MonkeyPatch.context() as p:
        p.setattr(ops, name, wrap)
        _, loss = m(**fwd)
        phase[0] = "bwd"
        loss.backward()
    return loss.detach(), {n: p.grad.clone() for n, p in m.named_parameters()}, calls["fwd"], calls["bwd"]


def _run(make, fwd, ckpt):
    torch.manual_seed(7)  # the dropout seed is drawn from the default generator
    m = make()
    if ckpt:
        m.enable_gradient_checkpointing()
    return _count_during_backward(m, fwd, "attn_fwd")


def _assert_equal(off, on):
    loss0, g0, f0, b0 = off
    loss1, g1, f1, b1 = on
    assert torch.equal(loss0, loss1)
    assert g0.keys() == g1.keys()
    for n in g0:
        assert torch.equal(g0[n], g1[n]), n
    assert f0 == f1 and f0 > 0
    assert b0 == 0 and b1 == f1  # every attention forward recomputed once in the backward, only with checkpointing


@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("name", V1_FIXTURES)
def test_v1_gradients_are_equal_with_and_without_checkpointing(golden, monkeypatch, name, p):
    g = golden(name)
    D.install(monkeypatch)
    cfg = dict(g["config"], hidden_dropout=p, attention_dropout=p)

    def make():
        m = MaskGitTransformer(**cfg)
        m.load_state_dict(g["state_dict"])
        return m.train()

    fwd = _v1_inputs(g)
    _assert_equal(_run(make, fwd, False), _run(make, fwd, True))


def test_v1_checkpointing_needs_a_backward(golden, monkeypatch):
    """no_grad and eval forwards are the plain forward: nothing is recomputed and the logits do not change"""
    g = golden("micro_t2i_transformer.pt")
    D.install(monkeypatch)
    m = MaskGitTransformer(**g["config"])
    m.load_state_dict(g["state_dict"])
    m.eval()
    fwd = _v1_inputs(g)
    with torch.no_grad():
        ref = m(**fwd)[0]
        m.enable_gradient_checkpointing()
        assert m.is_gradient_checkpointing
        assert torch.equal(m(**fwd)[0], ref)


@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("name", UVIT_FIXTURES)
def test_uvit_gradients_are_equal_with_and_without_checkpointing(golden, monkeypatch, name, p):
    g = golden(name)
    UD.install(monkeypatch)
    monkeypatch.setattr(MaskGiTUViT_v2, "device", property(lambda self: torch.device("cpu")), raising=False)
    cfg = dict(g["config"], hidden_dropout=p, attention_dropout=p)

    def make():
        m = MaskGiTUViT_v2(**cfg)
        m.load_state_dict(g["state_dict"])
        return m.train()

    fwd = _uvit_inputs(g)
    _assert_equal(_run(make, fwd, False), _run(make, fwd, True))


def test_uvit_stage_flags_select_the_recomputed_units(golden, monkeypatch):
    """each flag checkpoints only its own units: the transformer layers (model flag) and each stage's pairs (stage flag);
    every AttentionBlock2D runs two attention forwards, every transformer layer two"""
    g = golden("micro_uvit_v2.pt")
    cfg = g["config"]
    R, L = cfg["num_res_blocks"], cfg["num_hidden_layers"]
    UD.install(monkeypatch)
    fwd = _uvit_inputs(g)
    for which, expect in (("model", 2 * L), ("down", 2 * R), ("up", 2 * R)):
        m = MaskGiTUViT_v2(**cfg)
        m.load_state_dict(g["state_dict"])
        m.train()
        target = {"model": m, "down": m.down_blocks[0], "up": m.up_blocks[0]}[which]
        target.gradient_checkpointing = True
        _, _, f, b = _count_during_backward(m, fwd, "attn_fwd")
        assert f == 2 * (2 * R + L) and b == expect, which


STEPS = ("enable_gradient_checkpointing", "disable_gradient_checkpointing", "enable_gradient_checkpointing")


def _flag_trace(m):
    def flags():
        return [m.gradient_checkpointing, m.down_blocks[0].gradient_checkpointing, m.up_blocks[0].gradient_checkpointing,
                m.is_gradient_checkpointing]

    out = [flags()]
    for step in STEPS:
        getattr(m, step)()
        out.append(flags())
    return out


# in a fresh interpreter: the reference imports its own accelerate stand-in, which other test modules may have replaced
REF_SIDE = r'''
import json, sys
sys.path.insert(0, sys.argv[1])
from oracle.ref_snapshot import import_reference
import_reference()
from muse.modeling_transformer_v2 import MaskGiTUViT_v2
from tests.test_recompute_cpu import _flag_trace
print(json.dumps(_flag_trace(MaskGiTUViT_v2(**json.loads(sys.argv[2])))))
'''


@pytest.mark.skipif(not ref_snapshot.available(), reason="oracle/_ref snapshot of the reference not available")
def test_uvit_enable_disable_set_the_flags_the_reference_sets(golden):
    cfg = golden("micro_uvit_v2.pt")["config"]
    ours = _flag_trace(MaskGiTUViT_v2(**cfg))
    run = subprocess.run([sys.executable, "-c", REF_SIDE, ROOT, json.dumps(cfg)], capture_output=True, text=True,
                         timeout=600, cwd=ROOT)
    assert run.returncode == 0, run.stderr[-2000:]
    ref = json.loads(run.stdout.strip().splitlines()[-1])
    assert ours == ref
    assert ours[1][:3] == [True] * 3 and ours[2][:3] == [False] * 3


# ------------------------------------------------------------------------------------------------ DDP, gloo world 2
def _ddp_worker(rank, world, port, g, batches, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    sys.path.insert(0, ROOT)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(1)
    from open_muse_b200 import MaskGitTransformer
    from tests import cpu_math_ops

    real_bf16 = torch.bfloat16
    cpu_math_ops.install(cpu_math_ops.PlainSetter, exact=True)
    result = {}
    for ckpt in (False, True):
        m = MaskGitTransformer(**dict(g["config"], hidden_dropout=0.0, attention_dropout=0.0))
        m.load_state_dict(g["state_dict"])
        m.train()
        if ckpt:
            m.enable_gradient_checkpointing()
        model = torch.nn.parallel.DistributedDataParallel(m)
        inp, lab = batches[rank]
        _, loss = model(inp, labels=lab)
        loss.backward()
        result[ckpt] = {n: p.grad.clone() for n, p in m.named_parameters()}
    torch.bfloat16 = real_bf16  # the alias of exact mode confuses torch.save's dtype tables
    if rank == 0:
        torch.save(result, out)
    dist.destroy_process_group()


def test_ddp_all_reduced_gradients_are_equal_with_and_without_checkpointing(tmp_path, golden):
    """the per-layer backward still hands its parameter gradients to DDP's bucket hooks one layer at a time; the all-reduced
    gradients of a checkpointed model equal those of the plain one"""
    g = golden("micro_transformer.pt")
    gen = torch.Generator().manual_seed(2)
    batches = []
    for r in range(2):
        ids = g["batch"]["input_ids"][:1 + r].clone()
        lab = g["batch"]["labels"][:1 + r].clone()
        flip = torch.rand(ids.shape, generator=gen) < 0.3
        lab[flip] = -100
        batches.append((ids, lab))
    out = str(tmp_path / "r0.pt")
    mp.spawn(_ddp_worker, args=(2, 35500 + os.getpid() % 2000, g, batches, out), nprocs=2, join=True)
    got = torch.load(out, weights_only=False)
    assert got[False].keys() == got[True].keys()
    for n in got[False]:
        assert torch.equal(got[False][n], got[True][n]), n
