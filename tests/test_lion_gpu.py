"""GPU: FusedLion (Lion + EMA + bf16 operand packing in one pass) against the reference ``Lion`` (training/optimizer.py)
and ``EMAModel`` run by torch on the same GPU; CUDA-graph replays of fused steps with ``model=`` for MaskGitTransformer and
MaskGiTUViT_v2; and U-ViT training with FusedAdamW / FusedLion(model=...) against torch.optim.AdamW / the reference Lion.
CPU twin: tests/test_lion_cpu.py."""
import importlib.util
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import ref_snapshot  # noqa: E402
from open_muse_b200 import EMAModel, FusedAdamW, FusedLion, MaskGitTransformer, MaskGiTUViT_v2  # noqa: E402
from open_muse_b200.graphs import GraphedStep  # noqa: E402
from open_muse_b200.modeling_transformer import _PackedWeights  # noqa: E402

DEV = "cuda"


def _ref(rel, name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ref_snapshot.DEST, rel))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def Lion():
    return _ref("training/optimizer.py", "_ref_training_optimizer").Lion


@pytest.fixture(scope="module")
def RefEMA():
    return _ref("muse/modeling_ema.py", "_ref_muse_modeling_ema").EMAModel


# 112 tensors (three launches of at most 48 entries), among them tensors of 17 and 65 blocks of 1024 elements
NUMELS = [4, 8, 1020, 1024, 1028, 3076, 16388, 65540]
N = 112


def _params(seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return [torch.nn.Parameter(torch.randn(NUMELS[i % len(NUMELS)], generator=g, device=DEV)) for i in range(N)]


def _groups(ps, wd=0.1):
    return [{"params": ps[0::2], "weight_decay": wd}, {"params": ps[1::2], "weight_decay": 0.0}]


def _grads(ps, step):
    g = torch.Generator(device=DEV).manual_seed(1000 + step)
    out = []
    for i, p in enumerate(ps):
        x = torch.randn(p.shape, generator=g, device=DEV) * 1e-3
        x[::97] = 0.0  # exact zeros: u = 0 where m is zero too (first step), sign 0
        out.append(x)
    return out


@pytest.mark.parametrize("tensor_lr", [False, True], ids=["float_lr", "tensor_lr"])
def test_fused_lion_equals_reference_lion_on_the_gpu(Lion, RefEMA, tensor_lr):
    """12 steps over three launches: with a Python-float lr every parameter and every exp_avg equal torch's reference
    Lion bit for bit; with a tensor lr (1 - lr * wd formed in fp32 on the device) exp_avg still equal and the parameters
    within rtol 2e-6; the EMA shadows within test_optim_gpu.py's tolerance of EMAModel.step"""
    ref_ps, ps = _params(0), _params(0)
    kw = dict(betas=(0.9, 0.99))
    ekw = dict(decay=0.999, update_after_step=2, update_every=1, use_ema_warmup=True, inv_gamma=1.0, power=2 / 3)
    ref_opt = Lion(_groups(ref_ps), lr=3e-3, **kw)
    flat = lambda xs: [p for gr in _groups(xs) for p in gr["params"]]  # noqa: E731  (the EMA follows the groups' order)
    ref_ema, ema = RefEMA(flat(ref_ps), **ekw), EMAModel(flat(ps), **ekw)
    lr = torch.tensor([3e-3], device=DEV) if tensor_lr else 3e-3
    opt = FusedLion(_groups(ps), lr=lr, ema=ema, eps=1e-8, **kw)
    assert sum(len(pl["params"]) for pl in opt.param_groups) > 2 * 48
    for step in range(12):
        for a, b, gr in zip(ref_ps, ps, _grads(ref_ps, step)):
            a.grad, b.grad = gr, gr.clone()
        ref_opt.step(); ref_ema.step(flat(ref_ps))
        opt.step()
        for i, (a, b) in enumerate(zip(ref_ps, ps)):
            where = f"step {step} tensor {i} ({a.numel()} elements)"
            assert torch.equal(opt.state[b]["exp_avg"], ref_opt.state[a]["exp_avg"]), f"exp_avg differs at {where}"
            if tensor_lr:
                torch.testing.assert_close(b, a, rtol=2e-6, atol=1e-8, msg=lambda m_: f"{where}: {m_}")
            else:
                assert torch.equal(b, a), f"p differs at {where}: {(b - a).abs().max().item():.3e}"
        for i, (sa, sb) in enumerate(zip(ref_ema.shadow_params, ema.shadow_params)):
            torch.testing.assert_close(sb, sa, rtol=2e-6, atol=1e-8, msg=lambda m_: f"step {step} shadow {i}: {m_}")
            sb.copy_(sa)  # each step's EMA checked on its own, not its accumulated rounding
        if tensor_lr:
            with torch.no_grad():
                for a, b in zip(ref_ps, ps):
                    b.copy_(a)
    assert int(opt.state_dict()["state"][0]["step"]) == 12


def _tensors(W, prefix=""):
    out = {}
    for k, v in (W.items() if isinstance(W, dict) else enumerate(W)):
        if torch.is_tensor(v):
            out[prefix + str(k)] = v
        elif isinstance(v, (dict, list)):
            out.update(_tensors(v, f"{prefix}{k}."))
    return out


def _uvit(g):
    m = MaskGiTUViT_v2(**g["config"])
    m.load_state_dict(g["state_dict"])
    return m.to(DEV).train()


UVIT_ARGS = ("input_ids", "encoder_hidden_states", "cond_embeds", "micro_conds")


@pytest.mark.parametrize("opt_cls", [FusedAdamW, FusedLion])
@pytest.mark.parametrize("kind", ["v1", "uvit"])
def test_graph_replays_advance_step_weights_and_operands(golden, kind, opt_cls):
    """GraphedStep of forward + backward + fused step with model=: each replay advances the device step counter and the
    weights, and the operands the next forward reads equal a cache rebuilt from scratch"""
    if kind == "v1":
        g = golden("micro_transformer.pt")
        m = MaskGitTransformer(**g["config"])
        m.load_state_dict(g["state_dict"])
        m.to(DEV).train()
        inputs = (g["batch"]["input_ids"].to(DEV), g["batch"]["labels"].to(DEV))

        def fwd(i, l):
            return m(i, labels=l)[1]

        operands = lambda: {"flat": m._packed.flat}  # noqa: E731
        fresh = lambda: {"flat": _PackedWeights(m).refresh().flat}  # noqa: E731
        probe = m.transformer_layers[0].ffn.wo.weight
    else:
        g = golden("micro_uvit_v2.pt")
        m = _uvit(g)
        inputs = tuple(g[k].to(DEV) for k in UVIT_ARGS) + (g["labels"].to(DEV),)

        def fwd(*a):
            return m(*a[:4], labels=a[4])[1]

        operands = lambda: _tensors(m._cache)  # noqa: E731
        fresh = lambda: _tensors(m._build_weights()[0])  # noqa: E731
        probe = m.transformer_layers[0].ffn.wo.weight
    opt = opt_cls(m.parameters(), lr=1e-3, model=m)

    def step(*a):
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = fwd(*a)
        loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
        return loss.detach()

    gs = GraphedStep(step, inputs, warmup=2)
    before = int(opt._plans[0]["step"])
    w0 = probe.detach().clone()
    losses = [float(gs(*inputs)) for _ in range(3)]
    torch.cuda.synchronize()
    assert int(opt._plans[0]["step"]) == before + 3
    assert not torch.equal(w0, probe) and losses[-1] < losses[0], losses
    got, want = operands(), fresh()
    assert got.keys() == want.keys()
    stale = [k for k in want if not torch.equal(got[k], want[k])]
    assert stale == [], f"operands not current after graph replays: {stale}"


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-30))


@pytest.mark.parametrize("which", ["adamw", "lion"])
def test_uvit_training_with_fused_optimizer_and_model_matches_torch(golden, Lion, which):
    """a few U-ViT train steps: FusedAdamW / FusedLion(model=uvit) against torch.optim.AdamW / the reference Lion on an
    identical model whose operand cache is rebuilt after every step: each step's loss within the U-ViT loss tolerance (2e-3)
    and each parameter's update within its gradient tolerance (rel-L2 8e-2); the loss falls, and the cache the fused steps
    kept equals a rebuilt one"""
    g = golden("micro_uvit_v2.pt")
    a, b = _uvit(g), _uvit(g)
    args = [g[k].to(DEV) for k in UVIT_ARGS]
    labels = g["labels"].to(DEV)
    if which == "adamw":
        ref_opt, opt = torch.optim.AdamW(a.parameters(), lr=2e-3), FusedAdamW(b.parameters(), lr=2e-3, model=b)
    else:
        ref_opt = Lion(a.parameters(), lr=3e-4, weight_decay=0.01)
        opt = FusedLion(b.parameters(), lr=3e-4, weight_decay=0.01, model=b)
    losses = []
    for step in range(5):
        ls = []
        for m in (a, b):
            with torch.autocast("cuda", dtype=torch.bfloat16):
                _, loss = m(*args, labels=labels)
            loss.backward()
            ls.append(float(loss))
        assert abs(ls[1] - ls[0]) / ls[0] < 2e-3, (step, ls)
        losses.append(ls[1])
        p0 = [p.detach().clone() for p in a.parameters()]
        ref_opt.step(); opt.step()
        ref_opt.zero_grad(set_to_none=True); opt.zero_grad(set_to_none=True)
        for (n, pa), pb, q in zip(a.named_parameters(), b.parameters(), p0):
            if not torch.equal(pa, q):
                assert _rel(pb - q, pa - q) < 8e-2, (step, n, _rel(pb - q, pa - q))
    assert losses[-1] < losses[0], losses
    got, want = _tensors(b._weights()), _tensors(b._build_weights()[0])
    assert all(torch.equal(got[k], want[k]) for k in want)
