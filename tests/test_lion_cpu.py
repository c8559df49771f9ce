"""FusedLion WITHOUT a GPU, and the operand-cache coherence of both fused optimizers.

``muse_lion_ema_step`` (csrc/optim.cu) is restated here in torch, dereferencing the same host table of {p, g, m, -, ema,
packed, numel, -} rows, the device-resident step counter and the fp32 scalars the C ABI receives; ``ops._call`` is routed to
it (and ``muse_adamw_ema_step`` to tests/cpu_math_ops.py).  Against it: the unmodified reference ``Lion``
(training/optimizer.py) and ``EMAModel`` (muse/modeling_ema.py) from the oracle snapshot.  Then a numpy emulation of the
kernel's chunking and block search is accepted by the checks and four mutants are rejected, and after every step of either
fused optimizer, with or without ``model=``, each bf16 / fp32 operand of MaskGitTransformer and MaskGiTUViT_v2 equals a
cache rebuilt from scratch.  GPU twin: tests/test_lion_gpu.py."""
import copy
import ctypes
import importlib.util
import os

import numpy as np
import pytest
import torch

from oracle import ref_snapshot
from open_muse_b200 import EMAModel, FusedAdamW, FusedLion, MaskGitTransformer, MaskGiTUViT_v2, ops
from open_muse_b200.modeling_transformer import _PackedWeights
from tests import cpu_math_ops
from tests.local_error import BOUNDS, check_ulps, ema_ref, f32

F32 = torch.float32
needs_ref = pytest.mark.skipif(not ref_snapshot.available(), reason="oracle/_ref snapshot of the reference not available")


def _ref(rel, name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ref_snapshot.DEST, rel))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _ref_lion():
    return _ref("training/optimizer.py", "_ref_training_optimizer").Lion


def _ref_ema():
    return _ref("muse/modeling_ema.py", "_ref_muse_modeling_ema").EMAModel


# ------------------------------------------------------------------------------------------------ the kernel, restated
def lion_ema_step(entries_host, n_entries, scal_ptr, step_ptr, lr_dev_ptr, lr_host, wd_scale, beta1, beta2, one_minus_beta1,
                  one_minus_beta2, weight_decay, ema_enabled, ema_decay, ema_min_decay, ema_update_after_step,
                  ema_update_every, ema_use_warmup, ema_inv_gamma, ema_power, stream):
    """csrc/optim.cu's Lion pass: every float argument rounded to fp32 as the C ABI does, then per element p *= c_wd;
    u = m * beta1 + g * (1 - beta1); p -= lr * sign(u); m = m * beta2 + (1 - beta2) * g; the EMA of the updated p; bf16(p)"""
    view = cpu_math_ops._view
    step = view(step_ptr, 1, ctypes.c_int64, torch.int64)
    s = int(step[0]) + 1
    step[0] = s
    if lr_dev_ptr:  # a device lr: 1 - lr * wd formed in fp32
        lr = float(view(lr_dev_ptr, 1, ctypes.c_float, F32)[0])
        c_wd = f32(1.0 - f32(lr * f32(weight_decay)))
    else:
        lr, c_wd = f32(lr_host), f32(wd_scale)
    omd = None
    if ema_enabled:
        decay, st = 0.0, max(0, s - ema_update_after_step - 1)
        if st > 0:
            value = 1.0 - (1.0 + st / ema_inv_gamma) ** (-ema_power) if ema_use_warmup else (1.0 + st) / (10.0 + st)
            decay = max(min(value, ema_decay), ema_min_decay)
        if (s - 1) % max(1, ema_update_every) == 0:
            omd = f32(1.0 - decay)
    table = torch.frombuffer((ctypes.c_int64 * (8 * n_entries)).from_address(entries_host), dtype=torch.int64).view(-1, 8)
    two_byte = torch.bfloat16 != torch.float32
    for p_, g_, m_, _, e_, k_, numel, _ in table.tolist():
        assert numel > 0 and numel % 4 == 0
        p, g, m = (view(x, numel, ctypes.c_float, F32) for x in (p_, g_, m_))
        p.mul_(c_wd)
        u = m * f32(beta1) + g * f32(one_minus_beta1)
        p.add_(torch.sign(u), alpha=-lr)
        m.mul_(f32(beta2)).add_(g, alpha=f32(one_minus_beta2))
        if e_ and omd is not None:
            e = view(e_, numel, ctypes.c_float, F32)
            e -= omd * (e - p)
        if k_:
            dst = view(k_, numel, ctypes.c_uint16, torch.bfloat16) if two_byte else view(k_, numel, ctypes.c_float, F32)
            dst.copy_(p)


def install(mp):
    calls = []

    def call(name, *args):
        calls.append(name)
        if name == "muse_lion_ema_step":
            lion_ema_step(*args)
        elif name == "muse_adamw_ema_step":
            cpu_math_ops.adamw_ema_step(*args)
        else:
            raise AssertionError(f"unexpected library call on the CPU: {name}")

    mp.setattr(ops, "_call", call)
    mp.setattr(ops, "_prep", lambda t: 0)
    return calls


# ------------------------------------------------------------------------------------------------ against the reference
NO_DECAY = ["bias", "layer_norm.weight", "mlm_ln.weight", "embeddings.weight"]


def _groups(m, wd=0.05):
    """train_muse.py:427-437: weight decay on everything but biases, norms and embeddings"""
    return [{"params": [p for n, p in m.named_parameters() if not any(nd in n for nd in NO_DECAY)], "weight_decay": wd},
            {"params": [p for n, p in m.named_parameters() if any(nd in n for nd in NO_DECAY)], "weight_decay": 0.0}]


def _flat(m):
    return [p for gr in _groups(m) for p in gr["params"]]


def _models(g, n=2):
    out = []
    for _ in range(n):
        m = MaskGitTransformer(**g["config"])
        m.load_state_dict(g["state_dict"])
        out.append(m.train())
    return out


def _fwd_bwd(m, g):
    _, loss = m(g["batch"]["input_ids"], labels=g["batch"]["labels"])
    loss.backward()
    return loss.detach()


KW = dict(lr=2e-3, betas=(0.9, 0.99), weight_decay=0.05, eps=1e-8)  # eps: train_muse.py:444 passes it to every class


@needs_ref
@pytest.mark.parametrize("warmup", [False, True])
def test_fused_lion_matches_reference_lion_and_emamodel(golden, monkeypatch, warmup):
    """6 steps of the script's name-based groups: parameters and exp_avg equal the reference's bit for bit (the restatement
    runs the reference's ATen ops in its order), the shadows within rounding, the losses of the next forward equal (the
    fused pass wrote the bf16 operands the reference model re-packs), and the state_dict carries the step counter"""
    g = golden("micro_transformer.pt")
    cpu_math_ops.install(monkeypatch, exact=False)
    install(monkeypatch)
    a, b = _models(g)
    ekw = dict(decay=0.99, update_after_step=1, update_every=2, use_ema_warmup=warmup, inv_gamma=2.0, power=0.75)
    ref_opt, ref_ema = _ref_lion()(_groups(a), **KW), _ref_ema()(_flat(a), **ekw)
    ema = EMAModel(_flat(b), **ekw)
    opt = FusedLion(_groups(b), ema=ema, model=b, **KW)
    for step in range(6):
        la, lb = _fwd_bwd(a, g), _fwd_bwd(b, g)
        assert torch.equal(la, lb), step
        ref_opt.step(); ref_ema.step(_flat(a)); ref_opt.zero_grad(set_to_none=True)
        opt.step(); opt.zero_grad(set_to_none=True)
        for (n, pa), pb in zip(a.named_parameters(), b.parameters()):
            assert torch.equal(pb, pa), f"step {step} {n}"
            assert torch.equal(opt.state[pb]["exp_avg"], ref_opt.state[pa]["exp_avg"]), f"step {step} exp_avg {n}"
        for i, (sa, sb) in enumerate(zip(ref_ema.shadow_params, ema.shadow_params)):
            torch.testing.assert_close(sb, sa, rtol=2e-6, atol=1e-8, msg=lambda m_: f"step {step} shadow {i}: {m_}")
        assert ema.optimization_step == ref_ema.optimization_step
    sd = opt.state_dict()
    assert int(next(iter(sd["state"].values()))["step"]) == 6 and len(sd["param_groups"]) == 2


@needs_ref
def test_fused_lion_state_dict_round_trips_through_the_reference(golden, monkeypatch):
    """a FusedLion state loads into the reference Lion and back; a reference state (exp_avg only) loads into FusedLion, whose
    step counter then starts at 0; both continue exactly like the reference"""
    g = golden("micro_transformer.pt")
    cpu_math_ops.install(monkeypatch, exact=False)
    install(monkeypatch)
    Lion = _ref_lion()
    a, b, c = _models(g, 3)
    ref_opt, opt = Lion(_groups(a), **KW), FusedLion(_groups(b), **KW)
    for _ in range(2):
        _fwd_bwd(a, g), _fwd_bwd(b, g)
        ref_opt.step(); opt.step()
        ref_opt.zero_grad(set_to_none=True); opt.zero_grad(set_to_none=True)
    # FusedLion -> reference Lion -> FusedLion
    via_ref = Lion(_groups(c), **KW)
    via_ref.load_state_dict(copy.deepcopy(opt.state_dict()))  # load_state_dict keeps same-device tensors
    back = FusedLion(_groups(c), **KW)
    back.load_state_dict(copy.deepcopy(via_ref.state_dict()))
    for pb, pc in zip(b.parameters(), c.parameters()):
        assert torch.equal(back.state[pc]["exp_avg"], opt.state[pb]["exp_avg"])
        assert int(back.state[pc]["step"]) == 2
    # a reference state without a step counter
    d = _models(g, 1)[0]
    d.load_state_dict(a.state_dict())
    fresh = FusedLion(_groups(d), **KW)
    fresh.load_state_dict(copy.deepcopy(ref_opt.state_dict()))
    _fwd_bwd(a, g), _fwd_bwd(d, g)
    ref_opt.step(); fresh.step()
    for pa, pd in zip(a.parameters(), d.parameters()):
        assert torch.equal(pd, pa) and torch.equal(fresh.state[pd]["exp_avg"], ref_opt.state[pa]["exp_avg"])
    assert int(fresh.state[next(d.parameters())]["step"]) == 1


@needs_ref
def test_fused_lion_skips_parameters_without_grad_and_accepts_eps(monkeypatch):
    install(monkeypatch)
    gen = torch.Generator().manual_seed(0)
    ps = [torch.nn.Parameter(torch.randn(8, generator=gen)) for _ in range(3)]
    rs = [torch.nn.Parameter(p.detach().clone()) for p in ps]
    for p, r in zip(ps, rs):
        r.grad = torch.randn(8, generator=gen)
        p.grad = r.grad.clone()
    ps[1].grad = rs[1].grad = None
    opt, ref = FusedLion(ps, lr=1e-2, weight_decay=0.1, eps=1e-6), _ref_lion()(rs, lr=1e-2, weight_decay=0.1, eps=1e-6)
    before = ps[1].detach().clone()
    for _ in range(3):
        opt.step(); ref.step()
    assert torch.equal(ps[1], before) and ps[1] not in opt.state and rs[1] not in ref.state
    for p, r in zip(ps, rs):
        assert torch.equal(p, r)


@needs_ref
@pytest.mark.parametrize("kw", [dict(lr=-1e-3), dict(betas=(1.0, 0.99)), dict(betas=(0.9, 1.0)), dict(betas=(-0.1, 0.99)),
                                dict(betas=(0.9, -0.5))])
def test_fused_lion_rejects_what_the_reference_rejects(kw):
    ps = [torch.nn.Parameter(torch.zeros(4))]
    with pytest.raises(ValueError):
        _ref_lion()(ps, **kw)
    with pytest.raises(ValueError):
        FusedLion(ps, **kw)


def test_fused_lion_reads_a_tensor_lr(monkeypatch):
    """a one-element fp32 lr reaches the kernel as lr_dev; 1 - lr * wd is then formed in fp32 (within a few ulps of p)"""
    calls = install(monkeypatch)
    gen = torch.Generator().manual_seed(1)
    ps = [torch.nn.Parameter(torch.randn(64, generator=gen))]
    ps[0].grad = torch.randn(64, generator=gen)
    ref = ps[0].detach().double()
    FusedLion(ps, lr=torch.tensor([3e-3]), weight_decay=0.1).step()
    want = ref * (1 - f32(3e-3) * 0.1) - f32(3e-3) * torch.sign(ps[0].grad.double())
    torch.testing.assert_close(ps[0].detach().double(), want, rtol=3e-7, atol=0)
    assert calls == ["muse_lion_ema_step"]
    with pytest.raises(ValueError, match="float64"):
        FusedLion(ps, lr=torch.tensor([1e-3], dtype=torch.float64))


# ------------------------------------------------------------------------------------------------ emulation and mutants
KOPT = 48
NUMELS = [4, 8, 1020, 1024, 1028, 3076]
N_ENTRIES = 97
LR, WD, B1, B2 = 3e-3, 0.1, 0.9, 0.99
STEP0 = 9


def _fma(a, b, c):
    """one fp32 rounding of a * b + c (the product of two fp32 values is exact in fp64)"""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(np.float32)


@pytest.fixture(scope="module")
def operands():
    """per entry p, g, m, shadow; exact zero gradients, and elements where g = m = 0 (u = 0, sign 0)"""
    gen = torch.Generator().manual_seed(7)
    out = []
    for e in range(N_ENTRIES):
        n = NUMELS[e % len(NUMELS)]
        j = torch.arange(n)
        p, g, m, s = (torch.randn(n, generator=gen) * k for k in (1.0, 1e-3, 1e-3, 1.0))
        g[j % 97 == 3] = 0.0
        zero = j % 101 == 5
        g[zero], m[zero] = 0.0, 0.0
        out.append([t.numpy().astype(np.float32) for t in (p, g, m, s)])
    return out


def _omd():
    return np.float32(1.0 - EMAModel([], decay=0.9999, use_ema_warmup=True, power=2 / 3).get_decay(STEP0 + 1))


def _emulate(ops_in, mutant=None):
    """the kernel's outputs (p, m, shadow, bf16 operand) in its chunks of 48 entries and 1024-element blocks; the shadow is
    set on even entries, the bf16 operand on entries 0, 1 mod 4"""
    c_wd, lr = np.float32(1.0 - LR * WD), np.float32(LR)
    b1, b2, c1, c2 = np.float32(B1), np.float32(B2), np.float32(1.0 - B1), np.float32(1.0 - B2)
    omd = _omd()
    out = [[t.copy() for t in e] + [np.full_like(e[0], np.nan)] for e in ops_in]
    for base in range(0, N_ENTRIES, KOPT):
        if mutant == "last chunk skipped" and base + KOPT >= N_ENTRIES:
            continue
        chunk = list(range(base, min(base + KOPT, N_ENTRIES)))
        first, blocks = [], 0
        for e in chunk:
            first.append(blocks)
            blocks += -(-len(ops_in[e][0]) // 1024)
        for blk in range(blocks):
            lo = max(0, int(np.searchsorted(first, blk, side="right")) - 1)
            e = chunk[lo]
            sl = slice((blk - first[lo]) * 1024, (blk - first[lo] + 1) * 1024)
            p, g, m, sh = (t[sl] for t in ops_in[e])
            p1 = p if mutant == "decay after the update" else p * c_wd
            u = m * b1 + g * c1
            m1 = _fma(g, c2, m * b2)
            sg = np.sign(m1 if mutant == "sign of the new m" else u).astype(np.float32)
            p2 = (p1 - lr * sg).astype(np.float32)
            if mutant == "decay after the update":
                p2 = p2 * c_wd
            o = out[e]
            o[0][sl], o[2][sl] = p2, m1
            if e % 2 == 0:
                o[3][sl] = _fma(sh - (p if mutant == "EMA of the pre-step p" else p2), -omd, sh)
            if (e // 2) % 2 == 0:
                o[4][sl] = p2
    return out


def _verify(ops_in, out):
    """p and exp_avg equal to the reference Lion's step of the same tensors, the shadow within BOUNDS ulps of fp64 of the
    kernel's own updated p, the bf16 operand equal to bf16(p')"""
    Lion = _ref_lion()
    ps = [torch.nn.Parameter(torch.from_numpy(e[0].copy())) for e in ops_in]
    ref = Lion(ps, lr=LR, betas=(B1, B2), weight_decay=WD)
    for p, e in zip(ps, ops_in):
        p.grad = torch.from_numpy(e[1].copy())
        ref.state[p]["exp_avg"] = torch.from_numpy(e[2].copy())
    ref.step()
    t = lambda e, k: torch.from_numpy(np.ascontiguousarray(e[k]))  # noqa: E731
    for e, p in enumerate(ps):
        where = f"launch {e // KOPT}, entry {e % KOPT}"
        assert torch.equal(t(out[e], 0), p.detach()), f"p differs from the reference Lion at {where}"
        assert torch.equal(t(out[e], 2), ref.state[p]["exp_avg"]), f"exp_avg differs from the reference Lion at {where}"
        if (e // 2) % 2 == 0:
            assert torch.equal(t(out[e], 4).to(torch.bfloat16), p.detach().to(torch.bfloat16)), f"bf16 operand at {where}"
    ents = [e for e in range(N_ENTRIES) if e % 2 == 0]
    cat = lambda src, k: torch.cat([t(src[e], k) for e in ents])  # noqa: E731
    blk0 = np.cumsum([0] + [-(-len(ops_in[e][0]) // 1024) for e in ents])
    group = torch.cat([torch.arange(len(ops_in[e][0])) // 1024 + int(b) for e, b in zip(ents, blk0)])
    sref, terms = ema_ref(cat(ops_in, 3), cat(out, 0), float(_omd()))
    return check_ulps(cat(out, 3), sref, terms, group, lambda gid: f"(shadow block {gid})", BOUNDS["adamw.ema"][0],
                      "lion.ema")


@needs_ref
def test_lion_emulation_is_accepted(operands):
    res = _verify(operands, _emulate(operands))
    print(f"\nshadow {res.worst:.2f} ulps at {res.where}")


@needs_ref
@pytest.mark.parametrize("mutant", ["decay after the update", "sign of the new m", "EMA of the pre-step p",
                                    "last chunk skipped"])
def test_lion_mutant_is_rejected(operands, mutant):
    with pytest.raises(AssertionError) as info:
        _verify(operands, _emulate(operands, mutant))
    print(f"\n{mutant}: {str(info.value).splitlines()[0][:200]}")


# ------------------------------------------------------------------------------------------------ operand-cache coherence
UVIT = dict(hidden_size=128, num_attention_heads=2, in_channels=64, block_out_channels=(64,), block_num_heads=1,
            num_res_blocks=1, num_hidden_layers=1, intermediate_size=128, codebook_size=64, vocab_size=65,
            encoder_hidden_size=32, cond_embed_dim=32, micro_cond_encode_dim=8, micro_cond_embed_dim=40, num_vq_tokens=16)
V1 = dict(vocab_size=72, hidden_size=64, num_hidden_layers=1, num_attention_heads=1, intermediate_size=128,
          hidden_dropout=0.0, attention_dropout=0.0, max_position_embeddings=16)
MODELS = {"v1": lambda: MaskGitTransformer(**V1), "uvit": lambda: MaskGiTUViT_v2(**UVIT),
          "uvit_downup": lambda: MaskGiTUViT_v2(**UVIT, force_down_up_sample=True)}


def _tensors(W, prefix=""):
    """every tensor operand of a (nested) U-ViT operand dict, by path"""
    out = {}
    for k, v in (W.items() if isinstance(W, dict) else enumerate(W)):
        if torch.is_tensor(v):
            out[prefix + str(k)] = v
        elif isinstance(v, (dict, list)):
            out.update(_tensors(v, f"{prefix}{k}."))
    return out


@pytest.mark.parametrize("use_model", [True, False], ids=["model", "no_model"])
@pytest.mark.parametrize("opt_cls", [FusedAdamW, FusedLion])
@pytest.mark.parametrize("kind", list(MODELS))
def test_fused_step_keeps_the_operand_cache_current(monkeypatch, kind, opt_cls, use_model):
    """after each step the operands the next forward reads equal a cache rebuilt from scratch; with model= the step wrote
    them (and recomputed the depthwise / resample copies), so fetching them re-packs nothing"""
    cpu_math_ops.install(monkeypatch, exact=False)
    install(monkeypatch)
    torch.manual_seed(0)
    m = MODELS[kind]()
    with torch.no_grad():  # every operand non-trivial (adaLN mappers and conv1 start at zero)
        for p in m.parameters():
            p.add_(0.05 * torch.randn_like(p))
    v1 = kind == "v1"
    repacks = []
    if v1:
        pack = ops.pack_bf16
        monkeypatch.setattr(ops, "pack_bf16", lambda *a: (repacks.append(1), pack(*a))[1])
        current = lambda: {"flat": m._packed.refresh().flat}  # noqa: E731
        fresh = lambda: {"flat": _PackedWeights(m).refresh().flat}  # noqa: E731
    else:
        build = MaskGiTUViT_v2._build_weights
        monkeypatch.setattr(MaskGiTUViT_v2, "_build_weights", lambda self: (repacks.append(1), build(self))[1])
        current = lambda: _tensors(m._weights())  # noqa: E731
        fresh = lambda: _tensors(build(m)[0])  # noqa: E731
    before = {k: v.clone() for k, v in current().items()}
    opt = opt_cls(m.parameters(), lr=1e-2, model=m if use_model else None)
    gen = torch.Generator().manual_seed(1)
    for step in range(3):
        for p in m.parameters():
            p.grad = torch.randn(p.shape, generator=gen)
        repacks.clear()
        opt.step()
        got = current()
        if use_model:
            assert repacks == [], f"step {step}: the operands were re-packed after a step with model="
        want = fresh()
        assert got.keys() == want.keys()
        for k in want:
            assert torch.equal(got[k], want[k]), f"step {step}: operand {k} is stale"
    unchanged = [k for k in before if torch.equal(before[k], got[k])]
    assert unchanged == [], f"operands the steps did not move: {unchanged}"
