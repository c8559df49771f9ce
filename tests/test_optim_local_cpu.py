"""The bounds of the fused AdamW + EMA step (tests/local_error.py check_ulps, BOUNDS["adamw.*"]) catch subtly wrong kernels,
and two host-side defects of FusedAdamW stay fixed.

The kernel (csrc/optim.cu) is emulated in fp32 in its own order of operations -- the fused multiply-adds of its compiled
code, IEEE sqrt and division, the chunking of the table into launches of 48 entries and the binary search of each block for
its entry -- over a table of 97 entries (three launches).  The stored bounds accept the emulation and reject each mutant
below; the checks are those of tests/test_optim_local_gpu.py."""
import numpy as np
import pytest
import torch

from open_muse_b200 import EMAModel, FusedAdamW, ops
from tests import cpu_math_ops
from tests.local_error import BOUNDS, AdamHyper, adamw_ref, check_ulps, ema_ref, f32

KOPT = 48
NUMELS = [4, 8, 1020, 1024, 1028, 3076]
N_ENTRIES = 97


def _fma(a, b, c):
    """one fp32 rounding of a * b + c (the product of two fp32 values is exact in fp64)"""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(np.float32)


def _operands(seed=3):
    """per entry: p, g, m, v, shadow (fp32) with a distinct power of two per (entry, 1024-element block, operand), exact
    zero gradients and elements with m = v = g = 0 (as in the GPU test)"""
    gen = torch.Generator().manual_seed(seed)
    out = []
    for e in range(N_ENTRIES):
        n = NUMELS[e % len(NUMELS)]
        j = torch.arange(n)
        blk = j // 1024

        def pow2(role, lo, hi):
            return torch.pow(2.0, ((e * 7 + blk * 13 + role * 5) % (hi - lo + 1) + lo).float())

        p = torch.randn(n, generator=gen) * pow2(0, -8, 6)
        km = pow2(1, -20, 8)
        g, m = torch.randn(n, generator=gen) * km, torch.randn(n, generator=gen) * km
        v = (torch.randn(n, generator=gen) * km * pow2(2, -4, 4)) ** 2
        s = torch.randn(n, generator=gen) * pow2(3, -8, 6)
        g[j % 97 == 3] = 0.0
        zero = j % 101 == 5
        g[zero], m[zero], v[zero] = 0.0, 0.0, 0.0
        out.append([t.numpy().astype(np.float32) for t in (p, g, m, v, s)])
    return out


# (step before the call, update_every): an EMA update at s = 10, a skipped one at s = 11
SETTINGS = {"update": (9, 1), "skip": (10, 3)}
B1, B2, EPS, WD, LR_DEV, LR_HOST = f32(0.9), f32(0.95), f32(1e-8), f32(0.1), f32(3e-3), f32(2e-3)


def _ema(update_every):
    return EMAModel([], decay=f32(0.9999), update_every=update_every, use_ema_warmup=True, inv_gamma=1.0, power=f32(2 / 3))


def _emulate(ops_in, setting, mutant=None):
    """the kernel's outputs (p, m, v, shadow, bf16 operand) for a table whose shadow is set on even entries and whose bf16
    operand is set on entries 0, 1 mod 4; lr is given on the device (lr_host differs)"""
    step0, every = SETTINGS[setting]
    s = step0 + 1
    sb = s - 1 if mutant == "bias correction of step s - 1" else s
    inv_bc1 = np.float32(1.0 / (1.0 - float(B1) ** sb))
    inv_sqrt_bc2 = np.float32(1.0 / (1.0 - float(B2) ** sb) ** 0.5)
    lr = np.float32(LR_HOST if mutant == "lr_host used although lr_dev is given" else LR_DEV)
    ema = _ema(every)
    update = (s - 1) % every == 0 or mutant == "EMA on a skipped update_every step"
    omd = np.float32(1.0 - ema.get_decay(s)) if update else np.float32(-1.0)
    c1, c2 = np.float32(1.0) - np.float32(B1), np.float32(1.0) - np.float32(B2)
    lrwd, step_size = np.float32(lr * np.float32(WD)), np.float32(lr * inv_bc1)
    out = [[t.copy() for t in e] + [np.full_like(e[0], np.nan)] for e in ops_in]  # [5]: the bf16 operand, unwritten
    for base in range(0, N_ENTRIES, KOPT):
        chunk = list(range(base, min(base + KOPT, N_ENTRIES)))
        first, blocks = [], 0
        for e in chunk:
            first.append(blocks)
            blocks += -(-len(ops_in[e][0]) // 1024)
        if mutant == "later launches start one block late" and base > 0:
            first = [b + 1 for b in first]
        for blk in range(blocks):
            lo = max(0, int(np.searchsorted(first, blk, side="right")) - 1)
            e = chunk[lo]
            i0 = (blk - first[lo]) * 1024
            if i0 < 0 or i0 >= len(ops_in[e][0]) or (mutant == "second launch skips entry 48" and e == KOPT):
                continue
            sl = slice(i0, i0 + 1024)
            p, g, m, v, sh = (t[sl] for t in ops_in[e])
            if mutant == "weight decay after the Adam update":
                p1 = p
            else:
                p1 = _fma(p, -lrwd, p)
            m1 = _fma(g - m, c1, m)
            v1 = _fma(v, np.float32(B2), g * (g * c2))
            if mutant == "eps inside the sqrt":
                den = np.sqrt(v1 * inv_sqrt_bc2 * inv_sqrt_bc2 + np.float32(EPS)).astype(np.float32)
            else:
                den = _fma(np.sqrt(v1), inv_sqrt_bc2, np.float32(EPS))
            p2 = p1 - (step_size * m1) / den
            if mutant == "weight decay after the Adam update":
                p2 = _fma(p2, -lrwd, p2)
            o = out[e]
            o[0][sl], o[2][sl], o[3][sl] = p2, m1, v1
            if e % 2 == 0 and omd >= 0:
                src = p if mutant == "EMA of the pre-update p" else p2
                o[4][sl] = _fma(sh - src, -omd, sh)
            if (e // 2) % 2 == 0:
                o[5][sl] = p if mutant == "bf16 operand of the pre-update p" else p2
    return out


def _verify(ops_in, out, setting):
    """the checks of tests/test_optim_local_gpu.py: p, m, v and the shadow within BOUNDS ulps of fp64, a skipped shadow
    bit-unchanged, the bf16 operand bit-equal to the updated p"""
    step0, every = SETTINGS[setting]
    s = step0 + 1
    ema = _ema(every)
    omd = 1.0 - ema.get_decay(s) if (s - 1) % every == 0 else None
    h = AdamHyper(LR_DEV, B1, B2, EPS, WD, s, omd)
    t = lambda e, k: torch.from_numpy(np.ascontiguousarray(e[k]))  # noqa: E731
    cat = lambda src, k, ents=range(N_ENTRIES): torch.cat([t(src[e], k) for e in ents])  # noqa: E731
    nblk = [-(-len(e[0]) // 1024) for e in ops_in]
    blk0 = np.cumsum([0] + nblk)
    group = torch.cat([torch.arange(len(e[0])) // 1024 + int(b) for e, b in zip(ops_in, blk0)])

    def where(gid):
        e = int(np.searchsorted(blk0, gid, side="right")) - 1
        return f"(launch {e // KOPT}, entry {e % KOPT}, block {gid - blk0[e]})"

    ref = adamw_ref(cat(ops_in, 0), cat(ops_in, 1), cat(ops_in, 2), cat(ops_in, 3), h)
    res = {}
    for key, k in (("p", 0), ("m", 2), ("v", 3)):
        res[key] = check_ulps(cat(out, k), *ref[key], group, where, BOUNDS[f"adamw.{key}"][0], f"adamw.{key}")
    ema_ents = [e for e in range(N_ENTRIES) if e % 2 == 0]
    if omd is None:
        assert all(np.array_equal(out[e][4].view(np.int32), ops_in[e][4].view(np.int32)) for e in range(N_ENTRIES)), \
            "a shadow moved on a step the EMA skips"
    else:
        sel = torch.cat([torch.full((len(e[0]),), i % 2 == 0) for i, e in enumerate(ops_in)])
        sref, terms = ema_ref(cat(ops_in, 4, ema_ents), cat(out, 0, ema_ents), omd)
        res["ema"] = check_ulps(cat(out, 4, ema_ents), sref, terms, group[sel], where, BOUNDS["adamw.ema"][0], "adamw.ema")
    for e in range(N_ENTRIES):
        if (e // 2) % 2 == 0:
            want = t(out[e], 0).to(torch.bfloat16)
            assert torch.equal(t(out[e], 5).to(torch.bfloat16), want), f"bf16 operand of entry {e} is not bf16(p')"
    return res


@pytest.fixture(scope="module")
def operands():
    return _operands()


@pytest.mark.parametrize("setting", list(SETTINGS))
def test_adamw_emulation_is_accepted(operands, setting):
    res = _verify(operands, _emulate(operands, setting), setting)
    print("\n" + ", ".join(f"{k} {r.worst:.2f} ulps at {r.where}" for k, r in res.items()))


MUTANTS = [
    ("second launch skips entry 48", "update"),
    ("later launches start one block late", "update"),
    ("bias correction of step s - 1", "update"),
    ("eps inside the sqrt", "update"),
    ("weight decay after the Adam update", "update"),
    ("EMA on a skipped update_every step", "skip"),
    ("EMA of the pre-update p", "update"),
    ("bf16 operand of the pre-update p", "update"),
    ("lr_host used although lr_dev is given", "update"),
]


@pytest.mark.parametrize("mutant,setting", MUTANTS)
def test_adamw_mutant_is_rejected(operands, mutant, setting):
    with pytest.raises(AssertionError) as info:
        _verify(operands, _emulate(operands, setting, mutant), setting)
    print(f"\n{mutant}: {str(info.value).splitlines()[0][:200]}")


# ------------------------------------------------------------------------------------------------ FusedAdamW host fixes
def _params(seed=0):
    g = torch.Generator().manual_seed(seed)
    ps = [torch.nn.Parameter(torch.randn(8, generator=g)), torch.nn.Parameter(torch.randn(4, 4, generator=g))]
    for p in ps:
        p.grad = torch.randn(p.shape, generator=g)
    return ps


def test_fused_adamw_follows_shadows_replaced_by_load_state_dict(monkeypatch):
    """EMAModel.load_state_dict replaces the shadow tensors; with gradients kept in place (zero_grad(set_to_none=False))
    the launch table must still move the new shadows, and leave the old ones alone"""
    cpu_math_ops.install_optimizer(monkeypatch)
    params = _params()
    ema = EMAModel(params, decay=0.99)
    opt = FusedAdamW(params, lr=1e-2, ema=ema)
    opt.step()
    opt.zero_grad(set_to_none=False)
    for p in params:
        p.grad.copy_(torch.randn(p.shape, generator=torch.Generator().manual_seed(5)))
    old = list(ema.shadow_params)  # kept alive: the old tensors stay valid memory whatever the optimizer writes
    old_bits = [o.clone() for o in old]
    ema.load_state_dict({"shadow_params": [torch.full_like(p, 0.5) for p in params]})
    assert all(n.data_ptr() != o.data_ptr() for n, o in zip(ema.shadow_params, old))
    ref = EMAModel(params, decay=0.99)
    ref.load_state_dict({"shadow_params": [torch.full_like(p, 0.5) for p in params], "optimization_step": 1})
    opt.step()
    ref.step(params)
    for o, b in zip(old, old_bits):
        assert torch.equal(o, b), "the step wrote into the replaced shadow tensors"
    for n, r in zip(ema.shadow_params, ref.shadow_params):
        assert not torch.equal(n, torch.full_like(n, 0.5)), "the loaded shadows did not move"
        torch.testing.assert_close(n, r, rtol=2e-6, atol=1e-8)


@pytest.mark.parametrize("bad,what", [
    (lambda dev: torch.tensor([1e-3]), "on cpu"),                             # a host tensor for device parameters
    (lambda dev: torch.tensor([1e-3], dtype=torch.float64, device=dev), "torch.float64"),
    (lambda dev: torch.tensor([1e-3, 1e-3], device=dev), "2 element"),
])
def test_fused_adamw_rejects_a_tensor_lr_the_kernel_cannot_read(monkeypatch, bad, what):
    """the kernel dereferences a tensor lr as one fp32 value at a device address: anything else is refused before the first
    library call.  Parameters on the meta device stand in for device parameters where a host lr would be wrong."""
    calls = []
    monkeypatch.setattr(ops, "_call", lambda *a: calls.append(a))
    monkeypatch.setattr(ops, "_prep", lambda t: 0)
    dev = "meta" if what == "on cpu" else "cpu"
    params = [torch.nn.Parameter(torch.zeros(8, device=dev))]
    params[0].grad = torch.zeros(8, device=dev)
    opt = FusedAdamW(params, lr=1e-3)
    opt.param_groups[0]["lr"] = bad(dev)  # as a scheduler would assign it
    with pytest.raises(ValueError, match=what):
        opt.step()
    assert calls == []
    if what != "on cpu":
        with pytest.raises(ValueError, match=what):
            FusedAdamW(params, lr=bad(dev))


def test_fused_adamw_reads_a_valid_tensor_lr(monkeypatch):
    """a one-element fp32 lr on the parameters' device reaches the kernel as lr_dev"""
    cpu_math_ops.install_optimizer(monkeypatch)
    params, ref = _params(), _params()
    lr = torch.tensor([2e-2])
    opt, ref_opt = FusedAdamW(params, lr=lr), torch.optim.AdamW(ref, lr=2e-2)
    opt.step()
    ref_opt.step()
    for p, r in zip(params, ref):
        torch.testing.assert_close(p, r, rtol=2e-6, atol=1e-8)
