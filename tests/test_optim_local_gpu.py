"""Every tensor of the fused AdamW + EMA step (csrc/optim.cu) against fp64, past its first launch.

The kernel passes its parameter table as launch arguments, at most 48 entries per launch (kOptChunk), and every CTA finds
its entry with a binary search over the entries' first blocks.  Tables of 1 .. 145 entries reach the last entry of a
launch, the first of the next one and up to four launches; entry sizes that are not multiples of 1024 sit right before an
entry that starts on the next block.  Every buffer has guard zones of sentinel bits around every entry, which must stay
bit-unchanged, as must the shadow of an entry without one and every shadow on a step the EMA skips.

Inputs carry a distinct power of two per (entry, 1024-element block), so that a defect in one block shows as a large error
there; g has exact zeros and magnitudes from 1e-6 to 1e3, and some elements have m = v = g = 0 (the update is then the
weight decay alone, exactly).  The fp64 reference (tests/local_error.py adamw_ref / ema_ref) starts from the kernel's fp32
operands and fp32 hyper-parameters; the EMA reference starts from the kernel's own updated p.  Errors are in fp32 ulps of
each element's own terms (check_ulps): the update is a small part of p, and a whole-tensor norm would hide it.

The second half runs FusedAdamW on the base MaskGitTransformer (94 tensors; the decay group needs two launches) with two
parameter groups, EMA warm-up and a device learning rate, eagerly and as a replayed CUDA graph."""
import numpy as np
import pytest
import torch

from open_muse_b200 import EMAModel, FusedAdamW, MaskGitTransformer, ops
from tests.local_error import BOUNDS, AdamHyper, adamw_ref, check_ulps, ema_ref, f32

pytestmark = pytest.mark.gpu
DEV = "cuda"
KOPT = 48  # table entries per launch (kOptChunk, csrc/optim.cu)
NUMELS = [4, 8, 1020, 1024, 1028, 3076, 2 ** 18 + 4, 2 ** 20]  # 2^20: the largest weight of the base model
GUARD = 1024
SENT32, SENT16 = 0x7FBADBAD, 0x7FAB  # NaN bit patterns in the guard zones (fp32 buffers / the bf16 operand)

_worst = {}


def _record(key, res, case):
    if key not in _worst or res.worst > _worst[key][0].worst:
        _worst[key] = (res, case)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst element error per output, in fp32 ulps of its terms (bound; group; whole-tensor rel-L2 of that case):")
    for key in ("adamw.p", "adamw.m", "adamw.v", "adamw.ema"):
        if key in _worst:
            r, case = _worst[key]
            print(f"  {key:10s} {r.worst:.2f} (bound {BOUNDS[key][0]:g}) {case} {r.where}; whole {r.whole:.3e}")


# EMA settings: (enabled, decay, min_decay, update_after_step, update_every, use_warmup, inv_gamma, power)
EMA = {
    "off": (0, 0.9999, 0.0, 0, 1, 0, 1.0, 2 / 3),
    "plain": (1, 0.9999, 0.0, 0, 1, 0, 1.0, 2 / 3),
    "warmup": (1, 0.9999, 0.0, 0, 1, 1, 1.0, 2 / 3),
    "decay0": (1, 0.9999, 0.0, None, 1, 1, 1.0, 2 / 3),  # update_after_step past the step: decay 0, s' = p'
    "every3": (1, 0.999, 0.5, 2, 3, 0, 1.0, 2 / 3),
    "late": (1, 0.99, 0.1, 5, 1, 1, 2.0, 0.75),
}


def _ema_args(name, step0):
    en, d, md, ua, ue, w, ig, pw = EMA[name]
    return en, f32(d), f32(md), step0 + 3 if ua is None else ua, ue, w, f32(ig), f32(pw)


def _ema_args_of(ema):
    """the EMA arguments FusedAdamW passes for an EMAModel"""
    return (1, f32(ema.decay), f32(ema.min_decay), ema.update_after_step, ema.update_every, int(ema.use_ema_warmup),
            f32(ema.inv_gamma), f32(ema.power))


def _expected_scalars(beta1, beta2, lr, ema_args, s):
    """scal[0..5] as the fp64 formulas (EMAModel.get_decay for the EMA decay) give them, with the kernel's fp32 inputs"""
    en, d, md, ua, ue, w, ig, pw = ema_args
    decay, omd = 0.0, None
    if en:
        ref = EMAModel([], decay=d, min_decay=md, update_after_step=ua, update_every=ue, use_ema_warmup=bool(w),
                       inv_gamma=ig, power=pw)
        decay = ref.get_decay(s)
        if (s - 1) % ue == 0:
            omd = 1.0 - decay
    h = AdamHyper(lr, beta1, beta2, 0.0, 0.0, s, omd)
    return [float(s), h.inv_bc1, h.inv_sqrt_bc2, lr, -1.0 if omd is None else omd, decay], omd


def _check_scalars(scal, expected, case):
    got = scal[:6].cpu().numpy()
    for k, (a, e) in enumerate(zip(got, expected)):
        ulp = float(np.spacing(np.float32(abs(e))))
        assert abs(float(a) - e) <= ulp, f"{case}: scal[{k}] = {float(a)!r}, fp64 {e!r} (one ulp {ulp:.3e})"


def _call(table, n, scal, step_dev, lr_dev, lr_host, beta1, beta2, eps, wd, ema_args):
    en, d, md, ua, ue, w, ig, pw = ema_args
    ops._call("muse_adamw_ema_step", table.ctypes.data, n, scal.data_ptr(), step_dev.data_ptr(),
              None if lr_dev is None else lr_dev.data_ptr(), lr_host, beta1, beta2, eps, wd, en, d, md, ua, ue, w, ig, pw,
              ops._prep(scal))


# ------------------------------------------------------------------------------------------------ the kernel, C ABI
class Table:
    """n entries, numel cycled from NUMELS, the EMA shadow on even entries and the bf16 operand on entries 0, 1 mod 4 (all
    four combinations inside every launch and across every launch boundary), each entry's elements at its own offset in
    one guarded buffer per operand: [guard][entry 0][guard][entry 1]...[guard]"""

    def __init__(self, n):
        self.n = n
        self.numel = [NUMELS[i % len(NUMELS)] for i in range(n)]
        self.has_ema = [i % 2 == 0 for i in range(n)]
        self.has_packed = [(i // 2) % 2 == 0 for i in range(n)]
        off, pos = [], GUARD
        for k in self.numel:
            off.append(pos)
            pos += k + GUARD
        self.off, self.total = off, pos
        self.idx = torch.cat([torch.arange(o, o + k) for o, k in zip(off, self.numel)]).to(DEV)  # dense -> buffer
        self.ent = torch.cat([torch.full((k,), i) for i, k in enumerate(self.numel)]).to(DEV)
        self.j = torch.cat([torch.arange(k) for k in self.numel]).to(DEV)                     # index in the entry
        nblk = [-(-k // 1024) for k in self.numel]
        self.blk0 = np.cumsum([0] + nblk)
        self.group = torch.tensor(self.blk0[:-1], device=DEV)[self.ent] + self.j // 1024      # (entry, block) id

    def where(self, gid):
        e = int(np.searchsorted(self.blk0, gid, side="right")) - 1
        return (f"(launch {e // KOPT}, entry {e % KOPT} = table row {e}, block {gid - self.blk0[e]} of "
                f"{self.blk0[e + 1] - self.blk0[e]}, numel {self.numel[e]})")

    def dense_mask(self, flags):
        return torch.tensor(flags, device=DEV)[self.ent]

    def buffer(self, values, dtype=torch.float32):
        b = torch.empty(self.total, dtype=dtype, device=DEV)
        b.view(torch.int32 if dtype == torch.float32 else torch.int16).fill_(SENT32 if dtype == torch.float32 else SENT16)
        if values is not None:
            b[self.idx] = values
        return b

    def rows(self, bufs):
        """the int64 table of FusedAdamW._plan: {p, g, m, v, ema, packed, numel, 0} per entry"""
        p, g, m, v, s, k = bufs
        t = np.zeros((self.n, 8), dtype=np.int64)
        for i, (o, numel) in enumerate(zip(self.off, self.numel)):
            t[i] = (p.data_ptr() + 4 * o, g.data_ptr() + 4 * o, m.data_ptr() + 4 * o, v.data_ptr() + 4 * o,
                    s.data_ptr() + 4 * o if self.has_ema[i] else 0, k.data_ptr() + 2 * o if self.has_packed[i] else 0,
                    numel, 0)
        return np.ascontiguousarray(t)


def _pow2(tab, role, lo, hi):
    """2^k, k in [lo, hi], distinct per (entry, 1024-element block, operand)"""
    blk = tab.j // 1024
    k = (tab.ent * 7 + blk * 13 + role * 5) % (hi - lo + 1) + lo
    return torch.pow(2.0, k.float())


def _operands(tab, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    N = tab.idx.numel()
    rnd = lambda: torch.randn(N, device=DEV, generator=gen)  # noqa: E731
    p = rnd() * _pow2(tab, 0, -8, 6)
    km = _pow2(tab, 1, -20, 8)                               # |g|, |m| from ~1e-6 to ~1e3
    g = rnd() * km
    m = rnd() * km
    v = (rnd() * km * _pow2(tab, 2, -4, 4)) ** 2             # sqrt(v) within 2^+-4 of |m|
    s = rnd() * _pow2(tab, 3, -8, 6)
    g[tab.j % 97 == 3] = 0.0                                 # exact zero gradients
    zero = tab.j % 101 == 5                                  # m = v = g = 0: the update is the weight decay alone
    g[zero], m[zero], v[zero] = 0.0, 0.0, 0.0
    return p, g, m, v, s, zero


# (n_entries, step_dev before the call, EMA setting, learning rate on the host or on the device)
CASES = [(1, 0, "off", "host"), (47, 1, "plain", "dev"), (48, 9, "warmup", "host"), (49, 999, "decay0", "dev"),
         (96, 10 ** 6, "every3", "host"),   # (s - 1) % 3 != 0: the EMA skips this step
         (97, 9, "every3", "dev"),          # s = 10: an EMA step of update_every = 3
         (145, 0, "late", "dev")]


@pytest.mark.parametrize("n,step0,ema,lr_mode", CASES)
def test_adamw_ema_step_local(n, step0, ema, lr_mode):
    tab = Table(n)
    p, g, m, v, s, zero = _operands(tab, 100 + n)
    bufs = [tab.buffer(t) for t in (p, g, m, v, s)] + [tab.buffer(None, torch.bfloat16)]
    before = [b.clone() for b in bufs]
    beta1, beta2 = (f32(0.9), f32(0.95)) if n % 2 else (f32(0.9), f32(0.999))
    eps, wd, lr = f32(1e-8), f32(0.1), f32(2e-3 if lr_mode == "host" else 3e-3)
    lr_dev = torch.tensor([lr], device=DEV) if lr_mode == "dev" else None
    lr_host = lr if lr_mode == "host" else 7.0  # ignored when lr_dev is given
    ema_args = _ema_args(ema, step0)
    step_dev = torch.tensor([step0], dtype=torch.int64, device=DEV)
    scal = torch.full((8,), float("nan"), device=DEV)
    table = tab.rows(bufs)
    _call(table, n, scal, step_dev, lr_dev, lr_host, beta1, beta2, eps, wd, ema_args)
    torch.cuda.synchronize()
    case = f"(entries {n}, step {step0} -> {step0 + 1}, EMA {ema}, lr on the {lr_mode})"

    assert int(step_dev) == step0 + 1, case
    s_new = step0 + 1
    expected, omd = _expected_scalars(beta1, beta2, lr, ema_args, s_new)
    _check_scalars(scal, expected, case)

    # guards and entries without a shadow / bf16 operand: bit-unchanged; g: never written
    untouched = torch.ones(tab.total, dtype=torch.bool, device=DEV)
    untouched[tab.idx] = False
    no_ema, no_packed = untouched.clone(), untouched.clone()
    no_ema[tab.idx] = ~tab.dense_mask(tab.has_ema) if omd is not None else True
    no_packed[tab.idx] = ~tab.dense_mask(tab.has_packed)
    for name, b, b0, mask in zip("pgmvsk", bufs, before, (untouched, None, untouched, untouched, no_ema, no_packed)):
        bits = torch.int16 if b.dtype == torch.bfloat16 else torch.int32
        if mask is None:
            assert torch.equal(b.view(bits), b0.view(bits)), f"{case}: the kernel wrote into g"
        else:
            changed = (b.view(bits) != b0.view(bits)) & mask
            assert not bool(changed.any()), \
                f"{case}: buffer {name} changed outside what the table lets the kernel write, first at element " \
                f"{int(changed.nonzero()[0])}"

    p1, m1, v1, s1 = (bufs[k][tab.idx] for k in (0, 2, 3, 4))
    h = AdamHyper(lr, beta1, beta2, eps, wd, s_new, omd)
    ref = adamw_ref(p, g, m, v, h)
    for key, out in (("p", p1), ("m", m1), ("v", v1)):
        res = check_ulps(out, *ref[key], tab.group, tab.where, BOUNDS[f"adamw.{key}"][0], f"adamw.{key} {case}")
        _record(f"adamw.{key}", res, case)
    # m = v = g = 0: p' = p - (lr wd) p, one fp32 rounding of the exact value (the kernel's fma)
    t = f32(lr * wd)
    exact = (p[zero].double() - t * p[zero].double()).float()
    assert torch.equal(p1[zero], exact), f"{case}: update with m = v = g = 0 is not p - lr wd p"
    assert torch.equal(m1[zero], m[zero]) and torch.equal(v1[zero], v[zero]), case
    if omd is not None:
        sel = tab.dense_mask(tab.has_ema)
        sref, sterms = ema_ref(s[sel], p1[sel], omd)
        res = check_ulps(s1[sel], sref, sterms, tab.group[sel], tab.where, BOUNDS["adamw.ema"][0], f"adamw.ema {case}")
        _record("adamw.ema", res, case)
    sel = tab.dense_mask(tab.has_packed)
    k1 = bufs[5][tab.idx][sel]
    assert torch.equal(k1.view(torch.int16), p1[sel].to(torch.bfloat16).view(torch.int16)), \
        f"{case}: the bf16 operand is not the updated p rounded to bf16"


@pytest.mark.parametrize("ema", ["off", "plain", "warmup", "every3", "late"])
def test_adamw_step_scalars(ema):
    """scal[0..5] of the prepare kernel over a sweep of steps: the bias corrections approach 1, the EMA decay reaches its
    clamp; each within one fp32 ulp of fp64"""
    tab = Table(1)
    bufs = [tab.buffer(torch.ones(4, device=DEV)) for _ in range(5)] + [tab.buffer(None, torch.bfloat16)]
    table = tab.rows(bufs)
    scal = torch.zeros(8, device=DEV)
    beta1, beta2, lr = f32(0.9), f32(0.999), f32(1e-4)
    for s in list(range(1, 13)) + [99, 100, 101, 999, 1000, 12345, 10 ** 6, 10 ** 7]:
        ema_args = _ema_args(ema, s - 1)
        step_dev = torch.tensor([s - 1], dtype=torch.int64, device=DEV)
        _call(table, 1, scal, step_dev, None, lr, beta1, beta2, f32(1e-8), 0.0, ema_args)
        torch.cuda.synchronize()
        assert int(step_dev) == s
        _check_scalars(scal, _expected_scalars(beta1, beta2, lr, ema_args, s)[0], f"(EMA {ema}, step {s})")


# ------------------------------------------------------------------------------------------------ the base model
BASE_CFG = dict(vocab_size=2025, max_position_embeddings=257, hidden_size=512, num_hidden_layers=8,
                num_attention_heads=8, intermediate_size=2048, codebook_size=1024, num_vq_tokens=256, num_classes=1000,
                hidden_dropout=0.0, attention_dropout=0.0)
NO_DECAY = ["bias", "layer_norm.weight", "mlm_ln.weight", "embeddings.weight"]  # train_muse.py's name-based groups


def _batch(B=4, S=256):
    g = torch.Generator().manual_seed(7)
    tok = torch.randint(0, 1024, (B, S), generator=g)
    mask = torch.rand(B, S, generator=g) < 0.5
    ids = torch.cat([1024 + torch.randint(0, 1000, (B, 1), generator=g), torch.where(mask, 2024, tok)], 1)
    lab = torch.cat([torch.full((B, 1), -100), torch.where(mask, tok, -100)], 1)
    return ids.to(DEV), lab.to(DEV)


class Snapshot:
    """p, g, m, v and the EMA shadow of every parameter before a step (the reference of the step starts from them)"""

    def __init__(self, opt, ema, grads=None):
        flat = [p for gr in opt.param_groups for p in gr["params"]]
        shadow = {id(p): sh for p, sh in zip(flat, ema.shadow_params)}
        self.t = {}
        for i, p in enumerate(flat):
            st = opt.state[p]
            g = p.grad if grads is None else grads[i]
            assert g is not None, "every parameter must have a gradient at every step"
            z = torch.zeros_like(p)
            self.t[id(p)] = [x.detach().clone() for x in (p, g, st.get("exp_avg", z), st.get("exp_avg_sq", z),
                                                          shadow[id(p)])]
        self.step = [int(opt._plans[gi]["step"]) if gi in opt._plans else 0 for gi in range(len(opt.param_groups))]


def _check_model_step(opt, ema, names, snap, lr, case):
    flat = [p for gr in opt.param_groups for p in gr["params"]]
    shadow = {id(p): sh for p, sh in zip(flat, ema.shadow_params)}
    for gi, gr in enumerate(opt.param_groups):
        params = gr["params"]
        s = snap.step[gi] + 1
        plan = opt._plans[gi]
        assert int(plan["step"]) == s, f"{case}: group {gi} step counter {int(plan['step'])}, expected {s}"
        decay = ema.get_decay(s)
        b1, b2 = gr["betas"]
        h = AdamHyper(lr, f32(b1), f32(b2), f32(gr["eps"]), f32(gr["weight_decay"]), s, 1.0 - decay)
        _check_scalars(plan["scal"], _expected_scalars(f32(b1), f32(b2), lr, _ema_args_of(ema), s)[0],
                       f"{case} group {gi}")
        cat = lambda k: torch.cat([snap.t[id(p)][k].flatten() for p in params])  # noqa: E731
        p0, g0, m0, v0, s0 = (cat(k) for k in range(5))
        new = [torch.cat([t.detach().flatten() for t in ts]) for ts in
               ([p for p in params], [opt.state[p]["exp_avg"] for p in params],
                [opt.state[p]["exp_avg_sq"] for p in params], [shadow[id(p)] for p in params])]
        blk0 = np.cumsum([0] + [-(-p.numel() // 1024) for p in params])
        group = torch.cat([torch.arange(p.numel(), device=DEV) // 1024 + int(b) for p, b in zip(params, blk0)])

        def where(gid, blk0=blk0, params=params, gi=gi):
            e = int(np.searchsorted(blk0, gid, side="right")) - 1
            return (f"({names[id(params[e])]}: group {gi}, launch {e // KOPT}, entry {e % KOPT}, block "
                    f"{gid - blk0[e]} of {blk0[e + 1] - blk0[e]})")

        ref = adamw_ref(p0, g0, m0, v0, h)
        for key, out in zip(("p", "m", "v"), new[:3]):
            res = check_ulps(out, *ref[key], group, where, BOUNDS[f"adamw.{key}"][0], f"adamw.{key} {case} group {gi}")
            _record(f"adamw.{key}", res, f"{case} group {gi}")
        res = check_ulps(new[3], *ema_ref(s0, new[0], 1.0 - decay), group, where, BOUNDS["adamw.ema"][0],
                         f"adamw.ema {case} group {gi}")
        _record("adamw.ema", res, f"{case} group {gi}")


def test_fused_adamw_base_model_local():
    """FusedAdamW on the base model with the decay / no-decay groups of train_muse.py (58 and 36 tensors: the decay group
    takes two launches), EMA warm-up and a device learning rate changed in place: 3 eager steps, then 3 replays of the
    captured step, each checked against fp64 from the kernel's own state before it"""
    torch.manual_seed(0)
    model = MaskGitTransformer(**BASE_CFG).to(DEV).train()
    names = {id(p): n for n, p in model.named_parameters()}
    groups = [{"params": [p for n, p in model.named_parameters() if not any(nd in n for nd in NO_DECAY)],
               "weight_decay": 0.05},
              {"params": [p for n, p in model.named_parameters() if any(nd in n for nd in NO_DECAY)], "weight_decay": 0.0}]
    assert [len(g["params"]) for g in groups] == [58, 36]
    flat = [p for g in groups for p in g["params"]]
    ema = EMAModel(flat, decay=f32(0.9999), use_ema_warmup=True, inv_gamma=1.0, power=f32(2 / 3))
    lr = torch.tensor([1e-3], device=DEV)
    opt = FusedAdamW(groups, lr=lr, betas=(0.9, 0.95), eps=1e-8, ema=ema, model=model)
    ids, lab = _batch()

    def fwd_bwd():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            _, loss = model(ids, labels=lab)
        loss.backward()
        return loss.detach()

    for k, lr_k in enumerate((1e-3, 2.5e-3, 4e-4)):
        lr.fill_(lr_k)
        fwd_bwd()
        snap = Snapshot(opt, ema)
        opt.step()
        torch.cuda.synchronize()
        _check_model_step(opt, ema, names, snap, f32(lr_k), f"(base model, eager step {k + 1})")
        opt.zero_grad(set_to_none=True)

    from open_muse_b200.graphs import GraphedStep

    grads = [torch.empty_like(p) for p in flat]  # this step's gradients, copied out inside the graph

    def step(i, l):
        with torch.autocast("cuda", dtype=torch.bfloat16):
            _, loss = model(i, labels=l)
        loss.backward()
        for gbuf, p in zip(grads, flat):
            gbuf.copy_(p.grad)
        opt.step()
        opt.zero_grad(set_to_none=True)
        return loss.detach()

    gs = GraphedStep(step, (ids, lab), warmup=2)
    for k, lr_k in enumerate((3e-3, 5e-4, 1.5e-3)):
        lr.fill_(lr_k)
        torch.cuda.synchronize()
        snap = Snapshot(opt, ema, grads=[torch.zeros_like(p) for p in flat])
        decay_before = float(opt._plans[0]["scal"][5])
        gs(ids, lab)
        torch.cuda.synchronize()
        for i, gbuf in enumerate(grads):  # the reference takes the gradients of this replay
            snap.t[id(flat[i])][1] = gbuf.clone()
        assert float(opt._plans[0]["scal"][5]) > decay_before, "the EMA warm-up schedule did not advance"
        _check_model_step(opt, ema, names, snap, f32(lr_k), f"(base model, graph replay {k + 1})")
