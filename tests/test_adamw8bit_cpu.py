"""FusedAdamW8bit WITHOUT a GPU: the quantisation maps, the host logic, an fp64 verifier that accepts the kernel's contract
and rejects five mutants of it, state_dict round trips, the unmodified train_muse.py with ``optimizer.name: 8bit_adamw``,
operand-cache coherence and the state's memory.

``muse_adamw8bit_ema_step`` (csrc/optim.cu) is restated here in torch: it dereferences the same host table of {p, g, m, v,
ema, packed, numel, -, absmax1, absmax2} rows, the maps buffer, the device-resident step counter and the fp32 scalars the
C ABI receives; ``ops._call`` is routed to it (and ``muse_adamw_ema_step`` to tests/cpu_math_ops.py).  GPU twin:
tests/test_adamw8bit_gpu.py."""
import copy
import ctypes
import sys
import types
from dataclasses import dataclass

import numpy as np
import pytest
import torch

from open_muse_b200 import EMAModel, FusedAdamW, FusedAdamW8bit, MaskGitTransformer, MaskGiTUViT_v2, ops
from open_muse_b200.optim import (BUCKET_BASE, BUCKETS, MIN_8BIT_SIZE, QBLOCK, START_BYTES, _maps_buffer, bucket_starts,
                                  dynamic_map, midpoints)
from tests import cpu_math_ops
from tests.local_error import BOUNDS, AdamHyper, adamw_ref, check_ulps, f32

F32 = torch.float32
MUTANTS = ["absmax from the old state", "p takes the re-quantised m", "ties to the upper code",
           "blocks across tensor boundaries", "decay after the update"]


# ------------------------------------------------------------------------------------------------ the kernel, restated
@dataclass
class Hyper:
    """the fp32 values the kernel computes with: lr, 1 / bias_correction1, 1 / sqrt(bias_correction2), betas, eps, decay"""
    lr: float
    inv_bc1: float
    inv_sqrt_bc2: float
    beta1: float
    beta2: float
    eps: float
    wd: float


def _adamw(p, g, m, v, h, mutant=None):
    """FusedAdamW's element update in fp32 (tests/cpu_math_ops.adamw_ema_step's formula); returns new p, m, v"""
    if mutant != "decay after the update":
        p = p - h.lr * h.wd * p
    m = m + (1.0 - h.beta1) * (g - m)
    v = v * h.beta2 + (1.0 - h.beta2) * g * g
    den = v.sqrt() * h.inv_sqrt_bc2 + h.eps
    p1 = p - (h.lr * h.inv_bc1) * m / den
    if mutant == "decay after the update":
        p1 = p1 - h.lr * h.wd * p1
    return p1, m, v, p, den


def step8(entries, maps, h, mutant=None):
    """one 8-bit step over `entries`, lists [p, g, codes1, codes2, absmax1, absmax2] of fp32 / uint8 tensors, updated in
    place; `mutant` (one of MUTANTS) breaks one rule of the contract"""
    q1, q2, mid1, mid2 = maps[:256], maps[256:512], maps[512:767], maps[768:1023]
    upd = []
    for p, g, c1, c2, a1, a2 in entries:
        blk = torch.arange(p.numel()) // QBLOCK
        m0 = q1[c1.reshape(-1).long()] * a1[blk]  # decode: one fp32 product each
        v0 = q2[c2.reshape(-1).long()] * a2[blk]
        upd.append((blk,) + _adamw(p.reshape(-1), g.reshape(-1), m0, v0, h, mutant))
    if mutant == "blocks across tensor boundaries":  # blocks counted over the concatenated tensors
        gm, gv = torch.cat([u[2].abs() for u in upd]), torch.cat([u[3] for u in upd])
        gb = torch.arange(gm.numel()) // QBLOCK
        amax = [torch.zeros(int(gb.max()) + 1).scatter_reduce(0, gb, t, "amax", include_self=False) for t in (gm, gv)]
        first = 0
    for (p, g, c1, c2, a1, a2), (blk, p1, m, v, p_decayed, den) in zip(entries, upd):
        if mutant == "absmax from the old state":
            n1, n2 = a1.clone(), a2.clone()
        elif mutant == "blocks across tensor boundaries":
            own = (torch.arange(0, p.numel(), QBLOCK) + first) // QBLOCK  # the global block of each block's first element
            first += p.numel()
            n1, n2 = amax[0][own], amax[1][own]
        else:
            n1 = torch.zeros_like(a1).scatter_reduce(0, blk, m.abs(), "amax", include_self=False)
            n2 = torch.zeros_like(a2).scatter_reduce(0, blk, v, "amax", include_self=False)
        d1, d2 = n1[blk], n2[blk]
        x1 = torch.where(d1 > 0, m / torch.where(d1 > 0, d1, 1.0), 0.0)  # IEEE fp32 division; 0 where absmax is 0
        x2 = torch.where(d2 > 0, v / torch.where(d2 > 0, d2, 1.0), 0.0)
        side = "right" if mutant == "ties to the upper code" else "left"
        k1, k2 = torch.searchsorted(mid1, x1, side=side), torch.searchsorted(mid2, x2, side=side)
        if mutant == "p takes the re-quantised m":
            p1 = p_decayed - (h.lr * h.inv_bc1) * (q1[k1] * d1) / den
        p.copy_(p1.view(p.shape))
        c1.copy_(k1.to(torch.uint8).view(c1.shape))
        c2.copy_(k2.to(torch.uint8).view(c2.shape))
        a1.copy_(n1)
        a2.copy_(n2)


def _view(ptr, n, ctype, dtype):
    return cpu_math_ops._view(ptr, n, ctype, dtype)


def adamw8bit_ema_step(entries_host, n_entries, maps_ptr, scal_ptr, step_ptr, lr_dev_ptr, lr_host, beta1, beta2, eps,
                       weight_decay, ema_enabled, ema_decay, ema_min_decay, ema_update_after_step, ema_update_every,
                       ema_use_warmup, ema_inv_gamma, ema_power, stream):
    """csrc/optim.cu's 8-bit pass: rows with absmax1 == 0 through FusedAdamW's pass (tests/cpu_math_ops.py) on fp32
    moments; the others through step8 with every float argument rounded to fp32 as the C ABI does and the prepare kernel's
    scalars, then the EMA of the updated p and its bf16 copy"""
    step = _view(step_ptr, 1, ctypes.c_int64, torch.int64)
    s = int(step[0]) + 1
    table = torch.frombuffer((ctypes.c_int64 * (10 * n_entries)).from_address(entries_host), dtype=torch.int64).view(-1, 10)
    fp32_rows = table[table[:, 8] == 0, :8].numpy().copy()
    if len(fp32_rows):  # the fp32-moment entries: FusedAdamW's pass, on a copy of the step counter
        before = torch.tensor([s - 1], dtype=torch.int64)
        cpu_math_ops.adamw_ema_step(fp32_rows.ctypes.data, len(fp32_rows), scal_ptr, before.data_ptr(), lr_dev_ptr, lr_host,
                                    beta1, beta2, eps, weight_decay, ema_enabled, ema_decay, ema_min_decay,
                                    ema_update_after_step, ema_update_every, ema_use_warmup, ema_inv_gamma, ema_power,
                                    stream)
    step[0] = s
    beta1, beta2, eps, weight_decay = f32(beta1), f32(beta2), f32(eps), f32(weight_decay)
    lr = float(_view(lr_dev_ptr, 1, ctypes.c_float, F32)[0]) if lr_dev_ptr else f32(lr_host)
    h = Hyper(lr, f32(1.0 / (1.0 - beta1 ** s)), f32(1.0 / (1.0 - beta2 ** s) ** 0.5), beta1, beta2, eps, weight_decay)
    omd = None
    if ema_enabled:
        decay, st = 0.0, max(0, s - ema_update_after_step - 1)
        if st > 0:
            value = 1.0 - (1.0 + st / ema_inv_gamma) ** (-ema_power) if ema_use_warmup else (1.0 + st) / (10.0 + st)
            decay = max(min(value, ema_decay), ema_min_decay)
        if (s - 1) % max(1, ema_update_every) == 0:
            omd = f32(1.0 - decay)
    maps = _view(maps_ptr, 1024, ctypes.c_float, F32).clone()
    two_byte = torch.bfloat16 != torch.float32
    for p_, g_, m_, v_, e_, k_, numel, _, a1_, a2_ in table.tolist():
        assert numel > 0 and numel % 4 == 0
        if a1_ == 0:
            continue
        p, g = _view(p_, numel, ctypes.c_float, F32), _view(g_, numel, ctypes.c_float, F32)
        nb = -(-numel // QBLOCK)
        step8([[p, g, _view(m_, numel, ctypes.c_uint8, torch.uint8), _view(v_, numel, ctypes.c_uint8, torch.uint8),
                _view(a1_, nb, ctypes.c_float, F32), _view(a2_, nb, ctypes.c_float, F32)]], maps, h)
        if e_ and omd is not None:
            e = _view(e_, numel, ctypes.c_float, F32)
            e -= omd * (e - p)
        if k_:
            dst = _view(k_, numel, ctypes.c_uint16, torch.bfloat16) if two_byte else _view(k_, numel, ctypes.c_float, F32)
            dst.copy_(p)


def install(mp):
    calls = []

    def call(name, *args):
        calls.append(name)
        if name == "muse_adamw8bit_ema_step":
            adamw8bit_ema_step(*args)
        elif name == "muse_adamw_ema_step":
            cpu_math_ops.adamw_ema_step(*args)
        else:
            raise AssertionError(f"unexpected library call on the CPU: {name}")

    mp.setattr(ops, "_call", call)
    mp.setattr(ops, "_prep", lambda t: 0)
    return calls


# ------------------------------------------------------------------------------------------------ maps
def _recipe(signed):
    data = []
    for i in range(7):
        n = 2 ** i + 1 if signed else 2 ** (i + 1) + 1
        b = torch.linspace(0.1, 1, n)
        means = (b[:-1] + b[1:]) / 2.0
        data += ((10 ** (-6 + i)) * means).tolist()
        if signed:
            data += (-(10 ** (-6 + i)) * means).tolist()
    data += [0.0, 1.0]
    return torch.tensor(sorted(data), dtype=F32)


@pytest.mark.parametrize("signed", [True, False])
def test_maps_follow_the_recipe(signed):
    q = dynamic_map(signed)
    assert q.dtype == F32 and q.shape == (256,)
    assert torch.equal(q, _recipe(signed))
    assert bool((q[1:] > q[:-1]).all()), "the map is not strictly increasing"
    assert float(q[127 if signed else 0]) == 0.0 and float(q[-1]) == 1.0
    if signed:
        assert abs(float(q[0]) + 0.99297) < 1e-5
    buf = _maps_buffer("cpu")
    mid = midpoints(q)
    assert torch.equal(mid, (q[:-1] + q[1:]) / 2) and bool((mid > q[:-1]).all() and (mid < q[1:]).all())
    assert torch.equal(buf[(0 if signed else 256):][:256], q)
    assert torch.equal(buf[(512 if signed else 768):][:255], mid)


def kernel_search(mid, start_pos, start_neg, x):
    """csrc/optim.cu quantize(): the bucket's start code, then forward while mid[k] < x; returns (codes, steps taken)"""
    u = x.view(torch.int32).long() & 0xFFFFFFFF
    b = (((u & 0x7FFFFFFF) >> 18) - BUCKET_BASE).clamp(0, BUCKETS - 1)
    k = torch.where(u >> 31 == 1, start_neg[b], start_pos[b]).long()
    steps = torch.zeros_like(k)
    while True:
        adv = (k < 255) & (mid[k.clamp(max=254)] < x)
        if not bool(adv.any()):
            return k, steps
        k, steps = k + adv.long(), steps + adv.long()


@pytest.mark.parametrize("signed", [True, False])
def test_encoder_first_guess_gives_the_searchsorted_codes(signed):
    """the kernel's encoder (a start code per bucket of |x|, then a forward neighbour compare) equals
    searchsorted(M, x, side="left") on every midpoint and its fp32 neighbours, every bucket bound and its neighbours, 0,
    -0, +-1 and 4 M random values over the maps' decades, in at most 2 (signed) / 3 (unsigned) forward steps"""
    mid = midpoints(dynamic_map(signed))
    buf = _maps_buffer("cpu")
    tables = buf[1024:].view(torch.uint8).view(3, START_BYTES)[:, :BUCKETS].long()
    sp, sn = (tables[0], tables[1]) if signed else (tables[2], tables[2])
    assert torch.equal(sp, bucket_starts(mid, False)) and (not signed or torch.equal(sn, bucket_starts(mid, True)))
    gen = torch.Generator().manual_seed(0)
    b = torch.arange(1, BUCKETS, dtype=torch.int32)
    lo = ((b + BUCKET_BASE) << 18).view(torch.float32)
    big = torch.tensor(2.0)
    xs = [mid, torch.nextafter(mid, big), torch.nextafter(mid, -big), lo, torch.nextafter(lo, torch.tensor(0.0)),
          torch.tensor([0.0, -0.0, 1.0, 1e-30, 5.9e-8]), torch.rand(2_000_000, generator=gen),
          torch.randn(2_000_000, generator=gen) * 10.0 ** (-8 * torch.rand(2_000_000, generator=gen))]
    x = torch.cat([t.float() for t in xs])
    x = torch.cat([x, -x]) if signed else x.abs()
    x = x[x.abs() <= 1]
    k, steps = kernel_search(mid, sp, sn, x)
    want = torch.searchsorted(mid, x, side="left")
    bad = torch.nonzero(k != want).reshape(-1)
    assert bad.numel() == 0, f"x = {float(x[bad[0]])!r}: code {int(k[bad[0]])}, searchsorted {int(want[bad[0]])}"
    assert int(steps.max()) <= (2 if signed else 3), int(steps.max())


# ------------------------------------------------------------------------------------------------ host logic
NO_DECAY = ["bias", "layer_norm.weight", "mlm_ln.weight", "embeddings.weight"]


def _groups(m, wd=0.05):
    """train_muse.py:427-437: weight decay on everything but biases, norms and embeddings"""
    return [{"params": [p for n, p in m.named_parameters() if not any(nd in n for nd in NO_DECAY)], "weight_decay": wd},
            {"params": [p for n, p in m.named_parameters() if any(nd in n for nd in NO_DECAY)], "weight_decay": 0.0}]


UVIT = dict(hidden_size=128, num_attention_heads=2, in_channels=64, block_out_channels=(64,), block_num_heads=1,
            num_res_blocks=1, num_hidden_layers=1, intermediate_size=128, codebook_size=64, vocab_size=65,
            encoder_hidden_size=32, cond_embed_dim=32, micro_cond_encode_dim=8, micro_cond_embed_dim=40, num_vq_tokens=16)
V1 = dict(vocab_size=72, hidden_size=64, num_hidden_layers=1, num_attention_heads=1, intermediate_size=128,
          hidden_dropout=0.0, attention_dropout=0.0, max_position_embeddings=16)
MODELS = {"v1": lambda: MaskGitTransformer(**V1), "uvit": lambda: MaskGiTUViT_v2(**UVIT)}


@pytest.mark.parametrize("kind", list(MODELS))
def test_host_logic_on_the_script_groups(monkeypatch, kind):
    """the 8-bit / 32-bit split at 4096 elements, state shapes and dtypes, one step counter per group, and a table the
    restatement steps like the contract"""
    calls = install(monkeypatch)
    torch.manual_seed(0)
    m = MODELS[kind]()
    groups = _groups(m)
    opt = FusedAdamW8bit(groups, lr=1e-3, betas=(0.9, 0.99), weight_decay=0.05, eps=1e-8)
    gen = torch.Generator().manual_seed(1)
    for _ in range(2):
        for p in m.parameters():
            p.grad = torch.randn(p.shape, generator=gen)
        opt.step()
    assert calls == ["muse_adamw8bit_ema_step"] * 4
    sizes = {p.numel() >= MIN_8BIT_SIZE for p in m.parameters()}
    assert sizes == {True, False}, "the model should have parameters on both paths"
    for gi, g in enumerate(opt.param_groups):
        steps = {id(opt.state[p]["step"]) for p in g["params"]}
        assert len(steps) == 1 and int(opt.state[g["params"][0]]["step"]) == 2, f"group {gi}: one shared step counter"
        for p in g["params"]:
            st = opt.state[p]
            if p.numel() >= MIN_8BIT_SIZE:
                nb = -(-p.numel() // 256)
                assert set(st) == {"state1", "state2", "absmax1", "absmax2", "step"}
                assert st["state1"].dtype == torch.uint8 and st["state1"].shape == p.shape
                assert st["state2"].dtype == torch.uint8 and st["state2"].shape == p.shape
                assert st["absmax1"].dtype == F32 and st["absmax1"].shape == (nb,) and st["absmax2"].shape == (nb,)
                assert bool((st["absmax1"] > 0).all())
            else:
                assert set(st) == {"exp_avg", "exp_avg_sq", "step"}
                assert st["exp_avg"].dtype == F32 and st["exp_avg"].shape == p.shape
    assert opt._plans[0]["table"].shape[1] == 10


@pytest.mark.parametrize("numel,blocks", [(4096, 16), (4100, 17), (2 ** 20, 4096), (4092, None)])
def test_state_layout_by_size(monkeypatch, numel, blocks):
    install(monkeypatch)
    p = torch.nn.Parameter(torch.randn(numel))
    p.grad = torch.randn(numel)
    opt = FusedAdamW8bit([p])
    opt.step()
    st = opt.state[p]
    if blocks is None:
        assert "exp_avg" in st and "absmax1" not in st
    else:
        assert st["absmax1"].shape == (blocks,) and st["absmax2"].shape == (blocks,)
        row = opt._plans[0]["table"][0]
        assert row[8] == st["absmax1"].data_ptr() and row[9] == st["absmax2"].data_ptr()


def test_small_parameters_step_like_fused_adamw(monkeypatch):
    """below 4096 elements the restated pass is FusedAdamW's (restated by cpu_math_ops) value for value"""
    install(monkeypatch)
    gen = torch.Generator().manual_seed(3)
    shapes = [(8,), (64, 32), (4092,)]
    a = [torch.nn.Parameter(torch.randn(s, generator=gen)) for s in shapes]
    b = [torch.nn.Parameter(p.detach().clone()) for p in a]
    oa, ob = FusedAdamW(a, lr=3e-3, weight_decay=0.1), FusedAdamW8bit(b, lr=3e-3, weight_decay=0.1)
    for _ in range(4):
        for pa, pb in zip(a, b):
            pa.grad = torch.randn(pa.shape, generator=gen)
            pb.grad = pa.grad.clone()
        oa.step(), ob.step()
    for pa, pb in zip(a, b):
        assert torch.equal(pa, pb)
        assert torch.equal(oa.state[pa]["exp_avg_sq"], ob.state[pb]["exp_avg_sq"])


def test_tensor_lr_and_parameters_without_grad(monkeypatch):
    calls = install(monkeypatch)
    gen = torch.Generator().manual_seed(4)
    ps = [torch.nn.Parameter(torch.randn(n, generator=gen)) for n in (8192, 16, 4096)]
    for p in ps:
        p.grad = torch.randn(p.shape, generator=gen)
    ps[1].grad = None
    before = ps[1].detach().clone()
    opt = FusedAdamW8bit(ps, lr=torch.tensor([2e-3]))
    opt.step()
    assert calls == ["muse_adamw8bit_ema_step"] and ps[1] not in opt.state and torch.equal(ps[1], before)
    assert len(opt._plans[0]["table"]) == 2
    for bad in (torch.tensor([1e-3], dtype=torch.float64), torch.tensor([1e-3, 2e-3])):
        with pytest.raises(ValueError, match="tensor lr"):
            FusedAdamW8bit(ps, lr=bad)
    opt.param_groups[0]["lr"] = torch.tensor([1e-3], dtype=torch.float64)  # e.g. a scheduler's tensor
    with pytest.raises(ValueError, match="tensor lr"):
        opt.step()
    for kw in (dict(lr=-1.0), dict(betas=(1.0, 0.9)), dict(betas=(0.9, -0.1)), dict(eps=-1.0), dict(weight_decay=-1.0)):
        with pytest.raises(ValueError):
            FusedAdamW8bit(ps, **kw)


# ------------------------------------------------------------------------------------------------ verifier and mutants
NUMELS = [4100, 4096, 4352, 8196]  # partial last blocks and tensors that start mid-way through a global block
LR, WD, B1, B2, EPS, STEP = 1e-2, 0.1, 0.875, 0.99, 1e-8, 5   # 1 - 0.875 is a power of two: see _operands


def _hyper():
    b1, b2 = f32(B1), f32(B2)
    return Hyper(f32(LR), f32(1.0 / (1.0 - b1 ** STEP)), f32(1.0 / (1.0 - b2 ** STEP) ** 0.5), b1, b2, f32(EPS), f32(WD))


@pytest.fixture(scope="module")
def operands():
    return make_operands()


def make_operands():
    """per entry p, g, codes1, codes2, absmax1, absmax2.  Block 1 of every entry starts fresh (codes 0, absmax 0) and
    block 2 holds exact ties: its old m decodes to 0 (code 127), so m = (1 - beta1) g = g / 8 exactly, with one element
    at 1 (absmax 1) and the others on midpoints of the signed map"""
    gen = torch.Generator().manual_seed(11)
    mid1 = midpoints(dynamic_map(True))
    out = []
    for n in NUMELS:
        nb = -(-n // QBLOCK)
        p = torch.randn(n, generator=gen)
        g = torch.randn(n, generator=gen) * 1e-2
        c1 = torch.randint(0, 256, (n,), generator=gen, dtype=torch.uint8)
        c2 = torch.randint(0, 256, (n,), generator=gen, dtype=torch.uint8)
        a1 = torch.rand(nb, generator=gen) * 1e-2 + 1e-3
        a2 = torch.rand(nb, generator=gen) * 1e-4 + 1e-5
        c1[256:512], c2[256:512], a1[1], a2[1] = 0, 0, 0.0, 0.0
        c1[512:768] = 127
        g[512] = 8.0
        g[513:768] = 8.0 * mid1[torch.arange(255) % 255]
        out.append([p, g, c1, c2, a1, a2])
    return out


def _run(ops_in, mutant=None):
    ents = [[t.clone() for t in e] for e in ops_in]
    step8(ents, _maps_buffer("cpu"), _hyper(), mutant)
    return ents


def verify(ops_in, out, ah=None, tol_ulps=4.0, where=None):
    """the 8-bit contract, entry by entry, in fp64 from each entry's decoded old state (`ops_in`, `out`: lists [p, g,
    codes1, codes2, absmax1, absmax2]; `ah`: the step's AdamHyper): p within BOUNDS["adamw.p"] ulps of its terms; each
    absmax, the kernel's own m or v of the block's largest element, within that moment's element bound (BOUNDS["adamw.m"]
    / ["adamw.v"]) in ulps of that element's terms; every code equal to the fp64 code, except where x lies within
    tol_ulps ulps (of its terms) of a midpoint, where either neighbour passes -- but an x exactly on a midpoint must take
    the lower code.  Returns the number of elements in that tolerance zone and the worst absmax1 / absmax2 errors.

    Both tolerances are wider than "absmax within 2 ulps of the fp64 block max" and "x within 4 ulps of a midpoint", on
    purpose: the absmax is not computed on its own but is the fp32 m or v of one element, so it carries that element's
    rounding error (v reaches ~2.8 ulps of its terms on an H100, against the bound of 6 the fp32 AdamW kernel is held
    to), and x = m / absmax inherits the error of m in units of m's terms, which exceed |m| where g and m cancel."""
    h = _hyper()
    ah = ah or AdamHyper(h.lr, h.beta1, h.beta2, h.eps, h.wd, STEP, None)
    where = where or (lambda e: f"entry {e}")
    dev = ops_in[0][0].device
    maps = _maps_buffer(dev).double()
    q = (maps[:256].float(), maps[256:512].float())
    mids = (maps[512:767], maps[768:1023])
    near, worst = 0, [0.0, 0.0]
    bound = (BOUNDS["adamw.m"][0], BOUNDS["adamw.v"][0])
    for e, (inp, res) in enumerate(zip(ops_in, out)):
        p, g, c1, c2, a1, a2 = (t.reshape(-1) for t in inp)
        n = p.numel()
        nb = -(-n // QBLOCK)
        blk = torch.arange(n, device=dev) // QBLOCK
        m0 = (q[0][c1.long()].double() * a1[blk].double()).float()  # the kernel's fp32 decode (exact in fp64 first)
        v0 = (q[1][c2.long()].double() * a2[blk].double()).float()
        ref = adamw_ref(p, g, m0, v0, ah)
        at = lambda b, e=e: f"({where(e)}, block {b} of {nb})"  # noqa: E731
        check_ulps(res[0].reshape(-1), *ref["p"], blk, at, BOUNDS["adamw.p"][0], f"8-bit p, {where(e)}")
        for k, (val, terms) in enumerate((ref["m"], ref["v"])):
            a = val.abs()
            amax, arg = torch.nn.functional.pad(a, (0, nb * QBLOCK - n), value=-1.0).view(nb, QBLOCK).max(1)
            arg = arg + torch.arange(nb, device=dev) * QBLOCK
            got = res[4 + k].reshape(-1).double()
            err = (got - amax).abs() / (terms[arg] * 2.0 ** -24)
            worst[k] = max(worst[k], float(err.max()))
            bad = torch.nonzero(~(err <= bound[k])).reshape(-1)
            assert bad.numel() == 0, (f"absmax{k + 1} of {where(e)} block {int(bad[0])}: {float(got[bad[0]])!r}, fp64 "
                                      f"{float(amax[bad[0]])!r}, {float(err[bad[0]]):.2f} ulps of its terms")
            d = amax[blk]
            pos = torch.where(d > 0, d, torch.ones_like(d))
            x = torch.where(d > 0, val / pos, torch.zeros_like(val))
            xt = torch.where(d > 0, (terms + a) / pos, torch.zeros_like(val)) * 2.0 ** -24
            code = torch.searchsorted(mids[k], x, side="left")
            kc = res[2 + k].reshape(-1).long()
            lo = torch.searchsorted(mids[k], x - tol_ulps * xt, side="left")
            hi = torch.searchsorted(mids[k], x + tol_ulps * xt, side="left")
            tie = torch.isin(x, mids[k])
            zone = (lo != hi) & ~tie
            near += int(zone.sum())
            ok = torch.where(zone, (kc >= lo) & (kc <= hi), kc == code)
            bad = torch.nonzero(~ok).reshape(-1)
            assert bad.numel() == 0, (f"state{k + 1} of {where(e)}: code {int(kc[bad[0]])} at element {int(bad[0])} (block "
                                      f"{int(blk[bad[0]])}), fp64 code {int(code[bad[0]])} for x = {float(x[bad[0]])!r}"
                                      f"{' (an exact tie)' if bool(tie[bad[0]]) else ''}; {bad.numel()} such codes")
    return near, worst


def test_restatement_is_accepted(operands):
    out = _run(operands)
    near, _ = verify(operands, out)
    ties = sum(int(torch.isin(e[1] / 8, midpoints(dynamic_map(True))).sum()) for e in operands)
    assert ties >= 4 * 255
    print(f"\n{near} elements within 4 ulps of a midpoint; {ties} exact ties")


@pytest.mark.parametrize("mutant", MUTANTS)
def test_mutant_is_rejected(operands, mutant):
    with pytest.raises(AssertionError) as info:
        verify(operands, _run(operands, mutant))
    print(f"\n{mutant}: {str(info.value).splitlines()[0][:200]}")


# ------------------------------------------------------------------------------------------------ state dict
def _pair(seed=5):
    torch.manual_seed(seed)
    a = MaskGiTUViT_v2(**UVIT)
    b = MaskGiTUViT_v2(**UVIT)
    b.load_state_dict(a.state_dict())
    return a, b


def test_state_dict_round_trip_continues_bit_identically(monkeypatch):
    install(monkeypatch)
    a, b = _pair()
    oa = FusedAdamW8bit(_groups(a), lr=1e-3)
    gen = torch.Generator().manual_seed(6)
    grads = [[torch.randn(p.shape, generator=gen) for p in a.parameters()] for _ in range(6)]

    def step(m, opt, gs):
        for p, g in zip(m.parameters(), gs):
            p.grad = g.clone()
        opt.step()

    for k in range(3):
        step(a, oa, grads[k])
    b.load_state_dict(a.state_dict())
    ob = FusedAdamW8bit(_groups(b), lr=1e-3)
    ob.load_state_dict(copy.deepcopy(oa.state_dict()))
    for pa, pb in zip(a.parameters(), b.parameters()):
        for k, v in oa.state[pa].items():
            assert ob.state[pb][k].dtype == v.dtype and torch.equal(ob.state[pb][k].cpu(), v.cpu()), k
    for k in range(3, 6):
        step(a, oa, grads[k]), step(b, ob, grads[k])
    for pa, pb in zip(a.parameters(), b.parameters()):
        assert torch.equal(pa, pb)
        for k, v in oa.state[pa].items():
            assert torch.equal(ob.state[pb][k], v), k
    assert int(ob.state[next(b.parameters())]["step"]) == 6


def test_strided_state_loads_dense(monkeypatch):
    """a saved state whose buffers have the right shape but other strides (e.g. from a transpose) loads as dense buffers
    in logical order: the kernel walks them as flat arrays"""
    install(monkeypatch)
    a, b = _pair()
    oa = FusedAdamW8bit(a.parameters(), lr=1e-3)
    gen = torch.Generator().manual_seed(8)
    grads = [[torch.randn(p.shape, generator=gen) for p in a.parameters()] for _ in range(2)]
    for p, g in zip(a.parameters(), grads[0]):
        p.grad = g.clone()
    oa.step()
    sd = copy.deepcopy(oa.state_dict())
    strided = 0
    for st in sd["state"].values():
        for k, t in list(st.items()):
            if k != "step" and t.dim() == 2:
                st[k] = t.t().contiguous().t()  # same values and shape, column-major strides
                strided += 1
    assert strided > 0
    b.load_state_dict(a.state_dict())
    ob = FusedAdamW8bit(b.parameters(), lr=1e-3)
    ob.load_state_dict(sd)
    assert all(t.is_contiguous() for st in ob.state.values() for t in st.values())
    for m, o in ((a, oa), (b, ob)):
        for p, g in zip(m.parameters(), grads[1]):
            p.grad = g.clone()
        o.step()
    for pa, pb in zip(a.parameters(), b.parameters()):
        assert torch.equal(pa, pb)
        for k, v in oa.state[pa].items():
            assert torch.equal(ob.state[pb][k], v), k


def _codes_below_4096(big, small):
    small.update(state1=small["exp_avg"].to(torch.uint8), state2=small["exp_avg_sq"].to(torch.uint8),
                 absmax1=torch.zeros(1), absmax2=torch.zeros(1))
    del small["exp_avg"], small["exp_avg_sq"]


def _fp32_above_4096(big, small):
    big.update(exp_avg=big["state1"].float(), exp_avg_sq=big["state2"].float())
    for k in ("state1", "state2", "absmax1", "absmax2"):
        del big[k]


BAD_STATES = {  # every layout the loader must refuse: an edit of (an 8-bit parameter's state, a 32-bit one's)
    "uint8 codes below 4096": _codes_below_4096,
    "fp32 moments above 4096": _fp32_above_4096,
    "codes of the wrong shape": lambda big, small: big.update(state1=big["state1"].reshape(-1)[:-4]),
    "codes of the wrong dtype": lambda big, small: big.update(state2=big["state2"].float()),
    "absmax of the wrong length": lambda big, small: big.update(absmax1=big["absmax1"][:-1]),
    "absmax of the wrong dtype": lambda big, small: big.update(absmax2=big["absmax2"].double()),
    "moments of the wrong dtype": lambda big, small: small.update(exp_avg=small["exp_avg"].double()),
    "moments of the wrong shape": lambda big, small: small.update(exp_avg_sq=small["exp_avg_sq"][:-4]),
    "a missing absmax": lambda big, small: big.pop("absmax2"),
}


@pytest.mark.parametrize("case", list(BAD_STATES))
def test_load_state_dict_rejects_a_mismatched_layout(monkeypatch, case):
    install(monkeypatch)
    a, b = _pair()
    oa = FusedAdamW8bit(a.parameters(), lr=1e-3)
    for p in a.parameters():
        p.grad = torch.randn(p.shape)
    oa.step()
    sd = copy.deepcopy(oa.state_dict())
    params = list(a.parameters())
    big = next(i for i, p in enumerate(params) if p.numel() >= MIN_8BIT_SIZE)
    small = next(i for i, p in enumerate(params) if p.numel() < MIN_8BIT_SIZE)
    BAD_STATES[case](sd["state"][big], sd["state"][small])
    ob = FusedAdamW8bit(b.parameters(), lr=1e-3)
    with pytest.raises(ValueError, match="FusedAdamW8bit.load_state_dict"):
        ob.load_state_dict(sd)


# ------------------------------------------------------------------------------------------------ train_muse.py
def test_unmodified_train_muse_runs_with_8bit_adamw(monkeypatch, tmp_path):
    """``optimizer.name: 8bit_adamw`` imports bitsandbytes and takes ``bnb.optim.AdamW8bit``: a stand-in module hands it
    FusedAdamW8bit.  The script trains with EMA, saves checkpoint-2, resumes from it; the optimizer state it loads equals
    the saved one, codes still uint8"""
    from tests.train_script_harness import find_script, make_muse_config, run_script

    script = find_script("train_muse.py")
    if script is None:
        pytest.skip("reference training script not available")
    import yaml

    cpu_math_ops.install(monkeypatch, exact=False)
    install(monkeypatch)
    monkeypatch.setenv("ACCELERATE_USE_CPU", "1")
    monkeypatch.setenv("WANDB_MODE", "disabled")
    bnb = types.ModuleType("bitsandbytes")
    bnb.optim = types.SimpleNamespace(AdamW8bit=FusedAdamW8bit)
    monkeypatch.setitem(sys.modules, "bitsandbytes", bnb)
    loaded, made = [], []
    load = FusedAdamW8bit.load_state_dict
    init = FusedAdamW8bit.__init__

    def load_and_record(self, sd):
        load(self, sd)
        loaded.append(copy.deepcopy(self.state_dict()))

    def init_and_record(self, *a, **k):
        init(self, *a, **k)
        made.append(self)

    monkeypatch.setattr(FusedAdamW8bit, "load_state_dict", load_and_record)
    monkeypatch.setattr(FusedAdamW8bit, "__init__", init_and_record)
    cfg, out = make_muse_config(str(tmp_path), steps=2, batch=2, mixed_precision="no", save_every=2, use_ema=True)
    with open(cfg) as f:
        c = yaml.safe_load(f)
    c["optimizer"]["name"] = "8bit_adamw"
    with open(cfg, "w") as f:
        yaml.safe_dump(c, f)
    acc = run_script(script, cfg)
    losses = [v["step_loss"] for v, s in acc.logged if "step_loss" in v]
    assert len(losses) == 2 and all(np.isfinite(losses))
    assert len(made) == 1 and any("state1" in st for st in made[0].state.values())
    saved = torch.load(f"{out}/checkpoint-2/optimizer.bin")
    acc = run_script(script, cfg, extra_cli=("experiment.resume_from_checkpoint=latest", "training.max_train_steps=4"))
    assert [s for v, s in acc.logged if "step_loss" in v] == [3, 4]
    assert len(loaded) == 1
    assert saved["param_groups"] == loaded[0]["param_groups"]
    assert saved["state"].keys() == loaded[0]["state"].keys()
    for i, st in saved["state"].items():
        for k, v in st.items():
            got = loaded[0]["state"][i][k]
            assert got.dtype == v.dtype and torch.equal(got, v), (i, k)
    final = torch.load(f"{out}/checkpoint-4/optimizer.bin")
    assert int(next(iter(final["state"].values()))["step"]) == 4


# ------------------------------------------------------------------------------------------------ operand cache
def _tensors(W, prefix=""):
    out = {}
    for k, v in (W.items() if isinstance(W, dict) else enumerate(W)):
        if torch.is_tensor(v):
            out[prefix + str(k)] = v
        elif isinstance(v, (dict, list)):
            out.update(_tensors(v, f"{prefix}{k}."))
    return out


@pytest.mark.parametrize("kind", list(MODELS))
def test_step_with_model_keeps_the_operand_cache_current(monkeypatch, kind):
    """after each step with model= the operands the next forward reads equal a cache rebuilt from scratch, and fetching
    them re-packs nothing"""
    from open_muse_b200.modeling_transformer import _PackedWeights

    cpu_math_ops.install(monkeypatch, exact=False)
    install(monkeypatch)
    torch.manual_seed(0)
    m = MODELS[kind]()
    with torch.no_grad():
        for p in m.parameters():
            p.add_(0.05 * torch.randn_like(p))
    repacks = []
    if kind == "v1":
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
    ema = EMAModel(list(m.parameters()), decay=0.99)
    opt = FusedAdamW8bit(m.parameters(), lr=1e-2, ema=ema, model=m)
    gen = torch.Generator().manual_seed(1)
    for step in range(3):
        for p in m.parameters():
            p.grad = torch.randn(p.shape, generator=gen)
        repacks.clear()
        opt.step()
        got = current()
        assert repacks == [], f"step {step}: the operands were re-packed after a step with model="
        want = fresh()
        assert got.keys() == want.keys()
        for k in want:
            assert torch.equal(got[k], want[k]), f"step {step}: operand {k} is stale"
    assert [k for k in before if torch.equal(before[k], got[k])] == []


# ------------------------------------------------------------------------------------------------ memory
def test_state_bytes_at_the_uvit_default():
    """MaskGiTUViT_v2 at its defaults (603 M parameters), on the meta device: the moments take at most 2.05 B per
    parameter"""
    with torch.device("meta"):
        m = MaskGiTUViT_v2()
        opt = FusedAdamW8bit(_groups(m))
        n = total = 0
        for g in opt.param_groups:
            for p in g["params"]:
                n += p.numel()
                total += sum(t.numel() * t.element_size() for t in opt._init_state(p).values())
    assert n > 600e6
    print(f"\n{n / 1e6:.1f} M parameters, {total / n:.4f} B of optimizer state per parameter (FusedAdamW: 8)")
    assert total / n <= 2.05
