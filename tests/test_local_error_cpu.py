"""The bounds of tests/local_error.py catch subtly wrong kernels: on the CPU, each kernel is emulated in fp64 with bf16
rounding at its rounding points (inputs; the P and dS operands; outputs).  check_local() accepts the emulation and
rejects each mutant below -- defects a tiled kernel makes (a ragged tail tile, a missing key or query row, one scaled
tile) that the whole-tensor rel-L2 checks of tests/test_kernels_gpu.py pass.  Each mutant's whole-tensor rel-L2 is
printed next to the tolerance of that old check."""
import functools
import math

import pytest
import torch

from tests.local_error import (BOUNDS, attn_rows, balanced_rows, ce_fwd_ref, ce_inputs, check_abs, check_local, gemm_rows,
                               gemm_tiles, rows)

F64 = torch.float64


def _bf(t):
    return t.to(torch.bfloat16).to(F64)


def _randn(shape, seed):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed), dtype=F64)


def _whole(out, ref):
    return float((out - ref).norm() / ref.norm())


# ------------------------------------------------------------------------------------------------------------ attention
AB, AH, AS, AD = 4, 8, 257, 64  # the benchmark's sequence length; R = 52-row owned tiles, the last one ragged


@functools.lru_cache(maxsize=None)
def _attn(mutant=None):
    """(emulated, reference) dicts of o, dq, dk, dv as [B, nh, S, hd]."""
    scale = AD ** -0.5
    q, k, v, do = (_bf(_randn((AB, AH, AS, AD), s)) for s in (1, 2, 3, 4))
    s = q @ k.transpose(-1, -2) * scale
    lse = torch.logsumexp(s, -1, keepdim=True)
    p = torch.exp(s - lse)
    dp = do @ v.transpose(-1, -2)
    ref = {"o": p @ v}
    dd = (do * ref["o"]).sum(-1, keepdim=True)
    ds = p * (dp - dd)
    ref.update(dq=ds @ k * scale, dk=ds.transpose(-1, -2) @ q * scale, dv=p.transpose(-1, -2) @ do)
    # the kernels: P against the row maximum rounded to bf16 for P V (l is the unrounded sum), dS rounded to bf16
    m = s.amax(-1, keepdim=True)
    pm = torch.exp(s - m)
    o = (_bf(pm) @ v) / pm.sum(-1, keepdim=True)
    d_emu = dd.clone()
    if mutant == "O row 256 x 1.05":
        o[:, :, 256] *= 1.05
    if mutant == "dK/dV reads D = 0 for q row 256":
        d_emu[:, :, 256] = 0
    ds_q = _bf(p * (dp - dd))       # dQ kernel: its own D
    ds_kv = _bf(p * (dp - d_emu))   # dK/dV kernel: D from the dQ kernel's sweep
    pt = _bf(p)
    if mutant == "dK/dV missing q row 256":
        ds_kv[:, :, 256] = 0
        pt[:, :, 256] = 0
    emu = {"o": o, "dq": ds_q @ k * scale, "dk": ds_kv.transpose(-1, -2) @ q * scale, "dv": pt.transpose(-1, -2) @ do}
    if mutant == "dQ of the last q tile missing key 256":
        last = (AS - 1) // balanced_rows(AS) * balanced_rows(AS)
        emu["dq"][:, :, last:] -= ds_q[:, :, last:, 256:257] * k[:, :, 256:257] * scale
    if mutant == "one (b, h) tile of dV x 1.1":
        R = balanced_rows(AS)
        emu["dv"][2, 5, 2 * R:3 * R] *= 1.1
    return {n: _bf(t) for n, t in emu.items()}, ref


def _tok(t):
    return t.permute(0, 2, 1, 3).reshape(AB * AS, AH * AD)


def _check_attn(emu, ref, name):
    check_local(_tok(emu[name]), _tok(ref[name]), attn_rows(AB, AH, AS, AD), *BOUNDS[f"attn.{name}"], f"attn.{name}")


def test_attention_emulation_is_accepted():
    emu, ref = _attn()
    for name in ("o", "dq", "dk", "dv"):
        _check_attn(emu, ref, name)


@pytest.mark.parametrize("mutant,output,old_tol", [
    ("dK/dV reads D = 0 for q row 256", "dk", 1.5e-2),
    ("O row 256 x 1.05", "o", 8e-3),
    ("dQ of the last q tile missing key 256", "dq", 1.5e-2),
    ("dK/dV missing q row 256", "dk", 1.5e-2),
    ("dK/dV missing q row 256", "dv", 1.5e-2),
    ("one (b, h) tile of dV x 1.1", "dv", 1.5e-2),
])
def test_attention_mutant_is_rejected(mutant, output, old_tol):
    emu, ref = _attn(mutant)
    print(f"\n{mutant}: {output} whole-tensor rel-L2 {_whole(emu[output], ref[output]):.2e} (old tolerance {old_tol:.1e})")
    with pytest.raises(AssertionError, match="worst group error"):
        _check_attn(emu, ref, output)


# ------------------------------------------------------------------------------------------------------------ GEMM
GM, GN, GK = 2056, 512, 2048  # 17 m tiles, the last one 8 rows


@functools.lru_cache(maxsize=None)
def _gemm(mutant=None):
    a, b = _bf(_randn((GM, GK), 5)), _bf(_randn((GN, GK), 6))
    ref = a @ b.t()
    acc = ref.clone()
    if mutant == "8-row M tail tile x 1.05":
        acc[2048:] *= 1.05
    if mutant == "a 128 x 128 tile missing its last K block":
        acc[384:512, 128:256] -= a[384:512, GK - 64:] @ b[128:256, GK - 64:].t()
    return _bf(acc), ref


def test_gemm_emulation_is_accepted():
    out, ref = _gemm()
    check_local(out, ref, gemm_rows(GM, GN), *BOUNDS["gemm.bf16"], "gemm.bf16 rows")
    check_local(out, ref, gemm_tiles(GM, GN, 256), *BOUNDS["gemm.bf16"], "gemm.bf16 tiles")


@pytest.mark.parametrize("mutant", ["8-row M tail tile x 1.05", "a 128 x 128 tile missing its last K block"])
def test_gemm_mutant_is_rejected(mutant):
    out, ref = _gemm(mutant)
    print(f"\n{mutant}: whole-tensor rel-L2 {_whole(out, ref):.2e} (old tolerance 6.0e-03)")
    for groups in (gemm_rows(GM, GN), gemm_tiles(GM, GN, 256)):
        with pytest.raises(AssertionError, match="worst group error"):
            check_local(out, ref, groups, *BOUNDS["gemm.bf16"], "gemm.bf16")


# ------------------------------------------------------------------------------------------------------------ norm
def _norm(mutant=None):
    x = _bf(_randn((77, 1000), 7))
    w = 1 + 0.1 * _randn((1000,), 8)
    mu = x.mean(-1, keepdim=True)
    ref = (x - mu) * torch.rsqrt((x - mu).pow(2).mean(-1, keepdim=True) + 1e-6) * w
    out = ref.clone()
    if mutant:
        out[40] *= 1.04
    return _bf(out), ref


def test_norm_emulation_is_accepted():
    check_local(*_norm(), rows(77), *BOUNDS["norm.y_bf16"], "norm.y_bf16")


def test_norm_mutant_is_rejected():
    out, ref = _norm("one row x 1.04")
    print(f"\none row x 1.04: whole-tensor rel-L2 {_whole(out, ref):.2e} (old tolerance 5.0e-03)")
    with pytest.raises(AssertionError, match="worst group error"):
        check_local(out, ref, rows(77), *BOUNDS["norm.y_bf16"], "norm.y_bf16")


# ------------------------------------------------------------------------------------------------------------ add_norm_mod_bwd
NB, NR, NH = 3, 77, 520  # a warp's 8 rows cross a sample (77 % 8 != 0)


def _anm_bwd(mutant=None):
    """da (bf16 output) and dmod (fp32) of add_norm_mod_bwd with LayerNorm and a per-sample modulation"""
    T = NB * NR
    x = _randn((T, NH), 9)
    w = (1 + 0.1 * _randn((NH,), 10)).requires_grad_(True)
    mod = (0.3 * _randn((NB, 2 * NH), 11)).requires_grad_(True)
    xr = x.clone().requires_grad_(True)
    dy, dro = _bf(_randn((T, NH), 12)), _randn((T, NH), 13)
    mu = xr.mean(-1, keepdim=True)
    n = (xr - mu) * torch.rsqrt((xr - mu).pow(2).mean(-1, keepdim=True) + 1e-6) * w
    y = (n.view(NB, NR, NH) * (1 + mod[:, None, :NH]) + mod[:, None, NH:]).view(T, NH)
    ((y * dy).sum() + (xr * dro).sum()).backward()
    dmod = mod.grad.clone()
    if mutant:  # the flush of sample 1 misses the sample's last row
        r = 2 * NR - 1
        dmod[1, :NH] -= dy[r] * n[r].detach()
        dmod[1, NH:] -= dy[r]
    return {"da": (_bf(xr.grad), xr.grad), "dmod": (dmod.float().double(), mod.grad)}


def _dmod_groups():
    return rows(2 * NB, "sample, scale / shift half")


def test_add_norm_mod_bwd_emulation_is_accepted():
    out = _anm_bwd()
    check_local(*out["da"], rows(NB * NR), *BOUNDS["anm.da_bf16"], "anm.da_bf16")
    check_local(out["dmod"][0].view(2 * NB, NH), out["dmod"][1].view(2 * NB, NH), _dmod_groups(), *BOUNDS["anm.dmod"],
                "anm.dmod")


def test_add_norm_mod_bwd_mutant_is_rejected():
    out, ref = _anm_bwd("dmod of one sample missing its last row")["dmod"]
    print(f"\ndmod of one sample missing its last row: whole-tensor rel-L2 {_whole(out, ref):.2e} (old tolerance 1.0e-04)")
    with pytest.raises(AssertionError, match="worst group error"):
        check_local(out.view(2 * NB, NH), ref.view(2 * NB, NH), _dmod_groups(), *BOUNDS["anm.dmod"], "anm.dmod")


# ------------------------------------------------------------------------------------------------------------ CE forward
CR, CV, CLD = 389, 2025, 2048  # the real vocabulary: column 2024 is the scalar tail of the kernel's 8-wide loop


def _ce_fwd(ls, mutant=None):
    """(lse, row loss) of an fp32 emulation of ce_fwd (max, sum of exp, log and the logit sum in fp32) and the fp64
    reference"""
    logits, labels = ce_inputs(CR, CV, CLD, 15)
    x = logits[:, :CV - 1] if mutant == "tail column V - 1 dropped from the LSE" else logits[:, :CV]
    m = x.amax(-1)
    lse = m + torch.exp(x - m[:, None]).sum(-1).log()
    z = logits[:, :CV]
    div = CV - 1 if mutant == "smoothing term divides by V - 1" else CV
    zy = z.gather(1, labels.clamp_min(0)[:, None])[:, 0]
    loss = (1 - ls) * (lse - zy) + ls * (lse - z.sum(-1) / div)
    loss = torch.where(labels != -100, loss, torch.zeros_like(loss))
    return (lse, loss), ce_fwd_ref(logits, labels, CV, ls)


@pytest.mark.parametrize("ls", [0.0, 0.1])
def test_ce_fwd_emulation_is_accepted(ls):
    (lse, loss), (lse_ref, loss_ref) = _ce_fwd(ls)
    check_abs(lse, lse_ref, lambda r: f"row {r}", BOUNDS["ce.lse"][0], "ce.lse")
    check_abs(loss, loss_ref, lambda r: f"row {r}", BOUNDS["ce.loss"][0], "ce.loss")


@pytest.mark.parametrize("mutant,output", [("tail column V - 1 dropped from the LSE", 0),
                                           ("smoothing term divides by V - 1", 1)])
def test_ce_fwd_mutant_is_rejected(mutant, output):
    out, ref = _ce_fwd(0.1, mutant)
    key = ("ce.lse", "ce.loss")[output]
    print(f"\n{mutant}: {key} whole-tensor rel-L2 {_whole(out[output].double(), ref[output]):.2e}, mean loss error "
          f"{abs(float(out[1][ref[1] != 0].double().mean() - ref[1][ref[1] != 0].mean())):.2e}")
    with pytest.raises(AssertionError, match="worst absolute error"):
        check_abs(out[output], ref[output], lambda r: f"row {r}", BOUNDS[key][0], key)


def test_bf16_bounds_stay_below_the_mutation_floor():
    """bf16 outputs: no group bound above 2e-2, the level below which the mutants above are rejected"""
    bf16_outputs = ["attn.o", "attn.dq", "attn.dk", "attn.dv", "gemm.bf16", "gemm.resadd", "norm.y_bf16", "norm2.da",
                    "glu_norm.y", "glu_norm.dab", "ce.dlogits", "anm.y", "anm.da_bf16", "dwconv.y", "grn.out", "grn.dx"]
    assert all(BOUNDS[k][0] <= 2e-2 for k in bf16_outputs), {k: BOUNDS[k] for k in bf16_outputs}
    assert math.isfinite(sum(b for pair in BOUNDS.values() for b in pair))
