"""Every row, tile and head of the bf16 training kernels against an fp64 reference (tests/local_error.py).

References are fp64 on the GPU, computed from the operands exactly as the kernel receives them (bf16-rounded inputs);
they round only where a kernel's contract rounds (the bf16 GELU output of GRN, the GLU product of the fused GLU + norm,
the bf16 conv output before Norm2D).  Inputs are structured so that a local defect shows as a large error of one group:
planted attention rows (dominant first / last key, a running maximum that rises by 6 and by 10 log2 units from one kv
tile to the next, large scores in the rows a CTA computes for its neighbour), GEMM operands scaled by a distinct power
of two per row / column tile, norm rows with a large mean, a constant row and an outlier, special cross-entropy rows.
Shapes are the smallest that reach each path: ragged tail tiles, persistent GEMM CTAs that take a second and third tile,
norm-backward warps that take a second and third row, warps of add_norm_mod_bwd whose 8 rows cross a sample."""
import math

import pytest
import torch

from open_muse_b200 import ops
from tests.local_error import (ATTN_LSE_ABS, BOUNDS, Groups, Local, attn_rows, balanced_rows, ce_fwd_ref, ce_inputs,
                               check_abs, check_local, gemm_rows, gemm_tiles)
from tests.local_error import rows as by_row
from tests.test_dropout_cpu import keep_scale, unpack_bits
from tests.test_gemm_epilogue_gpu import EPI_SPLITK_F32, _gemm

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16
F64 = torch.float64

_worst = {}  # bound key -> (Local, case) with the largest group error seen
_lse_worst = [0.0, None]  # largest |lse - lse_ref| and its case


def _check(key, out, ref, groups, case):
    res = check_local(out, ref, groups, *BOUNDS[key], f"{key} {case}")
    if key not in _worst or res.worst > _worst[key][0].worst:
        _worst[key] = (res, case)
    return res


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst per-group error per kernel output (bound; group; whole-tensor rel-L2 of that case):")
    for key in BOUNDS:
        if key in _worst:
            r, case = _worst[key]
            print(f"  {key:14s} {r.worst:.3e} (bound {BOUNDS[key][0]:.1e}, elem {r.elem:.3e} / {BOUNDS[key][1]:.1e}) "
                  f"{case} {r.where}; whole {r.whole:.3e}")
    print(f"  attn.lse       max |lse - lse_ref| {_lse_worst[0]:.3e} (bound {ATTN_LSE_ABS:.1e}) {_lse_worst[1]}")


def _randn(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g) * scale


# ------------------------------------------------------------------------------------------------------------ attention
def _heads(t, B, S, nh, hd):
    return t.reshape(B, S, nh, hd).permute(0, 2, 1, 3)


def _plant_q(q4, k4, scale, Sq, Skv):
    """q4 [B, nh, Sq, hd] (fp32, scaled per head), k4 [B, nh, Skv, hd] (bf16-exact): planted rows, in place."""
    def aim(row, key, score):  # the row's score with `key` becomes `score`
        kk = k4[:, :, key]
        q4[:, :, row] = (score / ((kk * kk).sum(-1) * scale))[..., None] * kk

    def rise(row, key, log2_units):  # the row's maximum over kv tile 1 exceeds that over kv tile 0 by log2_units
        kk = k4[:, :, key]
        c0 = (k4[:, :, :64] * kk[:, :, None]).sum(-1).amax(-1) * scale
        cj = (kk * kk).sum(-1) * scale
        t = log2_units * math.log(2) / (cj - c0).clamp_min(0.5)
        q4[:, :, row] = t[..., None] * kk

    aim(0, Skv - 1, 10.0)        # dominant key in the ragged last kv tile
    aim(1, 0, 10.0)              # dominant key 0
    aim(Sq - 1, Skv - 1, 10.0)   # last q row (the ragged q tile) on the last key
    if Skv > 64 + 8 and Sq > 4:
        rise(2, 64 + 5, 6.0)     # lazy rescale: the reference point stays (rise < 8)
        rise(3, 64 + 7, 10.0)    # lazy rescale: the reference point moves
    R = balanced_rows(Sq)
    if R < 64:                   # rows of owned tile t >= 1 that the CTA of tile t - 1 also computes (and discards)
        for t in range(1, -(-Sq // R)):
            if t * R + 1 < Sq - 1:
                aim(t * R + 1, (7 * t) % Skv, 60.0)


def _attention_case(B, nh, Sq, Skv, hd, drop):
    H = nh * hd
    scale = 1.0 / math.sqrt(hd)
    cross = Sq != Skv
    case = f"(B {B}, nh {nh}, Sq {Sq}, Skv {Skv}, hd {hd}{', dropout' if drop else ''})"
    if cross:
        qbuf, kvbuf = _randn((B * Sq, H), 1).to(BF).float(), _randn((B * Skv, 2 * H), 2).to(BF).float()
        qcol, kbuf, kcol, vcol = 0, kvbuf, 0, H
    else:  # one [T, 3H] projection, q / k / v are column slices (the layout of training)
        qbuf = kbuf = _randn((B * Sq, 3 * H), 1).to(BF).float()
        qcol, kcol, vcol = 0, H, 2 * H
    k4 = _heads(kbuf[:, kcol:kcol + H], B, Skv, nh, hd)
    q4 = _heads(qbuf[:, qcol:qcol + H], B, Sq, nh, hd).clone()
    q4 *= torch.tensor([0.25, 1.0, 4.0]).repeat(B * nh)[:B * nh].view(B, nh, 1, 1)  # near-uniform .. peaked softmax
    _plant_q(q4, k4, scale, Sq, Skv)
    qbuf[:, qcol:qcol + H] = q4.permute(0, 2, 1, 3).reshape(B * Sq, H)
    qbuf = qbuf.to(BF).to(DEV)
    kvdev = qbuf if not cross else kvbuf.to(BF).to(DEV)
    q, k, v = qbuf[:, qcol:qcol + H], kvdev[:, kcol:kcol + H], kvdev[:, vcol:vcol + H]
    do = _randn((B * Sq, H), 3).to(BF).to(DEV)

    dropout = (0.1, torch.tensor([-1234567890123456789], dtype=torch.int64, device=DEV), 7) if drop else None
    res = ops.attn_fwd(q, k, v, B, nh, Sq, Skv, scale, head_dim=hd, dropout=dropout)
    o, lse = res[0], res[1]
    dq = torch.full((B * Sq, H), float("nan"), dtype=BF, device=DEV)
    dk = torch.full((B * Skv, H), float("nan"), dtype=BF, device=DEV)
    dv = torch.full((B * Skv, H), float("nan"), dtype=BF, device=DEV)
    ops.attn_bwd(q, k, v, o, do, lse, dq, dk, dv, B, nh, Sq, Skv, scale, head_dim=hd,
                 dropout=(0.1, res[2]) if drop else None)
    torch.cuda.synchronize()

    qd, kd, vd = (_heads(t.to(F64), B, S, nh, hd).clone().requires_grad_(True) for t, S in ((q, Sq), (k, Skv), (v, Skv)))
    s = (qd @ kd.transpose(-1, -2)) * scale
    p = s.softmax(-1)
    if drop:
        p = p * (unpack_bits(res[2].cpu(), Skv).to(DEV).to(F64) * keep_scale(0.1))
    od = p @ vd
    od.backward(_heads(do.to(F64), B, Sq, nh, hd))
    lse_ref = torch.logsumexp(s.detach(), -1)

    tok = lambda t, S: t.detach().permute(0, 2, 1, 3).reshape(B * S, H)  # noqa: E731
    gq, gkv = attn_rows(B, nh, Sq, hd), attn_rows(B, nh, Skv, hd)
    _check("attn.o", o, tok(od, Sq), gq, case)
    _check("attn.dq", dq, tok(qd.grad, Sq), gq, case)
    _check("attn.dk", dk, tok(kd.grad, Skv), gkv, case)
    _check("attn.dv", dv, tok(vd.grad, Skv), gkv, case)
    lse_err = (lse.to(F64) - lse_ref).abs()
    if float(lse_err.max()) > _lse_worst[0]:
        _lse_worst[:] = [float(lse_err.max()), case]
    assert float(lse_err.max()) <= ATTN_LSE_ABS, (case, float(lse_err.max()), divmod(int(lse_err.argmax()), Sq))


@pytest.mark.parametrize("B,nh,Sq,Skv,hd", [
    (2, 3, 257, 257, 64), (2, 3, 256, 256, 64), (2, 3, 65, 65, 64), (2, 3, 129, 129, 48), (2, 3, 321, 321, 64),
    (2, 3, 257, 257, 48), (2, 3, 256, 77, 64), (3, 2, 130, 5, 48),
    (8, 8, 257, 257, 64),  # the benchmark's per-sample layout: QKV column slices of one [T, 1536] projection
])
def test_attention_local(B, nh, Sq, Skv, hd):
    _attention_case(B, nh, Sq, Skv, hd, drop=False)


def test_attention_dropout_local():
    _attention_case(2, 2, 257, 257, 64, drop=True)


# ------------------------------------------------------------------------------------------------------------ GEMM
GEMM_EPI = {"bf16": ops.EPI_BF16, "f32": ops.EPI_F32, "resadd": ops.EPI_RESADD_F32, "splitk": EPI_SPLITK_F32,
            "atomic": ops.EPI_ATOMIC_F32}


def _tile_pow2(n, tile):
    """2^(t - T/2) for the tile t of each of n indices: a distinct power of two per tile"""
    t = torch.arange(n) // tile
    return torch.pow(2.0, (t - (-(-n // tile)) // 2).double()).float()


@pytest.mark.parametrize("epi", list(GEMM_EPI))
@pytest.mark.parametrize("majors", [(0, 0), (0, 1), (1, 1), (1, 0)])
@pytest.mark.parametrize("M,N,K,ldc", [(200, 72, 136, 80), (2056, 200, 200, 208), (200, 2025, 200, 2048),
                                       (2056, 2024, 136, 2048)])
def test_gemm_local(M, N, K, ldc, majors, epi):
    a_mn, b_mn = majors
    BN = 256 if N >= 256 else 128
    A = (_randn((M, K), 11) * _tile_pow2(M, 128)[:, None]).to(BF)
    Bm = (_randn((N, K), 12) * _tile_pow2(N, BN)[:, None]).to(BF)
    ref = A.to(DEV, F64) @ Bm.to(DEV, F64).t()
    A_dev = (A.t().contiguous() if a_mn else A).to(DEV)
    if b_mn:  # [K, N] in a pitched buffer: TMA needs 16-byte row strides
        Bt = torch.zeros(K, -(-N // 8) * 8, dtype=BF)
        Bt[:, :N] = Bm.t()
        B_dev = Bt.to(DEV)[:, :N]
    else:
        B_dev = Bm.to(DEV)
    dt = BF if epi == "bf16" else torch.float32
    mag = (_tile_pow2(M, 128)[:, None] * _tile_pow2(N, BN)[None] * math.sqrt(K)).to(DEV)
    base = torch.full((M, ldc), 7.0, device=DEV)  # pad columns past N must keep it
    res = None
    if epi == "resadd":
        res = torch.zeros(M, ldc, device=DEV)
        res[:, :N] = _randn((M, N), 13).to(DEV) * mag
        ref = ref + res[:, :N].to(F64)
    if epi == "atomic":  # accumulates into a non-zero C
        base[:, :N] = _randn((M, N), 14).to(DEV) * mag
        ref = ref + base[:, :N].to(F64)
    tiles = -(-M // 128) * -(-N // BN)
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    runs = [0]
    if tiles > 32:  # a persistent grid of `grid` CTAs: 2-3 tiles per CTA and a remainder
        grid = max(16, math.ceil(tiles / 2.5))
        grid += 1 if tiles % grid == 0 else 0
        runs.append(nsm - grid)
    key = f"gemm.{epi}"
    if N % (8 if epi == "bf16" else 4) and epi != "atomic":
        # the TMA-store epilogues write whole 16-byte units: an N they cannot clip is refused, C left as it was
        C = base.clone().to(dt)
        with pytest.raises(ops._lib.MuseB200Error, match="must be a multiple of"):
            _gemm(GEMM_EPI[epi], A_dev, B_dev, C, res, M, N, K, ldc, a_mn, b_mn)
        assert torch.equal(C, base.to(dt))
        return
    try:
        for reserve in runs:
            ops.reserve_sms(reserve)
            C = base.clone().to(dt)
            _gemm(GEMM_EPI[epi], A_dev, B_dev, C, res, M, N, K, ldc, a_mn, b_mn)
            torch.cuda.synchronize()
            case = f"(M {M}, N {N}, K {K}, ldc {ldc}, majors {majors}, {tiles} tiles, reserved SMs {reserve})"
            _check(key, C, ref, gemm_rows(M, N), case)
            _check(key, C, ref, gemm_tiles(M, N, BN), case)
            assert bool((C[:, N:] == 7.0).all()), case
    finally:
        ops.reserve_sms(0)


# ------------------------------------------------------------------------------------------------------------ norms
NORM_ROWS = 2 * 4224 + 77  # past the 528-CTA x 8-warp backward grid: every warp takes two rows, some three


def _norm_input(rows, H, seed, rms):
    x = _randn((rows, H), seed)
    x[5] = 300.0 + 0.05 * _randn((H,), seed + 1)  # large mean, small spread
    x[rows // 2] = 0.75                            # constant row: LayerNorm rstd = 1 / sqrt(eps)
    x[rows - 1] = 0.01 * _randn((H,), seed + 2)
    x[rows - 1, H // 3] = 10.0                     # one element 1e3 x the others
    return x


def _norm_ref(x, w, eps, rms):
    if rms:
        return x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps) * w
    mu = x.mean(-1, keepdim=True)
    return (x - mu) * torch.rsqrt((x - mu).pow(2).mean(-1, keepdim=True) + eps) * w


@pytest.mark.parametrize("H,rms,xdt", [(512, 0, torch.float32), (1000, 1, BF), (1024, 0, BF), (2048, 0, BF),
                                       (4096, 1, torch.float32)])
def test_norm_local(H, rms, xdt):
    rows, eps = NORM_ROWS, 1e-6
    case = f"(rows {rows}, H {H}, rms {rms}, x {xdt})"
    x = _norm_input(rows, H, 1, rms).to(xdt).to(DEV)
    w = (1 + 0.1 * _randn((H,), 3)).to(DEV)
    y, stats = ops.norm_fwd(x, w, eps, BF, rms=rms)
    dy = _randn((rows, H), 4).to(BF).to(DEV)
    dres = _randn((rows, H), 5).to(DEV)
    dx, dw = ops.norm_bwd(dy, x, w, stats, torch.float32, dres=dres, rms=rms, want_dw=True)
    dw_atomic = torch.zeros(H, device=DEV)
    dx2 = ops.norm_bwd(dy, x, w, stats, torch.float32, dw=dw_atomic, dres=dres, rms=rms)
    torch.cuda.synchronize()
    xd, wd = x.to(F64).requires_grad_(True), w.to(F64).requires_grad_(True)
    yr = _norm_ref(xd, wd, eps, rms)
    yr.backward(dy.to(F64))
    _check("norm.y_bf16", y, yr, by_row(rows), case)
    _check("norm.dx", dx, xd.grad + dres.to(F64), by_row(rows), case)
    _check("norm.dx", dx2, xd.grad + dres.to(F64), by_row(rows), case + " atomic dw")
    _check("norm.dw", dw, wd.grad, by_row(H, "column"), case)
    _check("norm.dw", dw_atomic, wd.grad, by_row(H, "column"), case + " atomic dw")


@pytest.mark.parametrize("H,rms1", [(1024, 0), (512, 1)])
def test_norm2_bwd_local(H, rms1):
    rows, eps = NORM_ROWS, 1e-6
    case = f"(rows {rows}, H {H}, rms1 {rms1})"
    a = _norm_input(rows, H, 6, rms1).to(BF).to(DEV)
    res = _randn((rows, H), 7).to(DEV)
    w1, w2 = (1 + 0.1 * _randn((H,), 8)).to(DEV), (1 + 0.1 * _randn((H,), 9)).to(DEV)
    x2, h2, st = ops.norm2_fwd(a, res, w1, w2, eps, rms1=rms1, rms2=0)
    d_h2, dres = _randn((rows, H), 10).to(BF).to(DEV), _randn((rows, H), 11).to(DEV)
    dx2, d_a, dw1, dw2 = ops.norm2_bwd(d_h2, x2, w2, dres, a, w1, st, rms1=rms1, rms2=0)
    torch.cuda.synchronize()
    ad, w1d, w2d = (t.to(F64).requires_grad_(True) for t in (a, w1, w2))
    x2r = res.to(F64) + _norm_ref(ad, w1d, eps, rms1)
    x2r.retain_grad()
    h2r = _norm_ref(x2r, w2d, eps, 0)
    ((h2r * d_h2.to(F64)).sum() + (x2r * dres.to(F64)).sum()).backward()
    _check("norm.y_bf16", h2, h2r, by_row(rows), case + " h2")
    _check("norm2.dx2", dx2, x2r.grad, by_row(rows), case)
    _check("norm2.da", d_a, ad.grad, by_row(rows), case)
    _check("norm2.dw", dw1, w1d.grad, by_row(H, "column"), case + " dw1")
    _check("norm2.dw", dw2, w2d.grad, by_row(H, "column"), case + " dw2")


def _bf16_st(t):
    """t rounded to bf16 in value, differentiated as the unrounded t (the kernels' rounding points)"""
    return t + (t.to(BF).to(t.dtype) - t).detach()


@pytest.mark.parametrize("rms", [0, 1])
def test_glu_norm_local(rms):
    rows, I, eps = 3277, 2048, 1e-6
    case = f"(rows {rows}, I {I}, rms {rms})"
    ab = _randn((rows, 2 * I), 12).to(BF).to(DEV)
    w = (1 + 0.1 * _randn((I,), 13)).to(DEV)
    y, stats = ops.norm_fwd(ab, w, eps, BF, act=2, rms=rms)
    dy = _randn((rows, I), 14).to(BF).to(DEV)
    dab, dw = ops.norm_bwd(dy, ab, w, stats, BF, act=2, rms=rms, want_dw=True)
    torch.cuda.synchronize()
    abd, wd = ab.to(F64).requires_grad_(True), w.to(F64).requires_grad_(True)
    v = _bf16_st(_bf16_st(torch.nn.functional.gelu(abd[:, :I])) * abd[:, I:])  # v = bf16(bf16(gelu(a)) * b)
    yr = _norm_ref(v, wd, eps, rms)
    yr.backward(dy.to(F64))
    _check("glu_norm.y", y, yr, by_row(rows), case)
    _check("glu_norm.dab", dab, abd.grad, by_row(2 * rows, "row, half"), case)
    _check("glu_norm.dw", dw, wd.grad, by_row(I, "column"), case)


# ------------------------------------------------------------------------------------------------------------ CE
@pytest.mark.parametrize("ls", [0.0, 0.1])
@pytest.mark.parametrize("weighted", [False, True])
def test_ce_bwd_local(ls, weighted):
    rows, V, ld = 389, 2025, 2048
    case = f"(rows {rows}, V {V}, ld {ld}, label smoothing {ls}, row_scale {weighted})"
    g = torch.Generator().manual_seed(15)
    logits = torch.zeros(rows, ld)
    logits[:, :V] = torch.randn(rows, V, generator=g) * 2
    labels = torch.randint(0, V, (rows,), generator=g)
    labels[torch.rand(rows, generator=g) < 0.3] = -100
    labels[0], labels[1], labels[rows - 1] = 0, V - 1, V - 1
    logits[2, 5], labels[2] = 60.0, 7          # one +60 logit, labelled elsewhere
    logits[3, 9], labels[3] = 60.0, 9          # one +60 logit on the label
    logits[4, :V], labels[4] = 1.5, 11         # all-equal row
    labels[6] = labels[rows - 2] = -100
    logits, labels = logits.to(BF).to(DEV), labels.to(DEV)
    row_scale = (torch.rand(rows, generator=g) + 0.1).to(DEV) if weighted else None
    out, ws = ops.ce_fwd(logits, labels, V, ls)
    dloss = torch.tensor([0.5], device=DEV)
    dl = ops.ce_bwd(logits, labels, ws, dloss, out, V, ls, row_scale=row_scale)
    torch.cuda.synchronize()
    valid = labels != -100
    x = logits[:, :V].to(F64)
    ref = torch.softmax(x, -1) - ls / V
    ref[valid.nonzero()[:, 0], labels[valid]] -= 1 - ls
    ref *= 0.5 * (row_scale.to(F64)[:, None] if weighted else 1.0 / float(valid.sum()))
    ref[~valid] = 0
    _check("ce.dlogits", dl[:, :V], ref, by_row(rows), case)
    assert bool((dl[:, V:] == 0).all()) and bool((dl[~valid] == 0).all()), case  # exact zeros


def _check_abs(key, out, ref, case):
    res = check_abs(out, ref, lambda r: f"row {r}", BOUNDS[key][0], f"{key} {case}")
    if key not in _worst or res.worst > _worst[key][0].worst:
        _worst[key] = (res, case)


def _check_rel(key, out, ref, case):
    err = abs(float(out) - float(ref)) / abs(float(ref))
    assert err <= BOUNDS[key][0], f"{key} {case}: relative error {err:.3e} (bound {BOUNDS[key][0]:.1e})"
    if key not in _worst or err > _worst[key][0].worst:
        _worst[key] = (Local(err, "-", 0.0, "-", err, "-", err), case)


@pytest.mark.parametrize("ls", [0.0, 0.1])
@pytest.mark.parametrize("V,ld", [(2025, 2048), (1024, 1024), (8192, 8192)])
def test_ce_fwd_local(V, ld, ls):
    """every row's log-sum-exp and loss (U-ViT v2 weights the row losses directly), the mean, the valid count and the
    row_scale-weighted loss as uvit_v2_train.TailFn forms it; V = 2025 sends column 2024 through the scalar tail loop"""
    rows = 389
    case = f"(rows {rows}, V {V}, ld {ld}, label smoothing {ls})"
    logits, labels = ce_inputs(rows, V, ld, 15)
    logits, labels = logits.to(BF).to(DEV), labels.to(DEV)
    out, ws = ops.ce_fwd(logits, labels, V, ls)
    lw = (torch.rand(rows, generator=torch.Generator().manual_seed(16)) + 0.1).to(DEV)
    row_scale = lw / lw.sum()
    weighted = (ws[1] * row_scale).sum()
    torch.cuda.synchronize()
    lse_ref, loss_ref = ce_fwd_ref(logits, labels, V, ls)
    valid = labels != -100
    _check_abs("ce.lse", ws[0], lse_ref, case)
    _check_abs("ce.loss", ws[1], loss_ref, case)
    assert bool((ws[1][~valid] == 0).all()), f"{case}: an ignored row has a non-zero loss"
    assert float(out[1]) == float(valid.sum()), case
    _check_rel("ce.mean", out[0], loss_ref[valid].mean(), case + " mean")
    _check_rel("ce.mean", weighted, (loss_ref * row_scale.double()).sum(), case + " row_scale-weighted")


def test_ce_fwd_all_rows_ignored():
    """no valid row: the mean is NaN and the count 0, as torch's mean cross-entropy gives"""
    rows, V, ld = 37, 2025, 2048
    logits, _ = ce_inputs(rows, V, ld, 17)
    labels = torch.full((rows,), -100, dtype=torch.int64)
    out, ws = ops.ce_fwd(logits.to(BF).to(DEV), labels.to(DEV), V, 0.1)
    torch.cuda.synchronize()
    want = torch.nn.functional.cross_entropy(logits[:, :V].to(BF).double(), labels, ignore_index=-100, label_smoothing=0.1)
    assert math.isnan(float(want)) and math.isnan(float(out[0])) and float(out[1]) == 0.0
    assert bool((ws[1] == 0).all())
    lse_ref = ce_fwd_ref(logits.to(BF).to(DEV), labels.to(DEV), V, 0.1)[0]
    check_abs(ws[0], lse_ref, lambda r: f"row {r}", BOUNDS["ce.lse"][0], "ce.lse (all rows ignored)")


# ------------------------------------------------------------------------------------------------------------ U-ViT
DT_PAIRS = [(BF, BF), (BF, torch.float32), (torch.float32, BF), (torch.float32, torch.float32)]  # (dy, da)
ANM_CASES = [(H, rps) for H in (72, 264, 520, 776, 1024) for rps in (77, 257, 256)]


@pytest.mark.parametrize("i", range(len(ANM_CASES)))
def test_add_norm_mod_local(i):
    H, rps = ANM_CASES[i]
    dy_dt, da_dt = DT_PAIRS[i % 4]
    rms, B, eps = i % 2, 3, 1e-6
    T = B * rps
    case = f"(H {H}, rows_per_sample {rps}, B {B}, rms {rms}, dy {dy_dt}, da {da_dt})"
    a = _randn((T, H), 16).to(BF).to(DEV)
    r = _randn((T, H), 17).to(DEV)
    w = (1 + 0.1 * _randn((H,), 18)).to(DEV)
    mod_all = (_randn((B, 2 * H + 64), 19) * 0.3).to(DEV)
    mod = mod_all[:, 32:32 + 2 * H]  # a pitched view, like the batched adaLN mapper output
    r_out, y = ops.add_norm_mod(a, w, eps, rms, residual=r, mod=mod, rows_per_sample=rps)
    dy = _randn((T, H), 20).to(dy_dt).to(DEV)
    dro = _randn((T, H), 21).to(DEV)
    dw = torch.zeros(H, device=DEV)
    dmod_all = torch.zeros_like(mod_all)
    dmod = dmod_all[:, 32:32 + 2 * H]
    da, dr = ops.add_norm_mod_bwd(dy, dro, r_out, w, eps, rms, da_dt, mod=mod, rows_per_sample=rps, dw=dw, dmod=dmod)
    torch.cuda.synchronize()

    def fwd(x, wd, md):
        n = _norm_ref(x, wd, eps, rms)
        return (n.view(B, rps, H) * (1 + md[:, None, :H]) + md[:, None, H:]).view(T, H)

    _check("anm.y", y, fwd(a.to(F64) + r.to(F64), w.to(F64), mod.to(F64)), by_row(T), case)
    xd, wd, md = (t.to(F64).requires_grad_(True) for t in (r_out, w, mod))
    ((fwd(xd, wd, md) * dy.to(F64)).sum() + (xd * dro.to(F64)).sum()).backward()
    _check("anm.da_bf16" if da_dt == BF else "anm.da_f32", da, xd.grad, by_row(T), case)
    _check("anm.da_f32", dr, xd.grad, by_row(T), case + " dr")
    _check("anm.dw", dw, wd.grad, by_row(H, "column"), case)
    sample = Groups(lambda t: t.reshape(2 * B, H), lambda g: f"(sample {g // 2}, {'shift' if g % 2 else 'scale'})")
    _check("anm.dmod", dmod, md.grad, sample, case)
    assert bool((dmod_all[:, :32] == 0).all() and (dmod_all[:, 32 + 2 * H:] == 0).all()), case


def _pixels(B, hh, ww, border):
    yy, xx = torch.meshgrid(torch.arange(hh), torch.arange(ww), indexing="ij")
    edge = ((yy == 0) | (yy == hh - 1) | (xx == 0) | (xx == ww - 1)).reshape(-1)
    sel = edge if border else ~edge
    idx = (torch.arange(B)[:, None] * hh * ww + torch.nonzero(sel)[:, 0][None]).reshape(-1)
    return idx.to(DEV)


def _pixel_groups(B, hh, ww, idx):
    def where(g):
        p = int(idx[g])
        return f"(image {p // (hh * ww)}, y {p % (hh * ww) // ww}, x {p % ww})"
    return Groups(lambda t: t[idx], where)


@pytest.mark.parametrize("hh,ww", [(8, 24), (32, 32), (5, 7)])
@pytest.mark.parametrize("C", [264, 520])
def test_dwconv3x3_norm_local(hh, ww, C):
    B, eps = 2, 1e-6
    rms = int(C == 520)
    T = B * hh * ww
    case = f"(B {B}, hh {hh}, ww {ww}, C {C}, rms {rms})"
    x = _randn((T, C), 22).to(DEV)
    wk = (_randn((9, C), 23) * 0.3).to(DEV)
    nw = (1 + 0.1 * _randn((C,), 24)).to(DEV)
    y, conv = ops.dwconv3x3_norm(x, wk, nw, B, hh, ww, eps, rms, save_conv=True)
    dy = _randn((T, C), 25).to(BF).to(DEV)
    dres = _randn((T, C), 26).to(DEV)
    dwk, dnw = torch.zeros(9, C, device=DEV), torch.zeros(C, device=DEV)
    dx = ops.dwconv3x3_norm_bwd(dy, conv, x, wk, nw, dres, dwk, dnw, B, hh, ww, eps, rms)
    torch.cuda.synchronize()
    xd, wkd, nwd = (t.to(F64).requires_grad_(True) for t in (x, wk, nw))
    img = xd.view(B, hh, ww, C).permute(0, 3, 1, 2)
    cv = torch.nn.functional.conv2d(img, wkd.t().reshape(C, 1, 3, 3), padding=1, groups=C)
    cv = cv.permute(0, 2, 3, 1).reshape(T, C)
    yr = _norm_ref(_bf16_st(cv), nwd, eps, rms)  # Norm2D of the bf16 conv output
    yr.backward(dy.to(F64))
    for border in (True, False):
        idx = _pixels(B, hh, ww, border)
        if idx.numel() == 0:
            continue
        g = _pixel_groups(B, hh, ww, idx)
        part = case + (" border pixels" if border else " interior pixels")
        _check("dwconv.y", y, yr, g, part)
        _check("dwconv.dx", dx, xd.grad + dres.to(F64), g, part)
    _check("dwconv.dwk", dwk, wkd.grad, by_row(9, "tap"), case)
    _check("dwconv.dnw", dnw, nwd.grad, by_row(C, "channel"), case)


@pytest.mark.parametrize("C", [72, 520])
def test_grn_local(C):
    B, hw = 3, 12
    HW = hw * hw
    case = f"(B {B}, HW {HW}, C {C})"
    x = _randn((B, HW, C), 27) * 1.5
    x[1, :, 5] = 0  # an all-zero (image, channel): ||gelu(x)|| = 0
    x = x.reshape(B * HW, C).to(BF).to(DEV)
    gamma, beta = (_randn((C,), 28) * 0.2).to(DEV), (_randn((C,), 29) * 0.2).to(DEV)
    out, stats = ops.grn(x, gamma, beta, B, HW, save_stats=True)
    dout = _randn((B * HW, C), 30).to(BF).to(DEV)
    dg, db = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    dx = ops.grn_bwd(x, dout, stats, gamma, dg, db, B, HW)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(dx.float()).all()), case
    xd, gd, bd = (t.to(F64).requires_grad_(True) for t in (x, gamma, beta))
    gg = _bf16_st(torch.nn.functional.gelu(xd)).view(B, HW, C)  # the bf16 GELU output
    gx = torch.norm(gg, p=2, dim=1, keepdim=True)                # torch's subgradient 0 at ||x|| = 0
    o = gd * (gg * (gx / (gx.mean(dim=-1, keepdim=True) + 1e-6))) + bd + gg
    o.backward(dout.to(F64).view(B, HW, C))
    chan = Groups(lambda t: t.reshape(B, HW, C).permute(0, 2, 1).reshape(B * C, HW),
                  lambda g: f"(image {g // C}, channel {g % C})")
    _check("grn.out", out, o.reshape(B * HW, C), chan, case)
    _check("grn.dx", dx, xd.grad, chan, case)
    _check("grn.dgamma", dg, gd.grad, by_row(C, "channel"), case)
    _check("grn.dbeta", db, bd.grad, by_row(C, "channel"), case)
