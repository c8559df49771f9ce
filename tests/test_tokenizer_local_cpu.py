"""The tokenizer bounds of tests/local_error.py have teeth, shown on the CPU.

GroupNorm statistics: both statistics paths are emulated in fp32 in the kernels' own summation order -- the statistics
pass (gn_stats_kernel: 64 rows per thread, 8 row lanes merged per block, sums of x less the image's first pixel) and the convolution epilogue (pairs of rows per
thread, an 8-way xor tree per warp, 8 warps) -- once as {sum, sumsq} with var = sumsq / n - mean^2 (before) and once as
{sum, M2} merged with Chan's formula and the shift beta - mean * scale carried as two floats (now).  With a group mean
30 x its spread the old statistics break the GroupNorm bound (2 x torch fp32 group_norm, floor 2e-7); the new ones hold
it up to 300.

bf16x3 convolution: one tile emulated as hi*hi + lo*hi + hi*lo.  The stored bound accepts it and rejects a tile without
its lo*hi pass, a tile missing its last tap, an upsample parity written to the wrong pixel and a tile without its bias.
The old whole-tensor checks (rel-L2 2e-5, max-abs 2e-4 x max) catch these at this size too; the printed margins show how
little it takes (a one-tile defect divides by the square root of the tile count)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.local_error import BOUNDS, check_local, conv_tiles

F32 = np.float32
RATIOS = (0, 10, 30, 100, 300)
G, C, HW, EPS = 32, 128, 64 * 64, 1e-6


def _fma(a, b, c):
    """fp32 fused multiply-add (the product is exact in fp64)"""
    return (a.astype(np.float64) * b + c).astype(F32)


def _planted(seed):
    """[HW, C] fp32 (one image, NHWC): group g has mean RATIOS[g % 5] x its spread 2^(g % 4 - 2)"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((HW, G, C // G))
    std = 2.0 ** (np.arange(G) % 4 - 2)
    mean = np.array([RATIOS[g % 5] for g in range(G)]) * std * np.where(np.arange(G) % 2, -1, 1)
    return (x * std[None, :, None] + mean[None, :, None]).reshape(HW, C).astype(F32)


def _stats_pass(x, new):
    """gn_stats_kernel: C = 128 -> 32 channel quads x 8 row lanes, 512 rows per block, 64 rows per thread"""
    rpb, rstep = 512, 8
    xb = x.reshape(HW // rpb, rpb // rstep, rstep, C)  # [block, row step, lane, C]
    nb, steps = xb.shape[0], xb.shape[1]
    if not new:
        s, ss = np.zeros((nb, rstep, C), F32), np.zeros((nb, rstep, C), F32)
        for r in range(steps):
            v = xb[:, r]
            s = (s + v).astype(F32)
            ss = _fma(v, v, ss)
        sb, ssb = np.zeros((nb, C), F32), np.zeros((nb, C), F32)
        for k in range(rstep):
            sb, ssb = (sb + s[:, k]).astype(F32), (ssb + ss[:, k]).astype(F32)
        return sb, ssb, rpb, np.zeros(C, F32)
    K = x[0]  # the image's first pixel: the sums are of v - K
    mu, m2 = np.zeros((nb, rstep, C), F32), np.zeros((nb, rstep, C), F32)
    for r in range(steps):
        v = (xb[:, r] - K).astype(F32)
        inv = F32(1) / F32(r + 1)
        d = (v - mu).astype(F32)
        mu = _fma(d, inv, mu)
        m2 = _fma(d, (v - mu).astype(F32), m2)
    n, mean, M2 = F32(0), np.zeros((nb, C), F32), np.zeros((nb, C), F32)
    nk = F32(steps)
    for k in range(rstep):
        d = (mu[:, k] - mean).astype(F32)
        nn = F32(n + nk)
        mean = _fma(d, F32(nk / nn), mean)
        M2 = (M2 + (m2[:, k] + (d * d).astype(F32) * F32(n * nk / nn)).astype(F32)).astype(F32)
        n = nn
    return (mean * n).astype(F32), M2, rpb, K


def _xor_tree(v):
    """__shfl_xor_sync over lane bits 2..4: [..., 8 row groups] -> the butterfly sum every lane holds"""
    for o in (1, 2, 4):
        v = (v + v[..., np.arange(8) ^ o]).astype(F32)
    return v[..., 0]


def _epilogue(x, new):
    """conv_tc_kernel epilogue statistics of 128-pixel tiles: consumer warp w holds pixels 16 w .. 16 w + 15, lane group
    i the pixels 16 w + i and 16 w + i + 8"""
    t = x.reshape(HW // 128, 8, 2, 8, C)  # [tile, warp, row half, row group, C]
    a, b = t[:, :, 0], t[:, :, 1]         # [tile, warp, row group, C]
    s = np.moveaxis((a + b).astype(F32), 2, -1)  # [tile, warp, C, row group]
    s = _xor_tree(s)
    if new:
        m = (s * F32(1 / 16)).astype(F32)[:, :, None]
        da, db = (a - m).astype(F32), (b - m).astype(F32)
        q = _xor_tree(np.moveaxis(_fma(db, db, (da * da).astype(F32)), 2, -1))
    else:
        q = _xor_tree(np.moveaxis(_fma(b, b, _fma(a, a, np.zeros_like(a))), 2, -1))
    st, qt = np.zeros(s[:, 0].shape, F32), np.zeros(s[:, 0].shape, F32)
    for w in range(8):
        st, qt = (st + s[:, w]).astype(F32), (qt + q[:, w]).astype(F32)
    if new:
        mean = (st * F32(1 / 128)).astype(F32)
        for w in range(8):
            d = _fma(s[:, w], F32(1 / 16), -mean)
            qt = _fma((F32(16) * d).astype(F32), d, qt)
    return st, qt, 128, np.zeros(C, F32)


def _finalize_apply(x, part, new, gamma, beta):
    """gn_finalize_kernel (fp64) + the fp32 apply: y = fma(x, scale, shift) before, fma(x, scale, shift_hi) + shift_lo now"""
    K = part[3].astype(np.float64)
    s, q, rows = np.asarray(part[0], np.float64) + part[2] * K, np.asarray(part[1], np.float64), part[2]
    cpg, n = C // G, HW * (C // G)
    sg = s.reshape(-1, G, cpg)
    mean = sg.sum((0, 2)) / n
    if new:
        ni = rows
        var = (q.reshape(-1, G, cpg).sum((0, 2)) + (ni * (sg / ni - mean[None, :, None]) ** 2).sum((0, 2))) / n
    else:
        var = np.maximum(q.reshape(-1, G, cpg).sum((0, 2)) / n - mean * mean, 0)
    rstd = (1.0 / np.sqrt(var + np.float64(F32(EPS)))).astype(F32)
    sc = (np.repeat(rstd, cpg) * gamma).astype(F32)
    if not new:
        sh = (beta - (np.repeat(mean.astype(F32), cpg) * sc).astype(F32)).astype(F32)
        return _fma(x, sc, sh)
    sh = beta.astype(np.float64) - np.repeat(mean, cpg) * sc  # fp64, carried as two floats
    sh_hi = sh.astype(F32)
    return (_fma(x, sc, sh_hi) + (sh - sh_hi).astype(F32)).astype(F32)


def _gn_errors(path, new):
    """worst per-group rel-L2 of the emulated GroupNorm, of torch fp32 group_norm, per mean / std"""
    x = _planted(1)
    rng = np.random.default_rng(2)
    gamma, beta = (1 + 0.1 * rng.standard_normal(C)).astype(F32), (0.1 * rng.standard_normal(C)).astype(F32)
    part = _stats_pass(x, new) if path == "stats" else _epilogue(x, new)
    y = _finalize_apply(x, part, new, gamma, beta)
    xt = torch.from_numpy(x).t().reshape(1, C, 64, 64)
    ref = F.group_norm(xt.double(), G, torch.from_numpy(gamma).double(), torch.from_numpy(beta).double(), EPS)
    t32 = F.group_norm(xt.contiguous(), G, torch.from_numpy(gamma), torch.from_numpy(beta), EPS).double()
    grp = lambda t: t.reshape(G, -1)  # noqa: E731
    yt = torch.from_numpy(y).double().t().reshape(1, C, 64, 64)
    e = ((grp(yt) - grp(ref)).norm(dim=1) / grp(ref).norm(dim=1)).numpy()
    et = ((grp(t32) - grp(ref)).norm(dim=1) / grp(ref).norm(dim=1)).numpy()
    bound = np.maximum(2 * et, 2e-7)
    out = {}
    for g in range(G):
        r = RATIOS[g % 5]
        out[r] = max(out.get(r, (0, 0, True))[0], e[g]), max(out.get(r, (0, 0, True))[1], et[g]), \
            out.get(r, (0, 0, True))[2] and bool(e[g] <= bound[g])
    return out


@pytest.mark.parametrize("path", ["stats", "epilogue"])
def test_groupnorm_statistics_old_fail_new_pass(path):
    old, new = _gn_errors(path, False), _gn_errors(path, True)
    print(f"\n{path}: mean/std, worst group error old -> new (torch fp32 group_norm)")
    for r in RATIOS:
        print(f"  {r:>4}: {old[r][0]:.2e} -> {new[r][0]:.2e} ({old[r][1]:.2e})")
    assert all(new[r][2] for r in RATIOS), new
    assert not any(old[r][2] for r in RATIOS if r >= 30), old


# ------------------------------------------------------------------------------------------- bf16x3 convolution tiles
def _split(t):
    h = t.to(torch.bfloat16).double()
    return h, (t - h).to(torch.bfloat16).double()


def _conv_emulation(mutant=None, up=False):
    """3 images (scales 1/2, 1, 2) 32 x 32 (upsample: from 16 x 16), 128 -> 128 channels, 3x3, bias: the bf16x3 sum of
    the three products (fp64, rounded to fp32) against the fp64 convolution; mutants hit one tile of image 0."""
    g = torch.Generator().manual_seed(5)
    B, Ci, Co, H = 3, 128, 128, 32
    hi = H // 2 if up else H
    x = (torch.randn(B, Ci, hi, hi, generator=g) * torch.tensor([0.5, 1.0, 2.0]).view(B, 1, 1, 1)).float().double()
    w = (torch.randn(Co, Ci, 3, 3, generator=g) / 34).float().double()
    bias = torch.randn(Co, generator=g).float().double()
    xin = F.interpolate(x, scale_factor=2.0, mode="nearest") if up else x
    ref = F.conv2d(xin, w, bias, padding=1)
    xh, xl = _split(xin)
    wh, wl = _split(w)
    prods = [F.conv2d(xh, wh, None, padding=1), F.conv2d(xl, wh, None, padding=1), F.conv2d(xh, wl, None, padding=1)]
    emu = prods[0] + prods[1] + prods[2] + bias.view(1, -1, 1, 1)
    ys, xs = slice(4, 8), slice(0, 32)  # tile 1 of image 0: rows 4..7 (32-wide tiles, 4 rows)
    if mutant == "one tile without its lo*hi pass":
        emu[0, :, ys, xs] -= prods[1][0, :, ys, xs]
    if mutant == "one tile missing its last tap":
        last = torch.zeros_like(w)
        last[:, :, 2, 2] = wh[:, :, 2, 2] + wl[:, :, 2, 2]
        emu[0, :, ys, xs] -= F.conv2d(xin, last, None, padding=1)[0, :, ys, xs]
    if mutant == "one tile without its bias":
        emu[0, :, ys, xs] -= bias.view(-1, 1, 1)
    if mutant == "one upsample parity written to the wrong pixel":
        # parity (0, 1) of low-resolution tile 0 (rows 0..7, all 16 columns) lands on the pixels of parity (0, 0)
        emu[0, :, 0:16:2, 0:32:2] = emu[0, :, 0:16:2, 1:32:2]
    nhwc = lambda t: t.float().double().permute(0, 2, 3, 1)  # noqa: E731
    return nhwc(emu), ref.permute(0, 2, 3, 1), (B, H, H, Co)


MUTANTS = ["one tile without its lo*hi pass", "one tile missing its last tap", "one tile without its bias",
           "one upsample parity written to the wrong pixel"]


@pytest.mark.parametrize("up", [False, True])
def test_conv_bf16x3_emulation_is_accepted(up):
    emu, ref, (B, H, W, Co) = _conv_emulation(up=up)
    res = check_local(emu, ref, conv_tiles(B, H, W, Co, up), *BOUNDS["conv.bf16x3"], "conv.bf16x3 emulation")
    print(f"\nbf16x3 emulation{' (upsample)' if up else ''}: worst tile {res.worst:.2e}, whole rel-L2 {res.whole:.2e}")


# whole-tensor rel-L2 / max-abs relative to the global max; measured with this emulation
OLD_CHECK_PASSES = {"one tile without its lo*hi pass": False, "one tile missing its last tap": False,
                    "one tile without its bias": False, "one upsample parity written to the wrong pixel": False}


@pytest.mark.parametrize("mutant", MUTANTS)
def test_conv_bound_rejects_mutant(mutant):
    up = "parity" in mutant
    emu, ref, (B, H, W, Co) = _conv_emulation(mutant, up)
    with pytest.raises(AssertionError, match="worst group error"):
        check_local(emu, ref, conv_tiles(B, H, W, Co, up), *BOUNDS["conv.bf16x3"], f"conv.bf16x3 {mutant}")
    whole = float((emu - ref).norm() / ref.norm())
    peak = float((emu - ref).abs().max() / ref.abs().max())
    old_pass = whole < 2e-5 and peak < 2e-4
    print(f"\n{mutant}: whole-tensor rel-L2 {whole:.2e} (old bound 2e-5), max-abs / max {peak:.2e} (old bound 2e-4): "
          f"old checks {'pass' if old_pass else 'fail'} it")
    assert old_pass == OLD_CHECK_PASSES[mutant]
