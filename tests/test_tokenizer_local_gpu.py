"""Every tile, image and group of the tokenizer kernels against fp64 (tests/local_error.py).

The tokenizer convolutions promise fp32-faithful results (csrc/conv_tc.cu: the arg-min token ids downstream flip on a
perturbation of ~1e-3), so their references are fp64 computed from exactly the fp32 operands the kernels receive.  Inputs
are structured so that a local defect is a large error of one group: a distinct power of two per 64-channel chunk, per
tap and per image (a skipped k-block or another image's weights shows), 4x values on image borders and 2x on tile edges
(a wrong halo or padding shows).  Shapes reach every tile shape, persistent CTAs that take a second and third tile, the
ragged second N tile, the upsample parities, the space-to-depth downsample, the im2col stem and per-image weights.

GroupNorm is checked group by group against torch's own fp32 group_norm: each (image, group) may be off by at most
max(2e-7, 2 x the error of torch fp32 group_norm on the same NCHW input), with planted groups whose mean is 0, 10, 30, 100
and 300 times their spread, a constant group and a group with one outlier pixel."""
import math

import pytest
import torch
import torch.nn.functional as F

from open_muse_b200 import _lib, ops
from tests.local_error import BOUNDS, Groups, check_local, conv_tile_pixels, conv_tiles, gemm_tiles, gn_groups
from tests.local_error import rows as by_row

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16
F64 = torch.float64

_worst = {}     # bound key -> (Local, case) with the largest group error seen
_gn_worst = {}  # (path, mean / std) -> (worst group error, torch fp32 error of that group, case)


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
            print(f"  {key:15s} {r.worst:.3e} (bound {BOUNDS[key][0]:.1e}, elem {r.elem:.3e} / {BOUNDS[key][1]:.1e}) "
                  f"{case} {r.where}; whole {r.whole:.3e}")
    print("GroupNorm: worst group error by mean / std (torch fp32 group_norm on the same group):")
    for (path, ratio), (e, et, case) in sorted(_gn_worst.items()):
        print(f"  {path:12s} mean/std {ratio:>6}: {e:.3e} (torch fp32 {et:.3e}) {case}")


def _randn(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g) * scale


def _pow2(i, period=3):
    """0.5, 1, 2, 0.5, ... for index tensor i"""
    return torch.pow(2.0, (i % period - 1).double()).float()


def _structured(B, C, H, W, seed):
    """NCHW fp32: a distinct power of two per 64-channel chunk and per image, 4x on image borders, 2x on the edges of the
    128-pixel tiles (tile_w = min(W, 128) wide, 128 / tile_w high)."""
    x = _randn((B, C, H, W), seed)
    x *= _pow2(torch.arange(C) // 64)[None, :, None, None] * _pow2(torch.arange(B))[:, None, None, None]
    tw = min(W, 128)
    th = max(1, 128 // tw)
    ys, xs = torch.arange(H), torch.arange(W)
    x[:, :, (ys % th == 0) | (ys % th == th - 1)] *= 2
    x[:, :, :, (xs % tw == 0) | (xs % tw == tw - 1)] *= 2
    x[:, :, [0, H - 1]] *= 4
    x[:, :, :, [0, W - 1]] *= 4
    return x


def _weight(Cout, Cin, k, seed):
    """a distinct power of two per tap (and per 64-input-channel chunk through the input)"""
    w = _randn((Cout, Cin, k, k), seed) / math.sqrt(Cin * k * k)
    return w * _pow2(torch.arange(k * k)).view(1, 1, k, k)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


# ------------------------------------------------------------------------------------------- tensor-core convolutions
CONV_CASES = [
    # B, H, W (output), Cin, Cout, k, bias, residual, mode
    (3, 128, 128, 64, 128, 3, True, True, "plain"),   # 384 tiles: CTAs take a second and a third tile
    (2, 32, 8, 128, 256, 1, False, True, "plain"),    # W 8: 8 x 16 tiles, 2 channel chunks, 1x1
    (2, 16, 16, 512, 128, 3, True, False, "plain"),   # W 16: 8 channel chunks
    (2, 32, 32, 64, 384, 3, True, True, "plain"),     # W 32: ragged second N tile (256 + 128)
    (1, 64, 64, 128, 48, 3, True, True, "plain"),     # W 64: C_out 48 in a 128-wide N tile
    (2, 4, 256, 64, 512, 3, True, True, "plain"),     # W 256: two tiles per image row, two N tiles
    (2, 16, 16, 128, 16, 3, True, True, "plain"),     # 16-wide N tile
    (2, 32, 32, 128, 3, 3, True, False, "plain"),     # the 3-channel decoder head
    (2, 64, 64, 128, 128, 3, True, True, "up"),       # nearest x2 + 3x3: 8 tiles per parity
    (1, 32, 256, 64, 256, 3, True, False, "up"),      # low-resolution W 128
    (1, 128, 32, 64, 512, 3, False, True, "up"),      # low-resolution W 16, two N tiles
    (3, 128, 128, 32, 128, 3, True, False, "down"),   # space-to-depth 2x2 (128 channels), 384 tiles
    (2, 16, 16, 128, 256, 3, True, False, "down"),    # space-to-depth 2x2 (512 channels: 8 chunks)
    (3, 128, 128, 3, 128, 3, True, True, "stem"),     # the 27-tap im2col stem, 384 tiles
]


def _conv_case(B, H, W, Cin, Cout, k, bias, res, mode, seed):
    hi, wi = {"up": (H // 2, W // 2), "down": (2 * H, 2 * W)}.get(mode, (H, W))
    x = _structured(B, Cin, hi, wi, seed)
    w = _weight(Cout, Cin, k, seed + 1)
    b = _randn((Cout,), seed + 2) if bias else None
    r = _structured(B, Cout, H, W, seed + 3) if res else None
    x64, w64 = x.to(DEV, F64), w.to(DEV, F64)
    b64 = None if b is None else b.to(DEV, F64)
    if mode == "down":
        ref = F.conv2d(F.pad(x64, (0, 1, 0, 1)), w64, b64, stride=2)
    else:
        ref = F.conv2d(F.interpolate(x64, scale_factor=2.0, mode="nearest") if mode == "up" else x64, w64, b64,
                       padding=k // 2)
    if r is not None:
        ref = ref + r.to(DEV, F64)
    xd = _nhwc(x).contiguous().to(DEV)
    bd = None if b is None else b.to(DEV)
    rd = None if r is None else _nhwc(r).contiguous().to(DEV)
    tc = ops._conv_state["route"] != "simt"
    if mode == "down":
        assert not tc or _lib.load().muse_conv2d_tc_supported(H, W, 4 * Cin, Cout, 2)
        y = ops.conv2d_down(xd, w.to(DEV), bd)
    else:
        assert not tc or ops.conv_uses_tensor_cores(H, W, Cin, Cout, k)
        y = ops.conv2d(xd, w.to(DEV), bias=bd, residual=rd, upsample2x=(mode == "up"))
    torch.cuda.synchronize()
    return y, _nhwc(ref)


def _check_stats(y, B, H, W, Cout, up, case):
    """the epilogue's {sum, M2} per (image, parity, tile, channel) against fp64 of the y the kernel wrote"""
    stats, tiles, _ = y._gn_stats
    pix = conv_tile_pixels(y.to(F64), up)  # [B, P, T, 128, C]
    P, T = pix.shape[1], pix.shape[2]
    assert stats.shape == (B, P * T, Cout, 2)
    st = stats.view(B, P, T, Cout, 2).to(F64)
    s_ref = pix.sum(3)
    m2_ref = (pix - pix.mean(3, keepdim=True)).pow(2).sum(3)

    def where(g):
        return f"(image {g // (P * T)}, parity {g // T % P}, tile {g % T}, all channels)"

    per_tile = Groups(lambda t: t.reshape(B * P * T, Cout), where)
    _check("conv.stats_sum", st[..., 0], s_ref, per_tile, case)
    _check("conv.stats_m2", st[..., 1], m2_ref, per_tile, case)


@pytest.mark.parametrize("i", range(len(CONV_CASES)))
def test_conv_tc_local(i):
    B, H, W, Cin, Cout, k, bias, res, mode = CONV_CASES[i]
    case = f"(B {B}, {H}x{W}, Cin {Cin}, Cout {Cout}, k {k}, bias {bias}, residual {res}, {mode})"
    y, ref = _conv_case(B, H, W, Cin, Cout, k, bias, res, mode, 100 + i)
    _check("conv.bf16x3", y, ref, conv_tiles(B, H, W, Cout, mode == "up"), case)
    if Cout > 16 and Cout % 32 == 0:
        _check_stats(y, B, H, W, Cout, mode == "up", case)


@pytest.mark.parametrize("i", [0, 3, 8, 11])
def test_conv_tc_single_pass_local(i):
    B, H, W, Cin, Cout, k, bias, res, mode = CONV_CASES[i]
    case = f"(B {B}, {H}x{W}, Cin {Cin}, Cout {Cout}, k {k}, {mode}, single-pass bf16)"
    with ops.conv_precision("bf16"):
        y, ref = _conv_case(B, H, W, Cin, Cout, k, bias, res, mode, 200 + i)
    _check("conv.bf16", y, ref, conv_tiles(B, H, W, Cout, mode == "up"), case)


@pytest.mark.parametrize("B,hw,C", [(3, 16, 512), (3, 32, 512)])
def test_attention_single_head_local(B, hw, C):
    """AttnBlock: both products as 1x1 convolutions with per-image weights (the image's own keys / values)"""
    HW = hw * hw
    case = f"(B {B}, {hw}x{hw}, C {C})"
    sc = _pow2(torch.arange(B))[:, None, None]
    q, k, v = (_randn((B, HW, C), 300 + j) * sc * (0.5 if j == 0 else 1.0) for j in range(3))
    k = k * sc  # keys and values scaled per image: another image's weights show
    lib = _lib.load()
    assert lib.muse_conv2d_tc_supported(hw, hw, C, HW, 1) and lib.muse_conv2d_tc_supported(hw, hw, HW, C, 1)
    o = ops.attention_single_head(*(t.reshape(-1, C).to(DEV) for t in (q, k, v)), B, hw, hw)
    torch.cuda.synchronize()
    q64, k64, v64 = (t.to(DEV, F64) for t in (q, k, v))
    ref = torch.softmax(q64 @ k64.transpose(1, 2) * C ** -0.5, -1) @ v64
    _check("attn1.out", o.view(B, hw, hw, C), ref.view(B, hw, hw, C), conv_tiles(B, hw, hw, C), case)


# ------------------------------------------------------------------------------------------- SIMT convolutions
SIMT_CASES = [
    # B, H, W (output), Cin, Cout, k, bias, residual, mode
    (2, 13, 11, 20, 8, 3, True, True, "plain"),     # M = 286 (ragged M block), scalar loader, C_out <= 16
    (1, 15, 17, 64, 200, 3, True, True, "plain"),   # M = 255, C_out 200: ragged N block
    (1, 12, 12, 32, 144, 1, False, True, "plain"),  # 1x1
    (2, 14, 18, 24, 40, 3, True, False, "up"),      # nearest x2 folded into the scalar gather
    (2, 9, 7, 16, 24, 3, True, False, "down"),      # stride 2, pad (0, 1, 0, 1)
]


@pytest.mark.parametrize("i", range(len(SIMT_CASES)))
def test_conv_simt_local(i):
    B, H, W, Cin, Cout, k, bias, res, mode = SIMT_CASES[i]
    case = f"(B {B}, {H}x{W}, Cin {Cin}, Cout {Cout}, k {k}, bias {bias}, residual {res}, {mode}, SIMT)"
    with ops.conv_route("simt"):
        y, ref = _conv_case(B, H, W, Cin, Cout, k, bias, res, mode, 400 + i)
    M = B * H * W
    _check("conv.simt", y.reshape(M, Cout), ref.reshape(M, Cout), gemm_tiles(M, Cout, 128 if Cout > 16 else 16), case)


# ------------------------------------------------------------------------------------------- GroupNorm
RATIOS = (0, 10, 30, 100, 300)
G = 32


def _planted_gn(B, C, HW, seed):
    """[B, C, HW] fp32: group g of image b has mean RATIOS[(g + b) % 5] x its spread 2^(g % 4 - 2) (alternating sign);
    group G - 1 of image 0 is constant, group G - 2 of the last image has one pixel 1e3 x its spread."""
    cpg = C // G
    x = _randn((B, G, cpg, HW), seed)
    for b in range(B):
        for g in range(G):
            std = 2.0 ** (g % 4 - 2)
            x[b, g] = x[b, g] * std + RATIOS[(g + b) % 5] * std * (-1 if g % 2 else 1)
    x[0, G - 1] = 0.75
    x[B - 1, G - 2, 0, HW // 3] = 1e3 * 2.0 ** ((G - 2) % 4 - 2)
    return x.reshape(B, C, HW)


def _gn_affine(C, seed):
    ga, be = 1 + 0.1 * _randn((C,), seed), 0.1 * _randn((C,), seed + 1)
    cpg = C // G
    ga[(G - 1) * cpg:], be[(G - 1) * cpg:] = 0.5, 0.125  # the constant group's output is exactly beta
    return ga, be


def _gn_labels(B, shift=1, const_images=(0,)):
    """mean / std label of each (image, group) of _planted_gn (shift 1) or _planted_conv_output (shift 0)"""
    return ["const" if (g == G - 1 and b in const_images) else
            ("outlier" if (g == G - 2 and b == B - 1) else str(RATIOS[(g + shift * b) % 5]))
            for b in range(B) for g in range(G)]


def _check_gn(out, x32, ga, be, silu, path, case, labels, planes=False):
    """out NHWC [B, H, W, C] (fp32, or hi + lo); x32 the fp32 NCHW input the kernel normalised.  Per (image, group):
    rel-L2 <= max(2e-7, 2 x torch fp32 group_norm's on the same group[, 2 x the hi + lo split of the exact result])."""
    B, C = x32.shape[:2]
    HW = x32[0, 0].numel()

    def fn(t, gamma, beta):
        y = F.group_norm(t, G, gamma, beta, 1e-6)
        return F.silu(y) if silu else y

    ref = fn(x32.double(), ga.double(), be.double())
    t32 = fn(x32.float().cpu().contiguous(), ga.float(), be.float()).double()
    groups = gn_groups(B, HW, C, G)
    to_g = lambda t: groups.view(t.reshape(B, C, HW).permute(0, 2, 1).to(F64).cpu())  # noqa: E731
    r = to_g(ref)
    rn = r.norm(dim=1)
    e = (to_g(out.permute(0, 3, 1, 2)) - r).norm(dim=1) / rn
    et = (to_g(t32) - r).norm(dim=1) / rn
    bound = (2 * et).clamp_min(2e-7)
    if planes:  # the planes cannot be closer than the hi + lo split of the exact result
        r32 = r.float()
        h = r32.to(BF).float()
        rep = (h + (r32 - h).to(BF).float()).double()
        bound = torch.maximum(bound, 2 * (rep - r).norm(dim=1) / rn)
    for gi in range(B * G):
        key = (path, labels[gi])
        if key not in _gn_worst or float(e[gi]) > _gn_worst[key][0]:
            _gn_worst[key] = (float(e[gi]), float(et[gi]), case)
    bad = (e > bound).nonzero()[:, 0].tolist()
    worst = int((e / bound).argmax())
    assert not bad, (f"{path} {case}: {len(bad)} groups over max(2e-7, 2 x torch fp32); worst {groups.where(worst)} "
                     f"mean/std {labels[worst]}: {float(e[worst]):.3e} vs torch fp32 "
                     f"{float(et[worst]):.3e}")


@pytest.mark.parametrize("C", [64, 128, 256, 512])
@pytest.mark.parametrize("silu", [0, 1])
def test_groupnorm_local(C, silu):
    """statistics pass (ragged last block: HW = 2115) + fp32 apply"""
    B, H, W = 2, 45, 47
    case = f"(B {B}, {H}x{W}, C {C}, silu {silu}, fp32 out)"
    x = _planted_gn(B, C, H * W, 500 + C).view(B, C, H, W)
    ga, be = _gn_affine(C, 501)
    y = ops.groupnorm_silu(_nhwc(x).contiguous().to(DEV), ga.to(DEV), be.to(DEV), G, 1e-6, silu=silu)
    _check_gn(y.cpu(), x, ga, be, silu, "stats pass", case, _gn_labels(B))


def _identity(C):
    return torch.eye(C).view(C, C, 1, 1).to(DEV)


@pytest.mark.parametrize("C", [64, 128, 256, 512])
@pytest.mark.parametrize("silu", [0, 1])
def test_groupnorm_planes_local(C, silu):
    """conv2d(gn=...): statistics pass (ragged last block for C <= 256) + the bf16 hi / lo planes, read back exactly
    through a 1x1 identity convolution (hi * 1 + lo * 1 is exact in fp32)"""
    B, H, W = 2, 136, 16
    case = f"(B {B}, {H}x{W}, C {C}, silu {silu}, hi + lo planes)"
    x = _planted_gn(B, C, H * W, 600 + C).view(B, C, H, W)
    ga, be = _gn_affine(C, 601)
    y = ops.conv2d(_nhwc(x).contiguous().to(DEV), _identity(C), gn=(ga.to(DEV), be.to(DEV), G, 1e-6, silu))
    _check_gn(y.cpu(), x, ga, be, silu, "stats pass", case, _gn_labels(B), planes=True)


def _planted_conv_output(B, C, H, W, up, seed):
    """conv2d whose output groups have planted mean / spread (through the bias and weight scale), a constant group (zero
    weights) and one outlier pixel (through the residual)"""
    cpg = C // G
    Ci = 64
    hi, wi = (H // 2, W // 2) if up else (H, W)
    x = _randn((B, Ci, hi, wi), seed)
    k = 3 if up else 1
    std = torch.tensor([2.0 ** (g % 4 - 2) for g in range(G)]).repeat_interleave(cpg)
    mean = torch.tensor([RATIOS[g % 5] * 2.0 ** (g % 4 - 2) * (-1 if g % 2 else 1) for g in range(G)]).repeat_interleave(cpg)
    w = _randn((C, Ci, k, k), seed + 1) * (std / math.sqrt(Ci * k * k)).view(C, 1, 1, 1)
    w[(G - 1) * cpg:] = 0
    mean[(G - 1) * cpg:] = 0.75
    r = torch.zeros(B, H, W, C)
    r[B - 1, H // 3, W // 2, (G - 2) * cpg] = 1e3 * 2.0 ** ((G - 2) % 4 - 2)
    return ops.conv2d(_nhwc(x).contiguous().to(DEV), w.to(DEV), bias=mean.to(DEV), residual=r.to(DEV), upsample2x=up)


@pytest.mark.parametrize("C", [64, 128, 256, 512])
@pytest.mark.parametrize("up", [False, True])
def test_groupnorm_from_conv_epilogue_local(C, up):
    """statistics {sum, M2} from the epilogue of the convolution that produced x (plain and upsample tiles)"""
    B, H, W = 2, 128, 16
    case = f"(B {B}, {H}x{W}, C {C}, statistics from the {'upsample ' if up else ''}conv epilogue)"
    y1 = _planted_conv_output(B, C, H, W, up, 700 + C)
    assert getattr(y1, "_gn_stats", None) is not None
    ga, be = _gn_affine(C, 701)
    y = ops.conv2d(y1, _identity(C), gn=(ga.to(DEV), be.to(DEV), G, 1e-6, 1))
    torch.cuda.synchronize()
    _check_gn(y.cpu(), y1.permute(0, 3, 1, 2).cpu(), ga, be, 1, "conv epilogue", case, _gn_labels(B, 0, range(B)),
              planes=True)


def test_groupnorm_stats_not_stale_after_in_place_update():
    """y modified in place after the convolution: conv2d(y, gn=...) must not use the epilogue statistics of the old y"""
    B, H, W, C = 2, 128, 16, 128
    y1 = _planted_conv_output(B, C, H, W, False, 800)
    y1[..., : C // 2].mul_(3.0).add_(5.0)
    ga, be = _gn_affine(C, 801)
    y = ops.conv2d(y1, _identity(C), gn=(ga.to(DEV), be.to(DEV), G, 1e-6, 1))
    torch.cuda.synchronize()
    _check_gn(y.cpu(), y1.permute(0, 3, 1, 2).cpu(), ga, be, 1, "in-place y", "(B 2, 128x16, C 128, y changed in place)",
              _gn_labels(B, 0, range(B)), planes=True)


# ------------------------------------------------------------------------------------------- softmax_split_rows
@pytest.mark.parametrize("n", [256, 1024])
def test_softmax_split_rows_local(n):
    rows, scale = 203, 1.0 / 16  # 203 = 25 blocks of 8 rows + 3; scale of the C = 256 AttnBlock (x * scale is exact)
    x = _randn((rows, n), 900 + n, 2.0 / scale)
    x[0, 7] = 60.0 / scale                          # one dominant logit
    x[1] = 1.5 / scale                              # all equal
    x[2] = x[2] - 200.0 / scale                     # far below zero: exp underflows without the max subtraction
    x[rows - 1, n - 1] = 40.0 / scale               # dominant logit in the last lane of the ragged last block
    xd = x.to(DEV)
    ref = torch.softmax(x.to(DEV, F64) * scale, -1)
    hi, lo = torch.empty(rows, n, dtype=BF, device=DEV), torch.empty(rows, n, dtype=BF, device=DEV)
    out = torch.empty(rows, n, device=DEV)
    st = ops._prep(xd)
    ops._call("muse_softmax_split_rows", ops._p(xd), ops._p(hi), ops._p(lo), None, rows, n, scale, st)
    ops._call("muse_softmax_split_rows", ops._p(xd), None, None, ops._p(out), rows, n, scale, st)
    torch.cuda.synchronize()
    case = f"(rows {rows}, n {n})"
    _check("softmax.split", hi.double() + lo.double(), ref, by_row(rows), case)
    _check("softmax.f32", out, ref, by_row(rows), case)


# ------------------------------------------------------------------------------------------- exact kernels
def _split(v):
    h = v.to(BF)
    return h, (v - h.float()).to(BF)


def _special(shape, seed):
    """random values plus round-to-nearest-even ties of bf16 and values whose lo part is itself a tie"""
    v = _randn(shape, seed).view(-1)
    ties = torch.tensor([1 + 2.0 ** -8, 1 + 3 * 2.0 ** -8, -(2 + 2.0 ** -7), 1 + 2.0 ** -8 + 2.0 ** -17, 3e-39, -1e30])
    v[: ties.numel()] = ties
    return v.view(shape)


@pytest.mark.parametrize("up", [0, 1])
def test_split_bf16_exact(up):
    B, H, W, C = 2, 6, 10, 24
    hi_, wi_ = (H // 2, W // 2) if up else (H, W)
    x = _special((B, hi_, wi_, C), 1000 + up)
    hi, lo = torch.empty(B, H, W, C, dtype=BF, device=DEV), torch.empty(B, H, W, C, dtype=BF, device=DEV)
    xd = x.to(DEV)
    ops._call("muse_split_bf16_nhwc", ops._p(xd), ops._p(hi), ops._p(lo), B, H, W, C, up, ops._prep(xd))
    src = x.repeat_interleave(2, 1).repeat_interleave(2, 2) if up else x
    h, lo_ref = _split(src)
    assert torch.equal(hi.cpu(), h) and torch.equal(lo.cpu(), lo_ref)


def test_split_s2d_exact():
    B, Ho, Wo, C = 2, 5, 3, 16
    x = _special((B, 2 * Ho, 2 * Wo, C), 1100)
    hi, lo = (torch.empty(B, Ho, Wo, 4 * C, dtype=BF, device=DEV) for _ in range(2))
    xd = x.to(DEV)
    ops._call("muse_split_s2d_bf16_nhwc", ops._p(xd), ops._p(hi), ops._p(lo), B, Ho, Wo, C, ops._prep(xd))
    # channel (2 * row parity + column parity) * C + c
    s2d = x.view(B, Ho, 2, Wo, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(B, Ho, Wo, 4 * C)
    h, lo_ref = _split(s2d)
    assert torch.equal(hi.cpu(), h) and torch.equal(lo.cpu(), lo_ref)


@pytest.mark.parametrize("Cin,k", [(3, 3), (7, 3), (64, 1)])
def test_im2col_split_exact(Cin, k):
    B, H, W = 2, 5, 9
    x = _special((B, H, W, Cin), 1200 + Cin)
    hi, lo = (torch.full((B, H, W, 64), float("nan"), dtype=BF, device=DEV) for _ in range(2))
    xd = x.to(DEV)
    ops._call("muse_im2col_split_nhwc", ops._p(xd), ops._p(hi), ops._p(lo), B, H, W, Cin, k, ops._prep(xd))
    p = k // 2
    xp = F.pad(x, (0, 0, p, p, p, p))
    cols = torch.zeros(B, H, W, 64)
    for tap in range(k * k):
        cols[..., tap * Cin:(tap + 1) * Cin] = xp[:, tap // k:tap // k + H, tap % k:tap % k + W]
    h, lo_ref = _split(cols)
    assert torch.equal(hi.cpu(), h) and torch.equal(lo.cpu(), lo_ref)


def test_avgpool_and_layout_exact():
    B, C, H, W = 2, 12, 10, 14
    x = _special((B, C, H, W), 1300).to(DEV)
    x[0, 0, :2, :2] = torch.tensor([[1.0, 2.0 ** -24], [2.0 ** -24, 2.0 ** -24]], device=DEV)  # the order of the sum shows
    xn = ops.to_nhwc(x)
    assert torch.equal(xn, x.permute(0, 2, 3, 1))
    assert torch.equal(ops.to_nchw(xn), x)
    assert torch.equal(ops.to_nchw(ops.avg_pool2x2(xn)), F.avg_pool2d(x, 2, 2))
