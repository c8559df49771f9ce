"""The SpatialNorm pass of MOVQ (muse_spatial_groupnorm_silu_nhwc through ops.groupnorm_silu / ops.conv2d(spatial=...))
per (image, pixel row, GroupNorm group) against fp64 (tests/local_error.check_local), on the planted inputs of the
GroupNorm tests in test_tokenizer_local_gpu.py: groups whose mean is 0 .. 300 times their spread, a constant group and an
outlier pixel.

The latent alternates sign and scale between neighbouring latent pixels, so that a wrong nearest-neighbour index (a row
or column taken from the next latent pixel) is an O(1) error of whole pixel rows, not a small whole-tensor error.  Each
output form is held to max(a fixed floor, 2 x the error of the ideally rounded result): torch's fp32 GroupNorm and
modulation, and for the planes also the hi + lo split / the bf16 rounding of the exact result."""
import pytest
import torch
import torch.nn.functional as F
from torch import nn

from open_muse_b200 import ops
from tests.local_error import Groups, check_local
from tests.test_tokenizer_local_gpu import G, _gn_affine, _identity, _planted_conv_output, _planted_gn

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16
F64 = torch.float64
FLOOR = {"fp32": (1e-6, 1e-5), "planes": (2e-5, 3e-4), "hi": (5e-3, 7e-2)}


def _latent(B, hz, wz, dq, seed):
    """a latent whose modulation flips sign and scale between neighbouring latent pixels"""
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(B, hz, wz, dq, generator=g)
    ys, xs = torch.arange(hz), torch.arange(wz)
    sign = (1 - 2 * ((ys[:, None] + xs[None, :]) % 2)).float()
    scale = 1.0 + 3.0 * ((ys[:, None] * 3 + xs[None, :]) % 4 == 0).float()
    return (z + 2.0 * sign[None, :, :, None]) * scale[None, :, :, None]


def _mod(C, dq, seed):
    torch.manual_seed(seed)
    cy, cb = nn.Conv2d(dq, C, 1), nn.Conv2d(dq, C, 1)
    with torch.no_grad():
        cy.bias.copy_(1.0 + 0.3 * torch.randn(C))
    return cy.to(DEV), cb.to(DEV)


def _ref(x, ga, be, zq, cy, cb, silu, dtype):
    """GN(x) * conv_y(up(zq)) + conv_b(up(zq)) (+ SiLU) in `dtype` on the CPU; x NCHW, zq NHWC -> NHWC"""
    z = F.interpolate(zq.permute(0, 3, 1, 2).to(dtype), size=x.shape[2:], mode="nearest")
    conv = lambda m: F.conv2d(z, m.weight.detach().cpu().to(dtype), m.bias.detach().cpu().to(dtype))  # noqa: E731
    y = F.group_norm(x.to(dtype), G, ga.to(dtype), be.to(dtype), 1e-6) * conv(cy) + conv(cb)
    return (F.silu(y) if silu else y).permute(0, 2, 3, 1)


def _rows(B, H, W, C):
    cpg = C // G
    return Groups(lambda t: t.reshape(B, H, W, G, cpg).permute(0, 1, 3, 2, 4).reshape(B * H * G, W * cpg),
                  lambda g: f"(image {g // (H * G)}, row {g // G % H}, group {g % G})")


def _check(out, x, ga, be, zq, cy, cb, silu, form, case):
    B, C, H, W = x.shape
    ref = _ref(x, ga, be, zq.cpu(), cy, cb, silu, F64)
    groups = _rows(B, H, W, C)
    ideals = [_ref(x.float(), ga, be, zq.cpu(), cy, cb, silu, torch.float32).double()]  # fp32 arithmetic
    if form != "fp32":  # the planes cannot be closer than the split (or the bf16 rounding) of the exact result
        r32 = ref.float()
        h = r32.to(BF).float()
        ideals.append((h + (r32 - h).to(BF).float() if form == "planes" else h).double())
    es = [check_local(i, ref, groups, float("inf"), float("inf"), "ideal") for i in ideals]
    bound = max(FLOOR[form][0], 2 * max(e.worst for e in es))
    elem = max(FLOOR[form][1], 2 * max(e.elem for e in es))
    res = check_local(out.cpu(), ref, groups, bound, elem, f"spatial groupnorm {form} {case}")
    print(f"{form:6s} {case}: worst row-group {res.worst:.2e} (bound {bound:.1e}), elem {res.elem:.2e}, whole {res.whole:.2e}")


@pytest.mark.parametrize("C", [32, 64, 128, 256, 512])
@pytest.mark.parametrize("silu", [0, 1])
def test_spatial_groupnorm_fp32_local(C, silu):
    """statistics pass with a ragged last block (HW = 2016), fp32 output (the SIMT route and the AttnBlock norm); a
    non-square grid with ratios 8 x 6"""
    B, H, W, hz, wz = 2, 48, 42, 6, 7
    dq = {32: 8, 64: 4, 128: 16}.get(C, 4)
    case = f"(B {B}, {H}x{W} from {hz}x{wz}, C {C}, dq {dq}, silu {silu})"
    x = _planted_gn(B, C, H * W, 900 + C).view(B, C, H, W)
    ga, be = _gn_affine(C, 901)
    zq = _latent(B, hz, wz, dq, 902).to(DEV)
    cy, cb = _mod(C, dq, 903)
    y = ops.groupnorm_silu(x.permute(0, 2, 3, 1).contiguous().to(DEV), ga.to(DEV), be.to(DEV), G, 1e-6, silu=silu,
                           spatial=(zq, cy, cb))
    _check(y, x, ga, be, zq, cy, cb, silu, "fp32", case)


@pytest.mark.parametrize("C", [64, 128, 256, 512])
@pytest.mark.parametrize("ratio", [1, 2, 4, 8])
def test_spatial_groupnorm_planes_local(C, ratio):
    """conv2d(gn=..., spatial=...): the bf16 hi / lo planes, read back exactly through a 1x1 identity convolution"""
    B, H, W = 2, 136, 16
    hz, wz = H // ratio, W // ratio
    case = f"(B {B}, {H}x{W} from {hz}x{wz}, C {C})"
    x = _planted_gn(B, C, H * W, 1000 + C).view(B, C, H, W)
    ga, be = _gn_affine(C, 1001)
    zq = _latent(B, hz, wz, 4, 1002 + ratio).to(DEV)
    cy, cb = _mod(C, 4, 1003)
    y = ops.conv2d(x.permute(0, 2, 3, 1).contiguous().to(DEV), _identity(C), gn=(ga.to(DEV), be.to(DEV), G, 1e-6, 1),
                   spatial=(zq, cy, cb))
    _check(y, x, ga, be, zq, cy, cb, 1, "planes", case)


def test_spatial_groupnorm_hi_only_local():
    """single-pass bf16 mode: the hi plane only"""
    B, H, W, C = 2, 64, 32, 256
    x = _planted_gn(B, C, H * W, 1100).view(B, C, H, W)
    ga, be = _gn_affine(C, 1101)
    zq = _latent(B, H // 2, W // 2, 4, 1102).to(DEV)
    cy, cb = _mod(C, 4, 1103)
    with ops.conv_precision("bf16"):
        y = ops.conv2d(x.permute(0, 2, 3, 1).contiguous().to(DEV), _identity(C), gn=(ga.to(DEV), be.to(DEV), G, 1e-6, 1),
                       spatial=(zq, cy, cb))
    _check(y, x, ga, be, zq, cy, cb, 1, "hi", f"(B {B}, {H}x{W} from {H // 2}x{W // 2}, C {C})")


@pytest.mark.parametrize("C", [64, 128, 256, 512])
@pytest.mark.parametrize("up", [False, True])
def test_spatial_groupnorm_from_conv_epilogue_local(C, up):
    """statistics {sum, M2} from the epilogue of the convolution that produced x (plain and upsample tiles)"""
    B, H, W = 2, 128, 16
    y1 = _planted_conv_output(B, C, H, W, up, 1200 + C)
    assert getattr(y1, "_gn_stats", None) is not None
    ga, be = _gn_affine(C, 1201)
    zq = _latent(B, H // 4, W // 4, 4, 1202).to(DEV)
    cy, cb = _mod(C, 4, 1203)
    y = ops.conv2d(y1, _identity(C), gn=(ga.to(DEV), be.to(DEV), G, 1e-6, 1), spatial=(zq, cy, cb))
    torch.cuda.synchronize()
    _check(y, y1.permute(0, 3, 1, 2).cpu(), ga, be, zq, cy, cb, 1, "planes",
           f"(B {B}, {H}x{W}, C {C}, statistics from the {'upsample ' if up else ''}conv epilogue)")


def test_spatial_groupnorm_past_one_wave_local():
    """24 images of the MOVQ decoder's 32 x 32 x 512 level: many waves of apply blocks, latent ratio 4"""
    B, H, W, C = 24, 32, 32, 512
    x = _planted_gn(B, C, H * W, 1300).view(B, C, H, W)
    ga, be = _gn_affine(C, 1301)
    zq = _latent(B, 8, 8, 4, 1302).to(DEV)
    cy, cb = _mod(C, 4, 1303)
    y = ops.conv2d(x.permute(0, 2, 3, 1).contiguous().to(DEV), _identity(C), gn=(ga.to(DEV), be.to(DEV), G, 1e-6, 1),
                   spatial=(zq, cy, cb))
    _check(y, x, ga, be, zq, cy, cb, 1, "planes", f"(B {B}, {H}x{W} from 8x8, C {C})")


def test_spatial_groupnorm_four_channel_planes_exact():
    """C % 8 != 0 takes the four-channel plane kernel: its planes are the exact bf16 split of the fp32 output"""
    B, H, W, C, groups = 3, 20, 12, 4, 2
    x = torch.randn(B, H, W, C, device=DEV) * 3 + 1
    ga, be = 1 + 0.1 * torch.randn(C, device=DEV), 0.1 * torch.randn(C, device=DEV)
    zq = _latent(B, 5, 3, 4, 1400).to(DEV)
    cy, cb = _mod(C, 4, 1401)
    wy, by, wb, bb = (t.detach().reshape(C, -1).contiguous() for t in (cy.weight, cy.bias, cb.weight, cb.bias))
    ws, ss = ops._gn_scratch(x)
    y = torch.empty_like(x)
    hi, lo = torch.empty(x.shape, dtype=BF, device=DEV), torch.empty(x.shape, dtype=BF, device=DEV)
    st = ops._prep(x)
    for out in ((y, None, None), (None, hi, lo)):
        ops._call("muse_spatial_groupnorm_silu_nhwc", ops._p(x), ops._p(ga), ops._p(be), ops._p(zq), ops._p(wy), ops._p(by),
                  ops._p(wb), ops._p(bb), *map(ops._p, out), ops._p(ws), ops._p(ss), B, H, W, C, groups, 1e-6, 5, 3, 4, 0, 1,
                  st)
    h = y.to(BF)
    assert torch.equal(hi, h) and torch.equal(lo, (y - h.float()).to(BF))
    ref = F.group_norm(x.permute(0, 3, 1, 2).double().cpu(), groups, ga.double().cpu(), be.double().cpu(), 1e-6)
    z = F.interpolate(zq.permute(0, 3, 1, 2).double().cpu(), size=(H, W), mode="nearest")
    ref = F.silu(ref * F.conv2d(z, cy.weight.double().cpu(), cy.bias.double().cpu()) +
                 F.conv2d(z, cb.weight.double().cpu(), cb.bias.double().cpu())).permute(0, 2, 3, 1)
    assert float((y.cpu().double() - ref).norm() / ref.norm()) < 1e-6
