"""Every pixel and tile of the Paella tokenizer kernels against fp64 (tests/local_error.check_local), with the bounds below.

* the ResBlock spatial pass (csrc/paella.cu): one group per pixel row of x1 and of LN2(x1); the image borders carry 4x
  values, so a wrong replication pad is one bad border pixel, not a small whole-tensor error;
* the GELU epilogue of the tensor-core convolution, per 128-pixel x N tile, with a ragged second N tile and persistent
  CTAs that take a second tile;
* ConvTranspose2d(4, 2, 1) per parity tile and Conv2d(4, 2, 1) per tile on the tensor cores (again past one wave), and
  both plus the PixelUnshuffle stem and the PixelShuffle store on the fp32 SIMT route, per pixel row;
* the quantiser at D = 4, bit-exact against oracle/vq_oracle.c.
References are fp64 from exactly the fp32 operands the kernels receive."""
import pytest
import torch
import torch.nn.functional as F

from open_muse_b200 import ops
from oracle import vq_oracle
from tests.local_error import check_local, conv_tiles
from tests.local_error import rows as by_row

pytestmark = pytest.mark.gpu
DEV = "cuda"
F64 = torch.float64

# (group bound, element bound), relative to the group's norm (check_local)
B_SPATIAL = (2e-6, 1e-5)   # fp32 LayerNorm + 9-tap fma chain: a few ulp
B_PLANES = (1e-5, 1e-4)    # the same written as bf16 hi + lo planes
B_TC = (3e-5, 2e-4)        # bf16x3 operands (the lo*lo term dropped, ~2^-18 per product) and fp32 accumulation
B_SIMT = (2e-6, 2e-5)      # fp32 fma chains of length K


def _nchw(x):
    return x.permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def _bordered(B, H, W, C, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, H, W, C, generator=g) + 0.3 * torch.randn(B, 1, 1, C, generator=g)
    x[:, 0] *= 4; x[:, -1] *= 4; x[:, :, 0] *= 4; x[:, :, -1] *= 4
    return x.to(DEV)


def _ln64(x):
    x = x.double()
    return (x - x.mean(-1, keepdim=True)) / torch.sqrt(x.var(-1, unbiased=False, keepdim=True) + 1e-6)


@pytest.mark.parametrize("B,H,W,C", [(2, 16, 16, 64), (3, 9, 7, 1024), (1, 32, 32, 200)])
@pytest.mark.parametrize("split", [False, True])
def test_spatial_pass(B, H, W, C, split):
    x = _bordered(B, H, W, C, 1)
    wk = torch.randn(9, C, device=DEV) * 0.3
    bias = torch.randn(C, device=DEV) * 0.1
    st = ops._prep(x)
    stats = torch.empty(2 * B * H * W, device=DEV)
    x1 = torch.empty_like(x)
    if split:
        hi = torch.empty(x.shape, dtype=torch.bfloat16, device=DEV)
        lo = torch.empty_like(hi)
        ops._call("muse_paella_resblock_spatial", ops._p(x), ops._p(wk), ops._p(bias), ops._p(stats), ops._p(x1), None,
                  ops._p(hi), ops._p(lo), B, H, W, C, 1e-6, st)
        n2 = hi.float() + lo.float()
    else:
        n2 = torch.empty_like(x)
        ops._call("muse_paella_resblock_spatial", ops._p(x), ops._p(wk), ops._p(bias), ops._p(stats), ops._p(x1),
                  ops._p(n2), None, None, B, H, W, C, 1e-6, st)
    t = F.pad(_nchw(_ln64(x)), (1, 1, 1, 1), mode="replicate")
    ref1 = x.double() + _nhwc(F.conv2d(t, wk.double().t().reshape(C, 1, 3, 3), bias.double(), groups=C))
    groups = by_row(B * H * W, "pixel")
    check_local(x1, ref1, groups, *B_SPATIAL, f"spatial x1 {B}x{H}x{W}x{C}")
    # LN2 of the kernel's own x1 (fp32), so the check isolates the second norm.  As planes, lo = bf16(v - hi) carries v to
    # 2^-18 |v| per element (measured: 3.6e-6 per pixel, 3.0e-5 per element relative to the pixel's rms)
    check_local(n2, _ln64(x1), groups, *(B_PLANES if split else B_SPATIAL), f"spatial n2 {B}x{H}x{W}x{C}")


def _planes(t):
    hi = t.to(torch.bfloat16)
    return hi, (t - hi.float()).to(torch.bfloat16)


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 16, 16, 64, 256), (3, 64, 64, 128, 320), (1, 32, 32, 192, 768)])
def test_gelu_epilogue(B, H, W, Cin, Cout):
    g = torch.Generator().manual_seed(2)
    x = torch.randn(B, H, W, Cin, generator=g).to(DEV)
    w = (torch.randn(Cout, Cin, generator=g) * Cin ** -0.5).to(DEV)
    b = (torch.randn(Cout, generator=g) * 0.5).to(DEV)
    (xh, xl), (wh, wl) = _planes(x), _planes(w)
    yh = torch.empty(B, H, W, Cout, dtype=torch.bfloat16, device=DEV)
    yl = torch.empty_like(yh)
    ops._call("muse_conv2d_nhwc_tc_gelu_split", ops._p(xh), ops._p(xl), ops._p(wh), ops._p(wl), ops._p(b), ops._p(yh),
              ops._p(yl), B, H, W, Cin, Cout, 1, 0, ops._prep(x))
    ref = F.gelu(x.double() @ w.double().t() + b.double())
    check_local(yh.float() + yl.float(), ref, conv_tiles(B, H, W, Cout), *B_TC, f"gelu epilogue {B}x{H}x{W} {Cin}->{Cout}")


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 16, 16, 128, 64), (40, 16, 16, 64, 128)])
def test_transposed_conv(B, H, W, Cin, Cout):
    x = _bordered(B, H, W, Cin, 3)
    w = torch.randn(Cin, Cout, 4, 4, device=DEV) * (4 * Cin) ** -0.5
    b = torch.randn(Cout, device=DEV) * 0.1
    ref = _nhwc(F.conv_transpose2d(_nchw(x).double(), w.double(), b.double(), stride=2, padding=1))
    y = ops.conv_transpose2d_s2(x, w, b)
    check_local(y, ref, conv_tiles(B, 2 * H, 2 * W, Cout, up=True), *B_TC, f"conv_transpose tc B={B} {Cin}->{Cout}")
    with ops.conv_route("simt"):
        y = ops.conv_transpose2d_s2(x, w, b)
    check_local(y, ref, by_row(B * 4 * H * W, "pixel"), *B_SIMT, f"conv_transpose simt B={B} {Cin}->{Cout}")


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 32, 32, 64, 128), (20, 32, 32, 96, 192), (2, 16, 16, 48, 96)])
def test_strided_conv(B, H, W, Cin, Cout):
    x = _bordered(B, 2 * H, 2 * W, Cin, 4)
    w = torch.randn(Cout, Cin, 4, 4, device=DEV) * (16 * Cin) ** -0.5
    b = torch.randn(Cout, device=DEV) * 0.1
    ref = _nhwc(F.conv2d(_nchw(x).double(), w.double(), b.double(), stride=2, padding=1))
    y = ops.conv2d_s2p1(x, w, b)
    if (4 * Cin) % 64 == 0:  # the tensor-core route (space-to-depth + 3x3 over 4 * Cin planes)
        check_local(y, ref, conv_tiles(B, H, W, Cout), *B_TC, f"conv4x4s2 tc B={B} {Cin}->{Cout}")
    with ops.conv_route("simt"):
        y = ops.conv2d_s2p1(x, w, b)
    check_local(y, ref, by_row(B * H * W, "pixel"), *B_SIMT, f"conv4x4s2 simt B={B} {Cin}->{Cout}")


@pytest.mark.parametrize("route", [None, "simt"])
def test_unshuffle_stem_and_shuffle_store(route):
    B, H, W = 2, 64, 64
    x = _bordered(B, 2 * H, 2 * W, 3, 5)
    w = torch.randn(128, 12, 1, 1, device=DEV) * 0.3
    b = torch.randn(128, device=DEV) * 0.1
    bound = B_SIMT if route else B_TC
    with ops.conv_route(route):
        y = ops.conv2d_unshuffle(x, w, b)
        ref = _nhwc(F.conv2d(F.pixel_unshuffle(_nchw(x).double(), 2), w.double(), b.double()))
        check_local(y, ref, by_row(B * H * W, "pixel"), *bound, f"unshuffle stem {route}")
        w2 = torch.randn(12, 128, 1, 1, device=DEV) * 0.1
        b2 = torch.randn(12, device=DEV) * 0.1
        out = ops.conv1x1_pixel_shuffle(y, w2, b2)
        ref2 = _nhwc(F.pixel_shuffle(F.conv2d(_nchw(y).double(), w2.double(), b2.double()), 2))
        check_local(out, ref2, by_row(B * 2 * H * W, "pixel"), *bound, f"pixel-shuffle store {route}")


def test_quantiser_d4_bit_exact():
    g = torch.Generator().manual_seed(6)
    z = torch.randn(20000, 4, generator=g)
    cb = torch.randn(8192, 4, generator=g)
    z[:64] = cb[:64]  # exact hits
    cb[100] = cb[101]  # a tie: the lower index wins
    z[64] = cb[101]
    ids, dmin = ops.vq_argmin(z.to(DEV), cb.to(DEV), return_dmin=True)
    ids_o, dmin_o = vq_oracle.argmin(z.numpy(), cb.numpy())
    assert (ids.cpu().numpy() == ids_o).all() and (dmin.cpu().numpy() == dmin_o).all()
    assert int(ids[64]) == 100
    soft, sids = ops.vq_soft_code(z[:512].to(DEV), cb.to(DEV), 1.0)
    assert (sids.cpu().numpy() == ids_o[:512]).all()
    assert torch.allclose(soft.sum(1), torch.ones(512, device=DEV), atol=1e-5)
