"""CPU: the host layer of the tokenizer convolutions (open_muse_b200/ops.py) -- the weight-pack cache, the packed weight
layouts each entry point hands the library, the route and the launch modes -- with the launches recorded instead of run.
The route queries are host functions of the library and need no GPU."""
import os
import re

import pytest
import torch
import torch.nn.functional as F

from open_muse_b200 import _lib, ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONV_CALLS = ("muse_conv2d_nhwc", "muse_conv2d_nhwc_tc", "muse_conv2d_nhwc_tc_gelu_split")


@pytest.fixture
def calls(monkeypatch):
    """Launches as (name, args), with the tensors themselves in the pointer slots."""
    from open_muse_b200 import build

    build.build()
    rec = []
    monkeypatch.setattr(ops, "_prep", lambda t: 0)
    monkeypatch.setattr(ops, "_p", lambda t: t)
    monkeypatch.setattr(ops, "_call", lambda name, *args: rec.append((name, args)))
    monkeypatch.setattr(ops, "_wk_cache", {})
    return rec


def _w(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def _tc_weight(calls):
    """fp64 hi + lo of the weight planes of the one tensor-core launch recorded."""
    (args,) = [a for n, a in calls if n == "muse_conv2d_nhwc_tc"]
    return args[2].double() + args[3].double()


def _simt_weight(calls):
    (args,) = [a for n, a in calls if n == "muse_conv2d_nhwc"]
    return args[1].double()


def _close(got, ref):
    torch.testing.assert_close(got, ref, rtol=0, atol=1e-5 * float(ref.abs().max()))


# ---------------------------------------------------------------------------------------------------- the cache
def test_pack_cache_hits_only_the_same_unchanged_tensor(monkeypatch):
    monkeypatch.setattr(ops, "_wk_cache", {})
    packs = []

    def pack(wf):
        packs.append(wf)
        return wf * 2

    w = _w(8, 4, 3, 3)
    first = ops._cached_pack("t", w, pack)
    assert ops._cached_pack("t", w, pack) is first and len(packs) == 1  # hit
    with torch.no_grad():
        w.add_(1.0)  # in-place update: the version counter moves
    torch.testing.assert_close(ops._cached_pack("t", w, pack), w * 2)
    assert len(packs) == 2
    ops._cached_pack("u", w, pack)  # another packing of the same tensor is a separate entry
    assert len(packs) == 3
    # a new tensor object at a recycled id(): same storage, version, shape and device, only the weakref tells them apart
    monkeypatch.setattr(ops, "id", lambda obj: 7, raising=False)
    ops._cached_pack("t", w, pack)
    alias = w.view(w.shape)
    assert alias is not w and alias.data_ptr() == w.data_ptr() and alias._version == w._version
    ops._cached_pack("t", alias, pack)
    assert len(packs) == 5


def test_pack_cache_is_bounded(monkeypatch):
    monkeypatch.setattr(ops, "_wk_cache", {})
    monkeypatch.setattr(ops, "_WK_CACHE_ENTRIES", 3)
    weights = [_w(4, seed=i) for i in range(10)]
    for w in weights:
        ops._cached_pack("t", w, torch.clone)
        assert len(ops._wk_cache) <= 4


# ---------------------------------------------------------------------------------------------------- packed layouts
def _parity_conv(v, wk, Cout):
    """Four 2x2 parity convolutions of v [B, Cin, h, w] with wk [4*Cout, 4*Cin] (row parity*Cout + co, column
    (a*2+b)*Cin + ci): output pixel (2y+py, 2x+px) reads v[y+a+py-1, x+b+px-1]."""
    B, Cin, h, w = v.shape
    vp = F.pad(v, (1, 1, 1, 1))
    y = torch.zeros(B, Cout, 2 * h, 2 * w, dtype=torch.float64)
    for py in (0, 1):
        for px in (0, 1):
            m = wk[(2 * py + px) * Cout:(2 * py + px + 1) * Cout].view(Cout, 2, 2, Cin)
            for a in (0, 1):
                for b in (0, 1):
                    window = vp[:, :, a + py:a + py + h, b + px:b + px + w]
                    y[:, :, py::2, px::2] += torch.einsum("oc,bchw->bohw", m[:, a, b], window)
    return y


def _s2d_conv(x, wk, taps, off):
    """Convolution over the space-to-depth grid of x [B, Cin, 2H, 2W] with wk [Cout, taps*taps*4*Cin] (column
    ((a*taps + b)*4 + p*2 + q)*Cin + ci): y[Y, X] reads x[2(Y + a + off) + p, 2(X + b + off) + q], zero outside."""
    B, Cin, Hi, Wi = x.shape
    H, W = Hi // 2, Wi // 2
    m = wk.view(wk.shape[0], taps, taps, 2, 2, Cin)
    pad = 2 * taps
    xp = F.pad(x, (pad, pad, pad, pad))
    y = torch.zeros(B, wk.shape[0], H, W, dtype=torch.float64)
    for a in range(taps):
        for b in range(taps):
            for p in (0, 1):
                for q in (0, 1):
                    r0, c0 = pad + 2 * (a + off) + p, pad + 2 * (b + off) + q
                    y += torch.einsum("oc,bchw->bohw", m[:, a, b, p, q], xp[:, :, r0:r0 + 2 * H:2, c0:c0 + 2 * W:2])
    return y


def test_upsample_parities_pack_the_nearest_x2_conv(calls):
    x, w = _w(1, 16, 16, 64), _w(32, 64, 3, 3, seed=1)
    ops.conv2d(x, w, upsample2x=True)
    assert [a[14] for n, a in calls if n == "muse_conv2d_nhwc_tc"] == [_lib.CONV_TC_UPSAMPLE2X]
    v = x.permute(0, 3, 1, 2).double()
    _close(_parity_conv(v, _tc_weight(calls), 32), F.conv2d(F.interpolate(v, scale_factor=2), w.double(), padding=1))


def test_stride2_space_to_depth_pack(calls):
    x, w = _w(1, 32, 32, 64), _w(32, 64, 3, 3, seed=1)
    ops.conv2d_down(x, w)
    v = x.permute(0, 3, 1, 2).double()
    _close(_s2d_conv(v, _tc_weight(calls), 2, 0), F.conv2d(F.pad(v, (0, 1, 0, 1)), w.double(), stride=2))


def test_s2p1_pack(calls):
    x, w = _w(1, 32, 32, 16), _w(32, 16, 4, 4, seed=1)
    ops.conv2d_s2p1(x, w)
    v = x.permute(0, 3, 1, 2).double()
    _close(_s2d_conv(v, _tc_weight(calls), 3, -1), F.conv2d(v, w.double(), stride=2, padding=1))


@pytest.mark.parametrize("route", [None, "simt"])
def test_transposed_parities_pack(calls, route):
    x, w = _w(1, 16, 16, 64), _w(64, 32, 4, 4, seed=1)
    with ops.conv_route(route):
        ops.conv_transpose2d_s2(x, w)
    # SIMT: the same four matrices, each transposed to [4*Cin, Cout]
    wk = _tc_weight(calls) if route is None else _simt_weight(calls).transpose(1, 2).reshape(4 * 32, -1)
    v = x.permute(0, 3, 1, 2).double()
    _close(_parity_conv(v, wk, 32), F.conv_transpose2d(v, w.double(), stride=2, padding=1))


def test_stem_pack_is_64_tap_major_columns(calls):
    x, w = _w(1, 16, 16, 3), _w(32, 3, 3, 3, seed=1)
    ops.conv2d(x, w)
    wk = _tc_weight(calls)
    assert wk.shape == (32, 64) and not wk[:, 27:].any()
    v = F.pad(x.permute(0, 3, 1, 2).double(), (1, 1, 1, 1))
    cols = torch.stack([v[:, ci, kh:kh + 16, kw:kw + 16] for kh in range(3) for kw in range(3) for ci in range(3)], 1)
    ref = F.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), padding=1)
    _close(torch.einsum("oc,bchw->bohw", wk[:, :27], cols), ref)


@pytest.mark.parametrize("route", [None, "simt"])
def test_unshuffle_pack(calls, route):
    Cin = 3 if route is None else 32  # the tensor-core form needs 4*Cin <= 64
    x, w = _w(1, 32, 32, Cin), _w(32, 4 * Cin, 1, 1, seed=1)
    with ops.conv_route(route):
        ops.conv2d_unshuffle(x, w)
    v = x.permute(0, 3, 1, 2).double()
    # x[2Y + dy, 2X + dx, c] pairs with column c*4 + dy*2 + dx (tensor cores: the im2col row) or with row
    # (dy*2 + dx)*Cin + c of the [K, Cout] SIMT weights
    if route is None:
        wk = _tc_weight(calls)[:, :4 * Cin].view(32, Cin, 2, 2)
    else:
        wk = _simt_weight(calls).view(2, 2, Cin, 32).permute(3, 2, 0, 1)
    y = sum(torch.einsum("oc,bchw->bohw", wk[:, :, dy, dx], v[:, :, dy::2, dx::2]) for dy in (0, 1) for dx in (0, 1))
    _close(y, F.conv2d(F.pixel_unshuffle(v, 2), w.double()))


# ---------------------------------------------------------------------------------------------------- route and modes
def _every_entry_point():
    g = (_w(64), _w(64, seed=2), 32, 1e-6)
    zq = (_w(1, 4, 4, 4), torch.nn.Conv2d(4, 64, 1), torch.nn.Conv2d(4, 64, 1))
    ops.conv2d(_w(1, 16, 16, 3), _w(64, 3, 3, 3))
    ops.conv2d(_w(1, 16, 16, 64), _w(64, 64, 3, 3), residual=_w(1, 16, 16, 64))
    ops.conv2d(_w(1, 16, 16, 64), _w(64, 64, 3, 3), upsample2x=True)
    ops.conv2d(_w(1, 8, 8, 64), _w(64, 64, 3, 3), upsample2x=True)
    ops.conv2d(_w(1, 16, 16, 64), _w(64, 64, 3, 3), gn=g)
    ops.conv2d(_w(1, 16, 16, 64), _w(3, 64, 3, 3), gn=g + (0,), spatial=zq)
    ops.groupnorm_silu(_w(1, 16, 16, 64), *g)
    ops.conv2d_down(_w(1, 32, 32, 64), _w(64, 64, 3, 3))
    ops.attention_single_head(_w(256, 64), _w(256, 64), _w(256, 64), 1, 16, 16)
    ops.paella_resblock(_w(1, 16, 16, 64), _w(9, 64), _w(64), _w(256, 64, 1, 1), _w(256), _w(64, 256, 1, 1), _w(64))
    ops.conv2d_unshuffle(_w(1, 32, 32, 3), _w(64, 12, 1, 1))
    ops.conv2d_s2p1(_w(1, 32, 32, 16), _w(64, 16, 4, 4))
    ops.conv_transpose2d_s2(_w(1, 16, 16, 64), _w(64, 32, 4, 4))
    ops.conv1x1_pixel_shuffle(_w(1, 16, 16, 64), _w(12, 64, 1, 1))


def test_simt_route_sends_every_convolution_to_the_fp32_kernel(calls):
    with ops.conv_route("simt"):
        _every_entry_point()
        assert not any(ops.conv_uses_tensor_cores(16, 16, c, 64, 3) for c in (3, 64, 512))
    assert all(ops.conv_uses_tensor_cores(16, 16, c, 64, 3) for c in (3, 64, 512))
    names = {n for n, _ in calls}
    assert "muse_conv2d_nhwc" in names
    assert not names & {"muse_conv2d_nhwc_tc", "muse_conv2d_nhwc_tc_gelu_split", "muse_split_bf16_nhwc",
                        "muse_split_s2d_bf16_nhwc", "muse_im2col_split_nhwc"}, names


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_single_pass_bit_follows_the_precision_but_not_attention(calls, precision):
    with ops.conv_precision(precision):
        _every_entry_point()
    tc = [(n, a[-2]) for n, a in calls if n in CONV_CALLS[1:]]
    assert {n for n, _ in tc} == set(CONV_CALLS[1:])
    attention = [m for _, m in tc if m & _lib.CONV_TC_PER_IMAGE_WEIGHTS]
    assert len(attention) == 2 and not any(m & _lib.CONV_TC_SINGLE_PASS for m in attention)
    others = [m for _, m in tc if not m & _lib.CONV_TC_PER_IMAGE_WEIGHTS]
    assert len(others) > 10
    assert all(bool(m & _lib.CONV_TC_SINGLE_PASS) == (precision == "bf16") for m in others)


def test_launch_modes_mirror_the_header():
    header = open(os.path.join(ROOT, "include", "muse_b200.h")).read()
    declared = {name: int(v) for name, v in re.findall(r"\bMUSE_(CONV_\w+) = (\d+)", header)}
    mirrored = {name: getattr(_lib, name) for name in dir(_lib) if name.startswith("CONV_")}
    assert declared and declared == mirrored
