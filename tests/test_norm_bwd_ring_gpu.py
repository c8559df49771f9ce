"""The row-ring norm backward kernels (bulk copies into a shared-memory ring of rows) against the register-path kernels
they replace, bit for bit: dx / d[a | b] / d_a per row, and the weight gradients, which keep the register path's row
mapping and reduction order.  MUSE_NORM_BWD_RING=0 selects the register path."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from open_muse_b200 import ops  # noqa: E402

DEV = "cuda"
BF = torch.bfloat16
# below one CTA of 8 rows, not a multiple of the 8 rows a CTA takes per round, and the bench shape (many waves)
ROWS = [5, 4099, 65792]


def _with_ring(setting, fn):
    old = os.environ.get("MUSE_NORM_BWD_RING")
    os.environ["MUSE_NORM_BWD_RING"] = setting
    try:
        out = fn()
        torch.cuda.synchronize()
        return out
    finally:
        if old is None:
            del os.environ["MUSE_NORM_BWD_RING"]
        else:
            os.environ["MUSE_NORM_BWD_RING"] = old


def _same(fn):
    """fn() on the register path and on the ring: identical bits."""
    ref = _with_ring("0", fn)
    got = _with_ring("", fn)
    for i, (r, g) in enumerate(zip(ref, got)):
        assert r.dtype == g.dtype and r.shape == g.shape
        assert torch.equal(r.view(-1).view(torch.int16 if r.dtype == BF else torch.int32),
                           g.view(-1).view(torch.int16 if g.dtype == BF else torch.int32)), \
            f"output {i} differs: max |d| = {(r.float() - g.float()).abs().max().item()}"


def _rand(shape, seed, dtype=BF, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (scale * torch.randn(*shape, generator=g)).to(dtype).to(DEV)


def _weight(H, seed=7):
    return (1 + 0.1 * torch.randn(H, generator=torch.Generator().manual_seed(seed))).to(DEV)


@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("H", [512, 768, 1024])
@pytest.mark.parametrize("rms", [0, 1])
def test_norm_bwd_ring_matches_register_path(rows, H, rms):
    """The attention pre-norm backward (bf16 dy, fp32 x, + dres, bf16 copy of dx), and fp32 dy / bf16 x / bf16 dx."""
    x = _rand((rows, H), 1, torch.float32)
    w = _weight(H)
    _, st = ops.norm_fwd(x, w, 1e-6, BF, rms=rms)
    dy = _rand((rows, H), 2)
    dres = _rand((rows, H), 3, torch.float32)

    def with_dres():
        dx, dw = ops.norm_bwd(dy, x, w, st, torch.float32, dres=dres, rms=rms, want_dw=True, bf16_copy=True)
        return dx, dw, ops.take_bf16_copy(dx)

    _same(with_dres)
    xb, dyf = x.to(BF), dy.float()
    _, stb = ops.norm_fwd(xb, w, 1e-6, BF, rms=rms)
    _same(lambda: ops.norm_bwd(dyf, xb, w, stb, BF, dres=dres, rms=rms, want_dw=True))


@pytest.mark.parametrize("rows", [5, 4099])
def test_norm_bwd_ring_gelu_and_no_weight(rows):
    """act = 1 (GELU first) and a norm without weight or weight gradient, both with dres."""
    H = 768
    x = _rand((rows, H), 1, torch.float32)
    w = _weight(H)
    _, st = ops.norm_fwd(x, w, 1e-6, BF, act=1)
    dy = _rand((rows, H), 2)
    dres = _rand((rows, H), 3, torch.float32)
    _same(lambda: ops.norm_bwd(dy, x, w, st, torch.float32, dres=dres, act=1, want_dw=True))
    _same(lambda: (ops.norm_bwd(dy, x, None, st, torch.float32, dres=dres, act=1),))


@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("H,rms1", [(512, 0), (512, 1), (256, 1)])
def test_norm2_bwd_ring_matches_register_path(rows, H, rms1):
    a = _rand((rows, H), 1)
    res = _rand((rows, H), 2, torch.float32)
    w1, w2 = _weight(H, 3), _weight(H, 4)
    x2, _, st = ops.norm2_fwd(a, res, w1, w2, 1e-6, rms1=rms1, rms2=0)
    d_h2 = _rand((rows, H), 5)
    dres = _rand((rows, H), 6, torch.float32)
    _same(lambda: ops.norm2_bwd(d_h2, x2, w2, dres, a, w1, st, rms1=rms1, rms2=0))


@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("H,rms", [(512, 0), (768, 0), (1024, 1), (2048, 0), (2048, 1)])
def test_glu_norm_bwd_ring_matches_register_path(rows, H, rms):
    """The GLU + mid-norm backward with the saved forward output."""
    if rows == 65792 and H != 2048:
        pytest.skip("the bench shape is H = 2048")
    ab = _rand((rows, 2 * H), 1)
    w = _weight(H)
    dy = _rand((rows, H), 2)
    y, st = ops.norm_fwd(ab, w, 1e-6, BF, act=2, rms=rms)
    _same(lambda: ops.norm_bwd(dy, ab, w, st, BF, act=2, rms=rms, y_fwd=y, want_dw=True))

