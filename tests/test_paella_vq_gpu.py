"""GPU: PaellaVQModel end to end against the outputs of the unmodified reference (tests/golden/micro_paella_vq.pt, f4 on
the tensor cores, f8 with its 48- / 96-wide levels on the fp32 SIMT route), the fp64 restatement (oracle/paella_vq_oracle.py)
at the default f4 architecture and 256 px on both routes, the C oracle's arg-min on the product's own z, the display
bytes of decode_code_uint8, and the launch count of a ResBlock (the fusion)."""
import pytest
import torch

from open_muse_b200 import PaellaVQModel, ops
from oracle import paella_vq_oracle as O
from oracle import vq_oracle
from tests import paella_fixture

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLD = torch.load(paella_fixture.PATH, weights_only=False)


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm())


def _model(name):
    g = GOLD[name]
    m = PaellaVQModel(**{k: v for k, v in g["config"].items() if not k.startswith("_")})
    m.load_state_dict(paella_fixture.state_dict(PaellaVQModel, GOLD, name), strict=True)
    return m.eval().to(DEV)


@pytest.mark.parametrize("name", ["f4", "f8"])
def test_fixture(name):
    g = GOLD[name]
    m = _model(name)
    img = g["image"].to(DEV)
    z = m._encode_nhwc(img)
    assert _rel(z.permute(0, 3, 1, 2), g["z"]) < 1e-4
    z_q, ids, loss = m.encode(img)
    assert loss is None
    sure = g["margin"] > 1e-3
    assert torch.equal(ids.cpu().reshape(-1)[sure], g["ids"].reshape(-1)[sure])
    cb = m.vquantizer.codebook.weight.detach().float().cpu().numpy()
    ids_o, _ = vq_oracle.argmin(z.reshape(-1, 4).cpu().numpy(), cb)
    assert (ids.cpu().reshape(-1).numpy() == ids_o).all()  # bit-exact on the product's own z
    assert torch.equal(m.get_code(img).cpu(), ids.cpu())
    dec = m.decode_code(g["ids"].to(DEV))
    assert _rel(dec, g["decode_code"]) < 1e-4
    # decode() multiplies by the scale factor, decode_code() does not; (x / s) * s is x to an fp32 ulp, which the decoder
    # carries through (measured 2.6e-6 on the f4 fixture)
    assert _rel(m.decode(m.vquantizer.get_codebook_entry(g["ids"].to(DEV)) / m.scale_factor), dec) < 1e-5
    if bool(sure.all()):
        assert _rel(m(img), g["forward"]) < 1e-4


def _default_f4(seed=0):
    torch.manual_seed(seed)
    m = PaellaVQModel()
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for k, p in m.named_parameters():
            if k.endswith("gammas"):
                p.copy_(torch.randn(6, generator=g) * 0.5)
        bn = m.down_blocks[-1][1]
        bn.running_mean.copy_(torch.randn(4, generator=g) * 0.2)
        bn.running_var.copy_(torch.rand(4, generator=g) + 0.5)
    return m.eval().to(DEV)


def test_default_f4_256px_routes_against_fp64():
    m = _default_f4()
    sd = {k: v.detach().to(DEV) for k, v in m.state_dict().items()}
    cfg = dict(m.config)
    img = torch.rand(1, 3, 256, 256, generator=torch.Generator().manual_seed(3)).to(DEV) * 2 - 1
    z64 = O.encoder(sd, cfg, img)
    with torch.no_grad():  # a codebook with the spread of z, so that the ids are not all near-ties
        cb = torch.randn(8192, 4, generator=torch.Generator().manual_seed(4)).to(DEV) * z64.std().float() + z64.mean().float()
        m.vquantizer.codebook.weight.copy_(cb)
    sd["vquantizer.codebook.weight"] = cb
    ids = m.get_code(img)
    z_tc = m._encode_nhwc(img).permute(0, 3, 1, 2)
    with ops.conv_route("simt"):
        z_simt = m._encode_nhwc(img).permute(0, 3, 1, 2)
        dec_simt = m.decode_code(ids)
    dec_tc = m.decode_code(ids)
    dec64 = O.decode_code(sd, cfg, ids)
    e = dict(z_tc=_rel(z_tc, z64), z_simt=_rel(z_simt, z64), z_routes=_rel(z_tc, z_simt), dec_tc=_rel(dec_tc, dec64),
             dec_simt=_rel(dec_simt, dec64), dec_routes=_rel(dec_tc, dec_simt))
    print("default f4 256 px rel-L2 vs fp64:", {k: f"{v:.2e}" for k, v in e.items()})
    assert e["z_tc"] < 1e-4 and e["z_simt"] < 1e-5 and e["z_routes"] < 1e-4, e
    assert e["dec_tc"] < 1e-4 and e["dec_simt"] < 1e-5 and e["dec_routes"] < 1e-4, e
    d = O.distances(sd, z64)
    top2 = d.topk(2, dim=1, largest=False).values.sqrt()
    sure = (top2[:, 1] - top2[:, 0]) > 1e-3
    assert int(sure.sum()) > 1000
    assert torch.equal(ids.reshape(-1)[sure], d.argmin(1)[sure])
    # the single-pass bf16 mode: same ids except near ties
    m.set_conv_precision("bf16")
    agree = float((m.get_code(img) == ids).float().mean())
    dec_bf = m.decode_code(ids)
    m.set_conv_precision("bf16x3")
    print(f"bf16 mode: id agreement {agree:.4f}, decode rel-L2 {_rel(dec_bf, dec64):.2e}")
    assert agree > 0.9 and _rel(dec_bf, dec64) < 3e-2


def test_decode_code_uint8_bytes():
    g = GOLD["f4"]
    m = _model("f4")
    ids = g["ids"].to(DEV)
    b = m.decode_code_uint8(ids)
    x = m.decode_code(ids).permute(0, 2, 3, 1)
    t = (torch.clamp(2.0 * x - 1.0, -1.0, 1.0) + 1.0) / 2.0  # pipeline_muse.py:245-252
    assert b.dtype == torch.uint8 and b.shape == (2, 64, 64, 3)
    assert torch.equal(b, (255.0 * t).to(torch.uint8))


@pytest.mark.parametrize("route", [None, "simt"])
def test_resblock_launch_count(route):
    m = _default_f4()
    blk = m.up_blocks[1]
    x = torch.randn(2, 64, 64, 384, device=DEV)
    with ops.conv_route(route):
        blk.run(x)
        n0 = ops.launches()
        blk.run(x)
        assert ops.launches() - n0 <= 4
