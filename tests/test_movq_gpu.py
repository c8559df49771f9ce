"""GPU: MOVQ end to end against the outputs of the unmodified reference (tests/golden/micro_movq.pt: "tc" on the tensor
cores, "f8" with its narrow and 8 x 8 layers on the fp32 SIMT route), the fp64 restatement (oracle/movq_oracle.py) at the
class defaults and 256 px on both routes, the C oracle's arg-min on the product's own z, the display bytes of
decode_code_uint8, and the unmodified train_maskgit_imagenet.py with vq_model.type movq."""
import math
import os

import pytest
import torch
import yaml

from open_muse_b200 import MOVQ, ops
from oracle import movq_oracle as O
from oracle import vq_oracle
from tests import movq_fixture
from tests.train_script_harness import find_script, make_config, run_script

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLD = torch.load(movq_fixture.PATH, weights_only=False)


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm())


def _model(name):
    g = GOLD[name]
    m = MOVQ(**{k: v for k, v in g["config"].items() if not k.startswith("_")})
    m.load_state_dict(movq_fixture.state_dict(MOVQ, GOLD, name), strict=True)
    return m.eval().to(DEV)


def test_fixture_routes():
    """tc: every 3x3 convolution of both halves on the tensor cores; f8: the 32-wide level on the SIMT route"""
    for hw, c in ((64, 64), (32, 64), (16, 128)):
        assert ops.conv_uses_tensor_cores(hw, hw, c, c, 3), (hw, c)
    assert ops.conv_uses_tensor_cores(16, 16, 64, 128, 3) and ops.conv_uses_tensor_cores(32, 32, 128, 64, 3)
    assert not ops.conv_uses_tensor_cores(64, 64, 32, 32, 3)


@pytest.mark.parametrize("name", ["tc", "f8"])
def test_fixture(name):
    g = GOLD[name]
    m = _model(name)
    img = g["image"].to(DEV)
    z = m._encode_nhwc(img)
    e_z = _rel(z.permute(0, 3, 1, 2), g["z"])
    z_q, ids = m.encode(img)
    sure = g["margin"] > 1e-3
    assert torch.equal(ids.cpu().reshape(-1)[sure], g["ids"].reshape(-1)[sure])
    cb = m.quantize.embedding.weight.detach().float().cpu().numpy()
    ids_o, _ = vq_oracle.argmin(z.reshape(-1, 4).cpu().numpy(), cb)
    assert (ids.cpu().reshape(-1).numpy() == ids_o).all()  # bit-exact on the product's own z
    assert torch.equal(m.get_code(img).cpu(), ids.cpu())
    e_dec = _rel(m.decode_code(g["ids"].to(DEV)), g["decode_code"])
    rec, fwd_ids = m(img)
    assert torch.equal(fwd_ids, ids)
    e_fwd = _rel(rec, g["forward"]) if bool(sure.all()) else float("nan")
    print(f"movq fixture {name}: rel-L2 z {e_z:.2e}, decode_code {e_dec:.2e}, forward {e_fwd:.2e}")
    assert e_z < 1e-4 and e_dec < 1e-4
    if bool(sure.all()):
        assert e_fwd < 1e-4


def test_default_256px_routes_against_fp64():
    torch.manual_seed(0)
    m = MOVQ().eval().to(DEV)
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    cfg = dict(m.config)
    img = torch.rand(2, 3, 256, 256, generator=torch.Generator().manual_seed(3)).to(DEV) * 2 - 1
    with torch.no_grad():
        z64 = O.encoder(sd, cfg, img)
        # a codebook with the spread of z, so that the ids are not all near-ties
        cb = torch.randn(16384, 4, generator=torch.Generator().manual_seed(4)).to(DEV) * z64.std().float() + z64.mean().float()
        m.quantize.embedding.weight.copy_(cb)
    sd["quantize.embedding.weight"] = cb
    ids = m.get_code(img)
    z_tc = m._encode_nhwc(img).permute(0, 3, 1, 2)
    with ops.conv_route("simt"):
        z_simt = m._encode_nhwc(img).permute(0, 3, 1, 2)
        dec_simt = m.decode_code(ids)
    dec_tc = m.decode_code(ids)
    with torch.no_grad():
        dec64 = O.decode_code(sd, cfg, ids)
    e = dict(z_tc=_rel(z_tc, z64), z_simt=_rel(z_simt, z64), z_routes=_rel(z_tc, z_simt), dec_tc=_rel(dec_tc, dec64),
             dec_simt=_rel(dec_simt, dec64), dec_routes=_rel(dec_tc, dec_simt))
    print("MOVQ class defaults, 256 px, batch 2, rel-L2 vs fp64:", {k: f"{v:.2e}" for k, v in e.items()})
    assert e["z_tc"] < 1e-4 and e["z_simt"] < 2e-5 and e["z_routes"] < 1e-4, e
    assert e["dec_tc"] < 1e-4 and e["dec_simt"] < 2e-5 and e["dec_routes"] < 1e-4, e
    d = O.distances(sd, z64)
    top2 = d.topk(2, dim=1, largest=False).values.sqrt()
    sure = (top2[:, 1] - top2[:, 0]) > 1e-3
    assert int(sure.sum()) > 1500
    assert torch.equal(ids.reshape(-1)[sure], d.argmin(1)[sure])
    m.set_conv_precision("bf16")
    agree = float((m.get_code(img) == ids).float().mean())
    dec_bf = m.decode_code(ids)
    m.set_conv_precision("bf16x3")
    print(f"bf16 mode: id agreement {agree:.4f}, decode rel-L2 {_rel(dec_bf, dec64):.2e}")
    assert agree > 0.85 and _rel(dec_bf, dec64) < 3e-2  # measured 0.898: 16384 codes in D = 4 leave many near-ties


def test_decode_code_uint8_bytes():
    g = GOLD["tc"]
    m = _model("tc")
    ids = g["ids"].to(DEV)
    b = m.decode_code_uint8(ids)
    x = m.decode_code(ids).permute(0, 2, 3, 1)
    t = (torch.clamp(2.0 * x - 1.0, -1.0, 1.0) + 1.0) / 2.0  # pipeline_muse.py:245-252
    assert b.dtype == torch.uint8 and b.shape == (2, 64, 64, 3)
    assert torch.equal(b, (255.0 * t).to(torch.uint8))


SCRIPT = find_script()


@pytest.mark.skipif(SCRIPT is None, reason="reference training script not available (build() snapshots it into oracle/_ref)")
def test_reference_training_script_runs_with_movq(tmp_path, monkeypatch):
    monkeypatch.setenv("WANDB_MODE", "disabled")
    steps = 3
    cfg_path, _ = make_config(str(tmp_path), steps=steps, batch=8, mixed_precision="bf16")
    torch.manual_seed(6)
    vq_dir = str(tmp_path / "movq")  # 32 px -> 16 x 16 = 256 tokens over 64 codes, as the harness's transformer expects
    MOVQ(resolution=32, hidden_channels=32, channel_mult=(1, 2), num_res_blocks=1, attn_resolutions=(16,),
         num_embeddings=64).save_pretrained(vq_dir)
    cfg = yaml.safe_load(open(cfg_path))
    cfg["model"]["vq_model"] = {"type": "movq", "pretrained": vq_dir}
    with open(cfg_path, "w") as f:
        yaml.safe_dump(cfg, f)
    n0 = ops.launches()
    acc = run_script(SCRIPT, cfg_path)
    assert ops.launches() - n0 > 100 * steps
    losses = [v["step_loss"] for v, s in acc.logged if "step_loss" in v]
    assert len(losses) == steps and all(math.isfinite(x) for x in losses)
    assert os.path.isdir(tmp_path / "movq")
