"""CPU: PaellaVQModel's host wiring (module order, gamma / BatchNorm folds, layouts, the quantiser hand-off, the entry
points' scale-factor quirks) against the outputs of the UNMODIFIED reference (tests/golden/micro_paella_vq.pt), with the
kernels replaced by torch restatements: tests/cpu_math_ops.py for the existing ops, and below for the five Paella ops, each
the documented contract of its ops wrapper.  The kernels themselves are checked on the GPU (test_paella_vq_gpu.py,
test_paella_vq_local_gpu.py)."""
import json
import math

import pytest
import torch
import torch.nn.functional as F
import yaml

from oracle import paella_vq_oracle as O
from tests import cpu_math_ops, paella_fixture

GOLD = torch.load(paella_fixture.PATH, weights_only=False)
_SD = {}


def _sd(name):
    """the fixture's state dict, rebuilt from its seeds and checked against the reference's (tests/paella_fixture.py)"""
    from open_muse_b200 import PaellaVQModel

    if name not in _SD:
        _SD[name] = paella_fixture.state_dict(PaellaVQModel, GOLD, name)
    return _SD[name]


def _nchw(x):
    return x.permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


# ---- contracts of the Paella ops (open_muse_b200/ops.py), fp32 NHWC in and out
def paella_resblock(x, wk, bias, w1, b1, w2, b2, eps=1e-6):
    """x1 = x + dw(LN1 x) (replication pad, wk [9, C] tap-major), y = x1 + Lin2(GELU(Lin1(LN2 x1)))"""
    C = x.shape[3]
    t = F.pad(_nchw(F.layer_norm(x, (C,), eps=eps)), (1, 1, 1, 1), mode="replicate")
    x1 = x + _nhwc(F.conv2d(t, wk.t().reshape(C, 1, 3, 3), bias, groups=C))
    h = F.gelu(F.layer_norm(x1, (C,), eps=eps) @ w1[:, :, 0, 0].t() + b1)
    return (x1 + h @ w2[:, :, 0, 0].t() + b2).contiguous()


def conv2d_unshuffle(x, w, bias=None):
    return _nhwc(F.conv2d(F.pixel_unshuffle(_nchw(x), 2), w.float(), bias))


def conv2d_s2p1(x, w, bias=None):
    return _nhwc(F.conv2d(_nchw(x), w.float(), bias, stride=2, padding=1))


def conv_transpose2d_s2(x, w, bias=None):
    return _nhwc(F.conv_transpose2d(_nchw(x), w.float(), bias, stride=2, padding=1))


def conv1x1_pixel_shuffle(x, w, bias=None):
    return _nhwc(F.pixel_shuffle(F.conv2d(_nchw(x), w.float(), bias), 2))


PAELLA_STAND_INS = dict(paella_resblock=paella_resblock, conv2d_unshuffle=conv2d_unshuffle, conv2d_s2p1=conv2d_s2p1,
                        conv_transpose2d_s2=conv_transpose2d_s2, conv1x1_pixel_shuffle=conv1x1_pixel_shuffle)


def install(mp, exact=True):
    from open_muse_b200 import ops

    cpu_math_ops.install(mp, exact=exact)
    for name, fn in PAELLA_STAND_INS.items():
        mp.setattr(ops, name, fn)


def _model(name):
    from open_muse_b200 import PaellaVQModel

    g = GOLD[name]
    m = PaellaVQModel(**{k: v for k, v in g["config"].items() if not k.startswith("_")})
    m.load_state_dict(_sd(name), strict=True)
    return m.eval()


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


@pytest.mark.parametrize("name", ["f4", "f8"])
def test_wiring_reproduces_reference(monkeypatch, name):
    install(monkeypatch)
    g = GOLD[name]
    m = _model(name)
    z = m._encode_nhwc(g["image"])
    assert _rel(_nchw(z), g["z"]) < 2e-5
    z_q, ids, loss = m.encode(g["image"])
    assert loss is None and ids.shape == g["ids"].shape
    sure = g["margin"] > 1e-4
    assert torch.equal(ids.reshape(-1)[sure], g["ids"].reshape(-1)[sure])
    if bool(sure.all()):
        assert torch.equal(z_q, g["z_q"])
    entry = m.vquantizer.get_codebook_entry(g["ids"])
    cb = g["codebook"]
    s = int(math.sqrt(g["ids"].shape[1]))
    assert torch.equal(entry, cb[g["ids"]].reshape(2, s, s, -1).permute(0, 3, 1, 2))
    dec = m.decode_code(g["ids"])
    assert _rel(dec, g["decode_code"]) < 2e-5
    # decode() multiplies by the scale factor, decode_code() does not: decode(z_q / scale) == decode_code(ids)
    assert _rel(m.decode(entry / m.scale_factor), dec) < 1e-6
    assert _rel(m(g["image"]), g["forward"]) < 2e-5
    assert torch.equal(m.get_code(g["image"]).reshape(-1)[sure], g["ids"].reshape(-1)[sure])


def test_margin_coverage():
    sure = sum(int((GOLD[n]["margin"] > 1e-4).sum()) for n in ("f4", "f8"))
    assert sure > 400


@pytest.mark.parametrize("name", ["f4", "f8"])
def test_oracle_reproduces_reference(name):
    g = GOLD[name]
    cfg = g["config"]
    sd = _sd(name)
    z = O.encoder(sd, cfg, g["image"])
    assert _rel(z, g["z"]) < 1e-5
    d = O.distances(sd, z)
    sure = g["margin"] > 1e-4
    assert torch.equal(d.argmin(1)[sure], g["ids"].reshape(-1)[sure])
    assert _rel(O.decode_code(sd, cfg, g["ids"]), g["decode_code"]) < 1e-5


@pytest.mark.parametrize("name", ["f4", "f8"])
def test_seeded_construction_and_state_dict(name):
    from open_muse_b200 import PaellaVQModel

    g = GOLD[name]
    torch.manual_seed(g["seed"])
    m = PaellaVQModel(**{k: v for k, v in g["config"].items() if not k.startswith("_")})
    sd = m.state_dict()
    assert list(sd) == list(g["init_signature"])
    for k, (s, n) in g["init_signature"].items():
        assert float(sd[k].double().sum()) == pytest.approx(s, rel=1e-9, abs=1e-9), k
        assert float(sd[k].double().norm()) == pytest.approx(n, rel=1e-9, abs=1e-9), k
    m.load_state_dict(_sd(name), strict=True)
    assert set(m.state_dict()) == set(g["state_signature"])
    assert int(m.state_dict()["down_blocks.{}.1.num_batches_tracked".format(len(m.down_blocks) - 1)]) == 123


def test_quirks(monkeypatch):
    install(monkeypatch)
    from open_muse_b200 import PaellaVQModel

    g = GOLD["f4"]
    m = _model("f4")
    with pytest.raises(ValueError):
        z_q, ids = m.encode(g["image"])  # 3 values (PipelineMuseInpainting :412 and train_muse :1145 unpack two)
    with pytest.raises(AttributeError):
        m.get_soft_code(g["image"])  # training.use_soft_code_target upstream (train_muse.py:625)
    soft, code = m.vquantizer.get_soft_code(_nchw(m._encode_nhwc(g["image"])))
    assert soft.shape == (2, 256, 512) and torch.allclose(soft.sum(-1), torch.ones(2, 256), atol=1e-5)
    with pytest.raises(NotImplementedError):
        m.train().encode(g["image"])  # BatchNorm would use batch statistics
    with pytest.raises(NotImplementedError):
        PaellaVQModel(levels=1, c_hidden=12, bottleneck_blocks=1)
    with pytest.raises(ValueError):
        m.eval().set_conv_precision("tf32")


def test_fold_cache_follows_parameter_updates(monkeypatch):
    install(monkeypatch)
    m = _model("f4")
    blk = m.down_blocks[0]
    first = blk._folded()
    assert blk._folded() is first
    with torch.no_grad():
        blk.gammas[2].mul_(2.0)
    assert blk._folded() is not first
    assert torch.allclose(blk._folded()[0], first[0] * 2.0, rtol=1e-6)


def test_compat_and_pipeline_load_paella(monkeypatch, tmp_path):
    from open_muse_b200 import MaskGiTUViT_v2, PaellaVQModel, PipelineMuse
    from open_muse_b200.compat import muse as compat_muse
    from tests.train_script_harness import UVIT_MICRO

    assert compat_muse.PaellaVQModel is PaellaVQModel
    torch.manual_seed(0)
    PaellaVQModel(levels=1, c_hidden=32, bottleneck_blocks=1, codebook_size=64).save_pretrained(str(tmp_path / "vae"))
    MaskGiTUViT_v2(**dict(UVIT_MICRO, add_cond_embeds=False, add_micro_cond_embeds=False,
                          use_empty_embeds_for_uncond=False)).save_pretrained(str(tmp_path / "transformer"))
    assert json.load(open(tmp_path / "vae" / "config.json"))["_class_name"] == "PaellaVQModel"
    pipe = PipelineMuse.from_pretrained(str(tmp_path), is_class_conditioned=True)
    assert isinstance(pipe.vae, PaellaVQModel) and pipe.vae.config.c_hidden == 32


def test_reference_train_muse_runs_with_paella(monkeypatch, tmp_path):
    from tests.train_script_harness import find_script, make_muse_config, run_script

    script = find_script("train_muse.py")
    if script is None:
        pytest.skip("reference training script not available")
    from open_muse_b200 import PaellaVQModel

    install(monkeypatch, exact=False)
    monkeypatch.setenv("ACCELERATE_USE_CPU", "1")
    monkeypatch.setenv("WANDB_MODE", "disabled")
    cfg_path, _ = make_muse_config(str(tmp_path), steps=3, batch=2, mixed_precision="no")
    torch.manual_seed(5)
    vq_dir = str(tmp_path / "paella")
    PaellaVQModel(levels=1, c_hidden=32, bottleneck_blocks=1, codebook_size=64).save_pretrained(vq_dir)  # 32 px -> 16 x 16
    cfg = yaml.safe_load(open(cfg_path))
    cfg["model"]["vq_model"] = {"type": "paella_vq", "pretrained": vq_dir}
    with open(cfg_path, "w") as f:
        yaml.safe_dump(cfg, f)
    acc = run_script(script, cfg_path)
    losses = [v["step_loss"] for v, s in acc.logged if "step_loss" in v]
    assert len(losses) == 3 and all(math.isfinite(x) for x in losses)
