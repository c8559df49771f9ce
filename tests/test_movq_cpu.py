"""CPU: MOVQ's host wiring (module tree and order, the shared taming blocks, the latent handed to every SpatialNorm, layouts,
the quantiser hand-off, the reference's quirks) against the outputs of the UNMODIFIED reference (tests/golden/micro_movq.pt),
with the kernels replaced by torch restatements: tests/cpu_math_ops.py for the existing ops, and below for the spatial mode
of conv2d / groupnorm_silu, the documented contract of its ops wrappers.  Also the argument checks of the new C entry point,
through the loaded library.  The kernels themselves are checked on the GPU (test_movq_gpu.py, test_movq_local_gpu.py)."""
import inspect
import json

import pytest
import torch
import torch.nn.functional as F

from oracle import movq_oracle as O
from tests import cpu_math_ops, movq_fixture

GOLD = torch.load(movq_fixture.PATH, weights_only=False)
_SD = {}
REFERENCE_ARGS = ["resolution", "num_channels", "out_channels", "hidden_channels", "channel_mult", "num_res_blocks",
                  "attn_resolutions", "z_channels", "double_z", "num_embeddings", "quantized_embed_dim", "dropout",
                  "resample_with_conv", "commitment_cost"]


def _sd(name):
    """the fixture's state dict, rebuilt from its seeds and checked against the reference's (tests/movq_fixture.py)"""
    from open_muse_b200 import MOVQ

    if name not in _SD:
        _SD[name] = movq_fixture.state_dict(MOVQ, GOLD, name)
    return _SD[name]


def _nchw(x):
    return x.permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


# ---- contract of the spatial mode (open_muse_b200/ops.py), fp32 NHWC in and out
def groupnorm_silu(x, gamma, beta, groups, eps, silu=1, spatial=None):
    """silu?(GN(x) * conv_y(up(zq)) + conv_b(up(zq))), zq NHWC, up = nearest resize to x's grid"""
    if spatial is None:
        return cpu_math_ops.groupnorm_silu(x, gamma, beta, groups, eps, silu)
    zq, cy, cb = spatial
    z = F.interpolate(_nchw(zq), size=x.shape[1:3], mode="nearest")
    y = cpu_math_ops.groupnorm_silu(x, gamma, beta, groups, eps, 0)
    y = y * _nhwc(F.conv2d(z, cy.weight, cy.bias)) + _nhwc(F.conv2d(z, cb.weight, cb.bias))
    return (F.silu(y) if silu else y).contiguous()


def conv2d(x, w, bias=None, residual=None, upsample2x=False, gn=None, spatial=None):
    if spatial is not None:
        x, gn = groupnorm_silu(x, *gn, spatial=spatial), None
    return cpu_math_ops.conv2d(x, w, bias, residual, upsample2x, gn)


def install(mp, exact=True):
    from open_muse_b200 import ops

    cpu_math_ops.install(mp, exact=exact)
    mp.setattr(ops, "conv2d", conv2d)
    mp.setattr(ops, "groupnorm_silu", groupnorm_silu)


def _model(name):
    from open_muse_b200 import MOVQ

    g = GOLD[name]
    m = MOVQ(**{k: v for k, v in g["config"].items() if not k.startswith("_")})
    m.load_state_dict(_sd(name), strict=True)
    return m.eval()


def _rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / b.norm())


@pytest.mark.parametrize("name", ["tc", "f8"])
def test_wiring_reproduces_reference(monkeypatch, name):
    install(monkeypatch)
    g = GOLD[name]
    m = _model(name)
    z = m._encode_nhwc(g["image"])
    assert _rel(_nchw(z), g["z"]) < 2e-5
    z_q, ids = m.encode(g["image"])
    assert ids.shape == g["ids"].shape
    sure = g["margin"] > 1e-4
    assert torch.equal(ids.reshape(-1)[sure], g["ids"].reshape(-1)[sure])
    if bool(sure.all()):
        assert torch.equal(z_q, g["z_q"])
    dec = m.decode_code(g["ids"])
    assert _rel(dec, g["decode_code"]) < 2e-5
    assert _rel(m.decode(g["z_q"]), g["decode_code"]) < 2e-5  # decode() takes the codebook rows, decode_code() the ids
    rec, fwd_ids = m(g["image"])
    assert torch.equal(fwd_ids, ids)
    if bool(sure.all()):
        assert _rel(rec, g["forward"]) < 2e-5
    assert torch.equal(m.get_code(g["image"]), ids)


def test_fixture_coverage():
    """both configs have ids spread over many codes and clear margins; their attention blocks are active"""
    for name, n_codes in (("tc", 40), ("f8", 20)):
        g = GOLD[name]
        assert g["ids"].unique().numel() >= n_codes
        assert float((g["margin"] > 1e-3).float().mean()) > 0.95
        m = _model(name)
        assert [len(d.attn) for d in m.encoder.down][-1] == 2 and [len(u.attn) for u in m.decoder.up][-1] == 3
        assert len(_sd(name)) == len(g["state_signature"])


@pytest.mark.parametrize("name", ["tc", "f8"])
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
    assert _rel(O.decode(sd, cfg, g["z_q"]), g["decode_code"]) < 1e-5


@pytest.mark.parametrize("name", ["tc", "f8"])
def test_seeded_construction_and_state_dict(name):
    from open_muse_b200 import MOVQ

    g = GOLD[name]
    torch.manual_seed(g["seed"])
    m = MOVQ(**{k: v for k, v in g["config"].items() if not k.startswith("_")})
    sd = m.state_dict()
    assert list(sd) == list(g["init_signature"])
    for k, (s, n) in g["init_signature"].items():
        assert float(sd[k].double().sum()) == pytest.approx(s, rel=1e-9, abs=1e-9), k
        assert float(sd[k].double().norm()) == pytest.approx(n, rel=1e-9, abs=1e-9), k


def test_surface_and_class_defaults():
    from open_muse_b200 import MOVQ
    from open_muse_b200.compat import muse as compat_muse

    assert compat_muse.MOVQ is MOVQ
    assert list(inspect.signature(MOVQ.__init__).parameters)[1:] == REFERENCE_ARGS
    for meth, args in (("encode", ["pixel_values", "return_loss"]), ("decode", ["quant"]),
                       ("decode_code", ["codebook_indices"]), ("get_code", ["pixel_values"]),
                       ("forward", ["pixel_values", "return_loss"])):
        assert list(inspect.signature(getattr(MOVQ, meth)).parameters)[1:] == args, meth
    torch.manual_seed(0)
    m = MOVQ()
    assert sorted(k for k in dict(m.config) if not k.startswith("_")) == sorted(REFERENCE_ARGS)
    sd = m.state_dict()
    assert len(sd) == 431 and sum(p.numel() for p in m.parameters()) == 67_832_495
    assert m.num_embeddings == 16384 and m.config.latent_size == 32 and m.config.reduction_factor == 8
    assert m.config.num_resolutions == 4
    assert sd["encoder.mid.attn_1.q.weight"].shape == (512, 512)
    assert sd["decoder.mid.block_1.norm1.conv_y.weight"].shape == (512, 4, 1, 1)
    assert "decoder.mid.block_1.norm1.norm_layer.weight" in sd and "decoder.norm_out.conv_b.bias" in sd
    assert sd["quantize.embedding.weight"].shape == (16384, 4)
    assert [k for k in sd if k.startswith(("quant_conv", "post_quant_conv"))] == [
        "quant_conv.weight", "quant_conv.bias", "post_quant_conv.weight", "post_quant_conv.bias"]
    # one 512-wide head over the 32 x 32 tokens: encoder level 3 (2 blocks) + mid, decoder level 3 (3 blocks) + mid
    assert [len(d.attn) for d in m.encoder.down] == [0, 0, 0, 2] and [len(u.attn) for u in m.decoder.up] == [0, 0, 0, 3]


def test_quirks(monkeypatch):
    install(monkeypatch)
    from open_muse_b200 import MOVQ
    from open_muse_b200.modeling_movq import SpatialNorm

    g = GOLD["f8"]
    m = _model("f8")
    assert len(m.encode(g["image"])) == 2 and len(m(g["image"])) == 2  # two values, unlike VQGANModel
    with pytest.raises(AttributeError, match="beta"):
        m.encode(g["image"], return_loss=True)
    with pytest.raises(AttributeError, match="beta"):
        m(g["image"], return_loss=True)
    assert not hasattr(m, "get_soft_code")  # training.use_soft_code_target raises AttributeError upstream
    with pytest.raises(NotImplementedError):
        m.quantize.get_soft_code(g["z"])
    # get_codebook_entry assumes a square grid: 8 x 16 tokens come back as 11 x 11 and the view fails
    with pytest.raises(RuntimeError):
        m.quantize.get_codebook_entry(torch.zeros(1, 128, dtype=torch.long))
    # out_channels and double_z are accepted and unused
    cfg = {k: v for k, v in g["config"].items() if not k.startswith("_")}
    torch.manual_seed(1)
    a = MOVQ(**cfg).state_dict()
    torch.manual_seed(1)
    b = MOVQ(**dict(cfg, out_channels=7, double_z=True)).state_dict()
    assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)
    with pytest.raises(NotImplementedError):
        SpatialNorm(32, 4, num_groups=32, eps=1e-6, affine=True, add_conv=True)
    with pytest.raises(NotImplementedError):
        MOVQ(**dict(cfg, resample_with_conv=False)).decode_code(g["ids"])
    with pytest.raises(ValueError):
        m.set_conv_precision("tf32")


def test_attention_runs_only_where_a_level_holds_more_than_one(monkeypatch):
    """num_res_blocks 1: one attention block per encoder level (not run), two per decoder level (run); the mid blocks
    always run theirs"""
    install(monkeypatch)
    from open_muse_b200 import MOVQ, ops

    calls = []
    real = ops.attention_single_head
    monkeypatch.setattr(ops, "attention_single_head", lambda q, k, v, B, hh, ww: calls.append(hh) or real(q, k, v, B, hh, ww))
    torch.manual_seed(2)
    m = MOVQ(resolution=32, hidden_channels=32, channel_mult=(1, 2), num_res_blocks=1, attn_resolutions=(16,),
             num_embeddings=16).eval()
    img = torch.rand(1, 3, 32, 32) * 2 - 1
    m.get_code(img)
    assert calls == [16]  # the encoder mid block only
    calls.clear()
    m.decode_code(torch.zeros(1, 256, dtype=torch.long))
    assert calls == [16, 16, 16]  # mid, then the two blocks of decoder level 1


def test_spatial_groupnorm_entry_point_checks():
    """muse_spatial_groupnorm_silu_nhwc refuses unsupported shapes before any launch (no device needed)"""
    from open_muse_b200 import _lib

    lib = _lib.load()
    MUSE_ERR_INVALID, MUSE_ERR_UNSUPPORTED = 1, 3
    fake = 1 << 20  # never dereferenced: every check runs before a launch

    def call(C=64, H=16, W=16, hz=8, wz=8, dq=4, zq=fake, y=fake, y_hi=None, groups=32):
        return lib.muse_spatial_groupnorm_silu_nhwc(fake, fake, fake, zq, fake, fake, fake, fake, y, y_hi, None, fake, fake,
                                                    2, H, W, C, groups, 1e-6, hz, wz, dq, 0, 1, None)

    def msg():
        return lib.muse_last_error().decode()

    assert call(H=16, hz=6) == MUSE_ERR_UNSUPPORTED and "integer multiple" in msg()  # ratio 16 / 6
    assert call(W=24, wz=16) == MUSE_ERR_UNSUPPORTED and "integer multiple" in msg()
    assert call(hz=0) == MUSE_ERR_UNSUPPORTED
    for dq in (0, 3, 6, 20):
        assert call(dq=dq) == MUSE_ERR_UNSUPPORTED and "latent channels" in msg()
    for C in (12, 2048, 68):
        assert call(C=C, groups=4) == MUSE_ERR_UNSUPPORTED and "unsupported" in msg()
    assert call(C=96, groups=32) == MUSE_ERR_UNSUPPORTED  # C / 4 = 24 does not divide 256
    assert call(y=None) == MUSE_ERR_INVALID  # neither output form
    assert call(y_hi=fake) == MUSE_ERR_INVALID  # both output forms
    assert call(zq=fake + 4) == MUSE_ERR_INVALID and "aligned" in msg()
    assert call(zq=None) == MUSE_ERR_INVALID


def test_pipeline_loads_movq(monkeypatch, tmp_path):
    from open_muse_b200 import MOVQ, MaskGiTUViT_v2, PipelineMuse
    from tests.train_script_harness import UVIT_MICRO

    torch.manual_seed(0)
    vq = MOVQ(resolution=32, hidden_channels=32, channel_mult=(1, 2), num_res_blocks=1, attn_resolutions=(), num_embeddings=64)
    vq.save_pretrained(str(tmp_path / "vae"))
    MaskGiTUViT_v2(**dict(UVIT_MICRO, add_cond_embeds=False, add_micro_cond_embeds=False,
                          use_empty_embeds_for_uncond=False)).save_pretrained(str(tmp_path / "transformer"))
    assert json.load(open(tmp_path / "vae" / "config.json"))["_class_name"] == "MOVQ"
    pipe = PipelineMuse.from_pretrained(str(tmp_path), is_class_conditioned=True)
    assert isinstance(pipe.vae, MOVQ) and pipe.vae.config.hidden_channels == 32
    sd = pipe.vae.state_dict()
    assert list(sd) == list(vq.state_dict()) and all(torch.equal(sd[k], v) for k, v in vq.state_dict().items())
    (tmp_path / "vae" / "config.json").write_text(json.dumps(dict(json.load(open(tmp_path / "vae" / "config.json")),
                                                                  _class_name="OtherVQ")))
    with pytest.raises(NotImplementedError, match="unknown tokenizer class OtherVQ"):
        PipelineMuse.from_pretrained(str(tmp_path), is_class_conditioned=True)


def test_latent_resize_is_nearest_integer_division():
    """the restated contract picks latent pixel (y // ry, x // rx), the kernel's index (F.interpolate nearest at integer
    ratios)"""
    zq = torch.arange(2 * 3 * 5 * 4, dtype=torch.float32).view(2, 3, 5, 4)
    up = F.interpolate(_nchw(zq), size=(12, 20), mode="nearest")
    ys, xs = torch.arange(12), torch.arange(20)
    assert torch.equal(_nhwc(up), zq[:, ys // 4][:, :, xs // 4])
