"""GPU parity: fused generate2 step kernel vs the oracle's sample_step on identical pre-drawn noise (token ids and
mask positions bit-exact on margin-screened tokens), and the MaskGitVQGAN path vs reference goldens."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from open_muse_b200 import ops  # noqa: E402
from oracle import transformer_oracle as T  # noqa: E402
from oracle import vq_oracle as VQ  # noqa: E402
from oracle import vqgan_oracle as G  # noqa: E402

DEV = "cuda"


def _step_inputs(B, L, K, ld, seed, known_frac):
    g = torch.Generator().manual_seed(seed)
    logits = (torch.randn(B, L + 1, ld, generator=g) * 2.0).to(torch.bfloat16)
    ids = torch.full((B, L), K + 7, dtype=torch.long)  # mask id
    known = torch.rand(B, L, generator=g) < known_frac
    ids[known] = torch.randint(0, K, (int(known.sum()),), generator=g)
    q = torch.empty(B * L, K).exponential_(1, generator=g).view(B, L, K)
    u = torch.zeros(B, L).uniform_(0, 1, generator=g)
    return logits, ids, q, u


@pytest.mark.parametrize("B,L,K,ld,known_frac,mask_len,temp", [
    (4, 16, 64, 72, 0.0, 9, 1.0), (3, 16, 64, 72, 0.5, 3, 0.4), (64, 256, 1024, 2048, 0.3, 100, 0.7),
    (2, 256, 1024, 2048, 0.99, 200, 0.0), (2, 1024, 1024, 1032, 0.0, 1000, 2.0)])
def test_sample_step_vs_oracle(B, L, K, ld, known_frac, mask_len, temp):
    logits, ids, q, u = _step_inputs(B, L, K, ld, B * L + K, known_frac)
    mask_id = K + 7
    sampled, nxt, conf = ops.sample_step(logits.to(DEV), ids.to(DEV), q.to(DEV).contiguous(), u.to(DEV), K, mask_id,
                                         mask_len, temp, skip_first_token=True, return_conf=True)
    probs = logits[:, 1:, :K].float().softmax(-1)
    unknown = ids == mask_id
    ml = torch.max(torch.tensor([1]), torch.min(unknown.sum(-1, keepdim=True) - 1, torch.tensor([[mask_len]])))
    o_sampled, o_next = T.sample_step(probs, ids, mask_id, q, u, ml, temp)
    # margin screen 1: categorical draw = argmax(p/q); skip tokens whose top-2 scores are within 1e-5 relative
    sc = (probs / q).topk(2, dim=-1).values
    safe = (sc[..., 0] - sc[..., 1]) > 1e-5 * sc[..., 0]
    assert float(safe.float().mean()) > 0.999
    assert torch.equal(sampled.cpu()[safe], o_sampled[safe])
    assert torch.equal(sampled.cpu()[~unknown], ids[~unknown])  # known tokens are never overwritten
    # margin screen 2: re-mask decision conf < cut; skip rows with a sampling mismatch or a near-tie at the cut
    row_ok = (sampled.cpu() == o_sampled).all(-1)
    c = conf.cpu()
    cut = c.sort(-1).values.gather(1, ml)
    near = ((c - cut).abs() < 1e-4).sum(-1) > 1  # another confidence within 1e-4 of the cut value itself
    rows = row_ok & ~near
    assert int(rows.sum()) >= max(1, int(0.9 * B))
    assert torch.equal(nxt.cpu()[rows], o_next[rows])
    # size-independent property: exactly k tokens are re-masked per row (no ties at the cut)
    assert torch.equal((nxt.cpu()[rows] == mask_id).sum(-1), ml[rows, 0])


def test_sample_step_cfg_matches_manual_mix():
    B, L, K, ld = 2, 16, 64, 72
    logits, ids, q, u = _step_inputs(B, L, K, ld, 5, 0.2)
    unc = (logits.float() * 0.5 + 0.1).to(torch.bfloat16)
    g = 3.0
    mixed = (unc.float() + g * (logits.float() - unc.float()))
    s1, n1 = ops.sample_step(logits.to(DEV), ids.to(DEV), q.to(DEV), u.to(DEV), K, K + 7, 5, 0.5,
                             logits_unc=unc.to(DEV), guidance=g, skip_first_token=True)
    probs = mixed[:, 1:, :K].softmax(-1)
    ml = torch.full((B, 1), 5)
    o_s, o_n = T.sample_step(probs, ids, K + 7, q, u, ml, 0.5)
    assert float((s1.cpu() == o_s).float().mean()) > 0.97


def test_generate2_full_size_properties():
    """BASELINE config 5 shape (base model, B=64, 256 tokens, 12 steps): ids in range, deterministic per seed."""
    from open_muse_b200.modeling_transformer import MaskGitTransformer

    cfg = dict(vocab_size=2025, max_position_embeddings=257, hidden_size=512, num_hidden_layers=8,
               num_attention_heads=8, intermediate_size=2048, codebook_size=1024, num_vq_tokens=256, num_classes=1000,
               hidden_dropout=0.0, attention_dropout=0.0)
    torch.manual_seed(0)
    m = MaskGitTransformer(**cfg).to(DEV).eval()
    outs = []
    for _ in range(2):
        cls = torch.randint(0, 1000, (64,), generator=torch.Generator().manual_seed(6)).to(DEV)
        gen = torch.Generator(device=DEV).manual_seed(7)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            ids = m.generate2(class_ids=cls, timesteps=12, generator=gen)
        assert ids.shape == (64, 256) and int(ids.min()) >= 0 and int(ids.max()) < 1024
        outs.append(ids)
    assert torch.equal(outs[0], outs[1])


# ----------------------------------------------------------------------------------------- VQGAN blocks
def test_conv_gn_pool_blocks_vs_torch():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 64, 12, 10, generator=g)
    for cout, k, up, bias in [(128, 3, False, False), (64, 1, False, True), (3, 3, False, True), (96, 3, True, True)]:
        w = torch.randn(cout, 64, k, k, generator=g) * 0.05
        b = torch.randn(cout, generator=g) if bias else None
        xin = torch.nn.functional.interpolate(x, scale_factor=2.0, mode="nearest") if up else x
        ref = G.conv_same(xin, w, b)
        res = torch.randn(ref.shape, generator=g)
        y = ops.conv2d(ops.to_nhwc(x.to(DEV)), w.to(DEV), bias=None if b is None else b.to(DEV),
                       residual=ops.to_nhwc(res.to(DEV)), upsample2x=up)
        torch.testing.assert_close(ops.to_nchw(y).cpu(), ref + res, rtol=1e-4, atol=1e-5)
    x3 = torch.rand(2, 3, 16, 16, generator=g)
    w3 = torch.randn(32, 3, 3, 3, generator=g) * 0.2
    torch.testing.assert_close(ops.to_nchw(ops.conv2d(ops.to_nhwc(x3.to(DEV)), w3.to(DEV))).cpu(), G.conv_same(x3, w3),
                               rtol=1e-4, atol=1e-5)
    ga, be = torch.randn(64, generator=g), torch.randn(64, generator=g)
    gn = ops.groupnorm_silu(ops.to_nhwc(x.to(DEV)), ga.to(DEV), be.to(DEV), 32, 1e-6)
    torch.testing.assert_close(ops.to_nchw(gn).cpu(), G.gn_silu(x, ga, be), rtol=1e-4, atol=1e-5)
    pooled = ops.avg_pool2x2(ops.to_nhwc(x.to(DEV)))
    torch.testing.assert_close(ops.to_nchw(pooled).cpu(), torch.nn.functional.avg_pool2d(x, 2, 2), rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("B,H,W,cin,cout,k,bias,res,up,gn", [
    (2, 16, 16, 128, 128, 3, False, True, False, True),    # ResnetBlock conv2 at the 16x16 level (8-row tiles)
    (1, 32, 32, 64, 256, 3, True, False, False, False),    # 4-row tiles, BN = 256
    (3, 16, 16, 128, 256, 1, False, True, False, False),   # nin_shortcut 1x1
    (1, 3, 128, 64, 64, 3, True, False, False, False),     # one image row per tile, C_out below the N tile
    (1, 2, 256, 64, 512, 3, False, False, False, True),    # two tiles per image row, two N tiles
    (2, 32, 32, 128, 128, 3, True, False, True, False),    # UpsamplingBlock as four 2x2 parity convs (swapped tiles)
    (1, 32, 64, 64, 256, 3, True, True, True, False),      # UpsamplingBlock, unswapped 256-wide N tile, residual
    (1, 64, 16, 64, 512, 3, False, False, True, False),    # UpsamplingBlock, narrow low-res grid (8 wide), two N tiles
    (1, 2, 256, 64, 128, 3, True, True, False, False),     # C_out = 128: swapped operands, one 256-pixel row per tile
    (1, 3, 128, 64, 128, 3, True, True, False, False),     # C_out = 128 but odd height: unswapped 128-wide N tile
    (2, 4, 128, 128, 3, 3, True, False, False, True),      # decoder conv_out: 3 output channels (16-wide N tile)
    (2, 32, 32, 3, 128, 3, False, False, False, False),    # encoder conv_in: 27 taps through the im2col stem
    (1, 8, 128, 64, 7, 1, True, True, False, False),       # odd narrow head with bias + residual
    (2, 16, 8, 128, 48, 3, True, True, False, True),       # narrow image: one 16-row tile per image, C_out = 48
])
def test_conv_tensor_core_path_vs_fp64(B, H, W, cin, cout, k, bias, res, up, gn):
    """bf16x3 wgmma implicit GEMM (csrc/conv_tc.cu) against an fp64 convolution: fp32-level accuracy is the contract
    (a single bf16 pass would sit at ~4e-3)."""
    if not ops.conv_uses_tensor_cores(H, W, cin, cout, k):
        pytest.skip("geometry routed to the SIMT kernel")
    g = torch.Generator().manual_seed(B * 1000 + W)
    hi, wi = (H // 2, W // 2) if up else (H, W)
    x = torch.randn(B, cin, hi, wi, generator=g)
    w = torch.randn(cout, cin, k, k, generator=g) / math.sqrt(cin * k * k)
    b = torch.randn(cout, generator=g) if bias else None
    r = torch.randn(B, cout, H, W, generator=g) if res else None
    ga, be = (torch.randn(cin, generator=g), torch.randn(cin, generator=g)) if gn else (None, None)
    xin = x.double()
    if gn:
        xin = torch.nn.functional.silu(torch.nn.functional.group_norm(xin, 32, ga.double(), be.double(), 1e-6))
    if up:
        xin = torch.nn.functional.interpolate(xin, scale_factor=2.0, mode="nearest")
    ref = torch.nn.functional.conv2d(xin, w.double(), None if b is None else b.double(), padding=k // 2)
    if res:
        ref = ref + r.double()
    y = ops.conv2d(ops.to_nhwc(x.to(DEV)), w.to(DEV), bias=None if b is None else b.to(DEV),
                   residual=None if r is None else ops.to_nhwc(r.to(DEV)), upsample2x=up,
                   gn=(ga.to(DEV), be.to(DEV), 32, 1e-6) if gn else None)
    y = ops.to_nchw(y).cpu().double()
    rel = float((y - ref).norm() / ref.norm())
    assert rel < 2e-5, rel
    assert float((y - ref).abs().max()) < 2e-4 * float(ref.abs().max())


@pytest.mark.parametrize("c_mid,H,W", [(128, 16, 16), (256, 16, 16), (128, 2, 256), (64, 8, 32)])
def test_conv_epilogue_groupnorm_statistics_feed_next_layer(c_mid, H, W):
    """conv -> GroupNorm+SiLU -> conv where the GroupNorm statistics come from the first convolution's epilogue
    (swapped and unswapped tiles) instead of a pass over its output."""
    g = torch.Generator().manual_seed(c_mid + W)
    x = torch.randn(2, 64, H, W, generator=g)
    w1 = torch.randn(c_mid, 64, 3, 3, generator=g) / 24.0
    b1 = torch.randn(c_mid, generator=g)
    w2 = torch.randn(64, c_mid, 3, 3, generator=g) / math.sqrt(9 * c_mid)
    ga, be = torch.randn(c_mid, generator=g), torch.randn(c_mid, generator=g)
    y1 = ops.conv2d(ops.to_nhwc(x.to(DEV)), w1.to(DEV), bias=b1.to(DEV))
    assert getattr(y1, "_gn_stats", None) is not None
    y2 = ops.to_nchw(ops.conv2d(y1, w2.to(DEV), gn=(ga.to(DEV), be.to(DEV), 32, 1e-6))).cpu().double()
    r1 = torch.nn.functional.conv2d(x.double(), w1.double(), b1.double(), padding=1)
    r1 = torch.nn.functional.silu(torch.nn.functional.group_norm(r1, 32, ga.double(), be.double(), 1e-6))
    r2 = torch.nn.functional.conv2d(r1, w2.double(), None, padding=1)
    assert float((y2 - r2).norm() / r2.norm()) < 3e-5


def test_micro_vqgan_vs_reference(golden):
    from open_muse_b200.modeling_maskgit_vqgan import MaskGitVQGAN

    g = golden("micro_vqgan.pt")
    m = MaskGitVQGAN(**g["config"])
    m.load_state_dict(g["state_dict"])
    m.to(DEV).eval()
    img = g["image"].to(DEV)
    z_q, ids = m.encode(img)
    ok = (g["margin"] > 1e-4).view(ids.shape)  # margin screen (fp32 re-association cannot flip these)
    assert float(ok.float().mean()) > 0.95
    assert torch.equal(ids.cpu()[ok], g["ids"][ok])
    assert torch.equal(m.get_code(img).cpu(), ids.cpu())
    rec = m.decode_code(g["ids"].to(DEV))
    torch.testing.assert_close(rec.cpu(), g["recon"], rtol=1e-3, atol=1e-4)
    zq_ref = m.quantize.get_codebook_entry(g["ids"].to(DEV))
    assert torch.equal(zq_ref.cpu(), g["z_q"])
    out = m(img)
    assert out[0].shape == g["recon"].shape and len(out) == 3


def test_vqgan_f16_256_vs_reference_fixture(golden):
    """BASELINE config 3 at its own architecture against the UNMODIFIED reference (tests/golden/f16_256_vqgan.pt: default
    init from the seed, codebook ~ N(0, std(z)), two rand images): encoder output, token ids bit-exact on every position
    whose top-2 distance margin is above 1e-4 relative, quantised latents, reconstruction -- all through the wgmma
    (bf16x3 implicit-GEMM) convolution route."""
    from open_muse_b200.modeling_maskgit_vqgan import MaskGitVQGAN

    g = golden("f16_256_vqgan.pt")
    torch.manual_seed(g["seed"])
    m = MaskGitVQGAN()
    for k, (s_, n_) in g["init_signature"].items():  # seeded construction == the reference's default init
        t = m.state_dict()[k].double()
        assert abs(float(t.sum()) - s_) <= 1e-9 * max(1.0, abs(s_)) and abs(float(t.norm()) - n_) <= 1e-9 * max(1.0, n_), k
    with torch.no_grad():
        m.quantize.embedding.weight.copy_(g["codebook"])
    m.to(DEV).eval()
    assert ops.conv_uses_tensor_cores(256, 256, 128, 128, 3) and ops.conv_uses_tensor_cores(16, 16, 512, 512, 3)
    img = torch.rand(2, 3, 256, 256, generator=torch.Generator().manual_seed(g["image_seed"])).to(DEV)
    z = ops.to_nchw(m.encoder.run(ops.to_nhwc(img))).cpu()
    rz = float((z - g["z"]).norm() / g["z"].norm())
    assert rz < 1e-4, rz
    z_q, ids = m.encode(img)
    ok = (g["margin"] > 1e-4 * g["dmin"].abs()).view(ids.shape)
    n_bad = int((~ok).sum())
    assert n_bad <= 8, n_bad  # 3 of 512 positions sit below the screen in the fixture
    same = ids.cpu() == g["ids"]
    assert bool(same[ok].all()), int((~same[ok]).sum())
    print(f"f16-256 vs reference: z rel-L2 {rz:.2e}; ids equal on all {int(ok.sum())} screened positions, "
          f"{int(same[~ok].sum())}/{n_bad} of the unscreened ones")
    assert torch.equal(m.get_code(img).cpu(), ids.cpu())
    assert torch.equal(m.quantize.get_codebook_entry(g["ids"].to(DEV)).cpu(), g["z_q"])
    rec = m.decode_code(g["ids"].to(DEV)).cpu()
    torch.testing.assert_close(rec, g["recon"], rtol=1e-3, atol=2e-4)
    assert float((rec - g["recon"]).norm() / g["recon"].norm()) < 2e-4
    # bit-exact ids against the C oracle on the kernel's own encoder output (every position, no screen)
    ids_o, _ = VQ.argmin(VQ.nchw_to_rows(z.numpy()), g["codebook"].numpy())
    assert np.array_equal(ids.cpu().numpy().reshape(-1), ids_o)


def test_vqgan_f16_256_single_pass_bf16_mode(golden):
    """Fast tokenizer mode (one bf16 tensor-core product per fp32 product, SURVEY H1 iii): same architecture and fixture as
    above; the encoder output stays within bf16-operand accuracy of the reference, most token ids agree with the exact
    ones (the rate is what bench.py reports), the default mode is untouched."""
    from open_muse_b200.modeling_maskgit_vqgan import MaskGitVQGAN

    g = golden("f16_256_vqgan.pt")
    torch.manual_seed(g["seed"])
    m = MaskGitVQGAN()
    with torch.no_grad():
        m.quantize.embedding.weight.copy_(g["codebook"])
    m.to(DEV).eval()
    img = torch.rand(2, 3, 256, 256, generator=torch.Generator().manual_seed(g["image_seed"])).to(DEV)
    exact = m.get_code(img)
    m.set_conv_precision("bf16")
    z = ops.to_nchw(m._encode_nhwc(img)).cpu()
    rz = float((z - g["z"]).norm() / g["z"].norm())
    fast = m.get_code(img)
    agree = float((fast == exact).float().mean())
    rec = m.decode_code(g["ids"].to(DEV)).cpu()
    rr = float((rec - g["recon"]).norm() / g["recon"].norm())
    print(f"single-pass bf16 tokenizer: z rel-L2 {rz:.2e}, id agreement with the exact mode {100 * agree:.1f} %, recon rel-L2 {rr:.2e}")
    assert rz < 3e-2 and rr < 3e-2 and agree > 0.5
    with pytest.raises(ValueError):
        m.set_conv_precision("fp8")
    m.set_conv_precision("bf16x3")
    assert torch.equal(m.get_code(img), exact)


def test_vqgan_f16_256_roundtrip_properties():
    """BASELINE config 3 architecture (f16, 256 px) on a small batch: decode_code(ids) depends only on ids,
    encode is deterministic, ids match the oracle's search on the encoder output bit-for-bit."""
    from open_muse_b200.modeling_maskgit_vqgan import MaskGitVQGAN

    torch.manual_seed(5)
    m = MaskGitVQGAN().to(DEV).eval()
    img = torch.rand(2, 3, 256, 256, generator=torch.Generator().manual_seed(5)).to(DEV)
    z = ops.to_nchw(m.encoder.run(ops.to_nhwc(img)))
    with torch.no_grad():
        m.quantize.embedding.weight.copy_(torch.randn(1024, 256, device=DEV) * z.std())
    z_q, ids = m.encode(img)
    z_q2, ids2 = m.encode(img)
    assert torch.equal(ids, ids2) and ids.shape == (2, 256) and z_q.shape == (2, 256, 16, 16)
    ids_o, _ = VQ.argmin(VQ.nchw_to_rows(z.cpu().numpy()), m.quantize.embedding.weight.detach().cpu().numpy())
    assert np.array_equal(ids.cpu().numpy().reshape(-1), ids_o)
    rec = m.decode_code(ids)
    assert rec.shape == (2, 3, 256, 256) and bool(torch.isfinite(rec).all())
    assert torch.equal(rec, m.decode(z_q))


def test_vqgan_f16_256_tensor_core_route_matches_fp32_simt_route(monkeypatch):
    """The wgmma bf16x3 convolutions must be interchangeable with the fp32 SIMT kernels: encoder output and decoded
    pixels agree to fp32-level tolerance and the token ids are identical wherever the arg-min margin is not tiny."""
    from open_muse_b200.modeling_maskgit_vqgan import MaskGitVQGAN

    torch.manual_seed(7)
    m = MaskGitVQGAN().to(DEV).eval()
    img = torch.rand(2, 3, 256, 256, generator=torch.Generator().manual_seed(8)).to(DEV)
    outs = {}
    for route in ("simt", "tc"):
        with ops.conv_route(None if route == "tc" else "simt"):
            assert ops.conv_uses_tensor_cores(16, 16, 512, 512, 3) == (route == "tc")
            z = m.encoder.run(ops.to_nhwc(img))
            if route == "simt":
                with torch.no_grad():
                    m.quantize.embedding.weight.copy_(torch.randn(1024, 256, device=DEV) * z.std())
            ids, dmin = ops.vq_argmin(z.reshape(-1, 256), m.quantize.embedding.weight.float(), return_dmin=True)
            outs[route] = (z, ids, m.decode_code(ids.view(2, -1)) if route == "tc" else None)
    z_s, ids_s, _ = outs["simt"]
    z_t, ids_t, rec_t = outs["tc"]
    assert float((z_t - z_s).norm() / z_s.norm()) < 1e-4  # measured 3e-5 over the 28 encoder convolutions
    d = torch.cdist(z_s.reshape(-1, 256), m.quantize.embedding.weight.float()) ** 2
    top2 = d.topk(2, dim=1, largest=False).values
    safe = (top2[:, 1] - top2[:, 0]) > 1e-3 * top2[:, 0].abs()
    assert int(safe.sum()) > 400 and torch.equal(ids_s[safe], ids_t[safe])
    with ops.conv_route("simt"):
        rec_s = m.decode_code(ids_t.view(2, -1))
    assert float((rec_t - rec_s).norm() / rec_s.norm()) < 1.5e-4  # measured 6.6e-5 over the 32 decoder convolutions


def test_pipeline_class_conditional_end_to_end():
    from open_muse_b200 import MaskGitTransformer, MaskGitVQGAN, PipelineMuse

    torch.manual_seed(0)
    vae = MaskGitVQGAN(resolution=32, hidden_channels=32, channel_mult=(1, 2), num_res_blocks=1, z_channels=16,
                       num_embeddings=64, quantized_embed_dim=16)
    tr = MaskGitTransformer(vocab_size=72, hidden_size=64, num_hidden_layers=2, num_attention_heads=1,
                            intermediate_size=128, max_position_embeddings=257, codebook_size=64, num_vq_tokens=256,
                            num_classes=7, hidden_dropout=0.0, attention_dropout=0.0)
    pipe = PipelineMuse(vae=vae, transformer=tr, is_class_conditioned=True).to(DEV)
    a = pipe(class_ids=[1, 5], timesteps=4, num_images_per_prompt=2, generator=torch.Generator(device=DEV).manual_seed(3))
    b = pipe(class_ids=[1, 5], timesteps=4, num_images_per_prompt=2, generator=torch.Generator(device=DEV).manual_seed(3))
    assert len(a) == 4 and a[0].size == (32, 32) and a[0].mode == "RGB"
    assert all(np.array_equal(np.asarray(x), np.asarray(y)) for x, y in zip(a, b))
    pt = pipe(class_ids=3, timesteps=2, output_type="pt")
    assert pt.shape == (1, 3, 32, 32)


def test_decode_code_uint8_matches_reference_pil_recipe(golden):
    """Device-side display bytes == the reference's host recipe (pipeline_muse.py:245-252) applied to the decoded tensor,
    byte for byte, including out-of-range decoder values (the recipe clamps) and the truncation."""
    from open_muse_b200 import MaskGitVQGAN, PipelineMuse

    g = golden("micro_vqgan.pt")
    m = MaskGitVQGAN(**g["config"])
    m.load_state_dict(g["state_dict"])
    with torch.no_grad():
        m.decoder.conv_out.bias.add_(torch.tensor([0.6, -0.4, 0.1]))  # push part of the output outside [0, 1]
    m.to(DEV).eval()
    ids = g["ids"].to(DEV)
    got = m.decode_code_uint8(ids).cpu().numpy()
    rec = m.decode_code(ids)
    assert float(rec.max()) > 1.0 and float(rec.min()) < 0.0
    pipe = PipelineMuse(vae=m, transformer=None, is_class_conditioned=True)
    for i in range(rec.shape[0]):
        assert np.array_equal(got[i], np.asarray(pipe.to_pil_image(rec[i])))


def test_pipeline_inpainting_keeps_known_tokens():
    from open_muse_b200 import MaskGitTransformer, MaskGitVQGAN, PipelineMuseInpainting

    torch.manual_seed(0)
    vae = MaskGitVQGAN(resolution=32, hidden_channels=32, channel_mult=(1, 2), num_res_blocks=1, z_channels=16,
                       num_embeddings=64, quantized_embed_dim=16)
    tr = MaskGitTransformer(vocab_size=72, hidden_size=64, num_hidden_layers=2, num_attention_heads=1,
                            intermediate_size=128, max_position_embeddings=257, codebook_size=64, num_vq_tokens=256,
                            num_classes=7, hidden_dropout=0.0, attention_dropout=0.0)
    pipe = PipelineMuseInpainting(vae=vae, transformer=tr, is_class_conditioned=True).to(DEV)
    image = torch.rand(1, 3, 32, 32, generator=torch.Generator().manual_seed(5))
    mask = torch.zeros(256, dtype=torch.bool)
    mask[64:192] = True
    seen = {}
    decode = vae.decode_code_uint8  # the pipeline's PIL path goes ids -> display bytes on the device
    vae.decode_code_uint8 = lambda ids: (seen.__setitem__("ids", ids.clone()), decode(ids))[1]
    out = pipe(image, mask, class_ids=[2], timesteps=4, num_images_per_prompt=3,
               generator=torch.Generator(device=DEV).manual_seed(1))
    assert len(out) == 3 and out[0].size == (32, 32)
    orig = vae.get_code(image.to(DEV))
    got = seen["ids"]
    assert got.shape == (3, 256) and int(got.max()) < 64 and int(got.min()) >= 0  # no mask ids left
    assert torch.equal(got[:, ~mask], orig[:, ~mask].expand(3, -1))  # unmasked tokens are never resampled
    # PIL input path: resize + centre crop + ToTensor
    from PIL import Image

    pil = Image.fromarray((np.random.RandomState(0).rand(40, 48, 3) * 255).astype(np.uint8))
    assert PipelineMuseInpainting._to_pixel_values(pil, 32).shape == (1, 3, 32, 32)
    out = pipe(pil, mask, class_ids=2, timesteps=2, image_size=32, output_type="pt")
    assert out.shape == (1, 3, 32, 32)


def test_generate2_loop_trace_vs_oracle_config5():
    """BASELINE config 5 (base model, B=64, 256 tokens, 12 steps, temperature 1.0) loop-level parity with pre-drawn noise.

    The kernel loop runs with the private ``_noise`` / ``_trace`` hooks; every step is then re-derived by the oracle's
    restatement of the reference loop (mask_len schedule, compounding temperature of quirk Q4, class-token skip, known
    tokens kept, per-row clamp of k) from the SAME state and noise:
      (i)  on the kernel's own bf16 logits: sampled ids and re-masked positions must be bit-exact (screen: exact ties only);
      (ii) on the oracle's own fp32 forward (run on the GPU in fp32): sampled ids equal wherever the top-2 categorical
           scores differ by more than the bf16 logit noise, agreement rate reported.
    The final ids contain no mask token, and the graph-captured loop reproduces the launched-one-by-one loop bit for bit
    through the torch generator."""
    from open_muse_b200.modeling_transformer import MaskGitTransformer

    cfg = dict(vocab_size=2025, max_position_embeddings=257, hidden_size=512, num_hidden_layers=8,
               num_attention_heads=8, intermediate_size=2048, codebook_size=1024, num_vq_tokens=256, num_classes=1000,
               hidden_dropout=0.0, attention_dropout=0.0)
    B, L, K, steps = 64, 256, 1024, 12
    torch.manual_seed(0)
    m = MaskGitTransformer(**cfg).to(DEV).eval()
    p = {k: v.detach().float() for k, v in m.state_dict().items()}  # fp32 oracle parameters, on the GPU
    cls0 = torch.randint(0, 1000, (B,), generator=torch.Generator().manual_seed(6)).to(DEV)
    gen = torch.Generator(device=DEV).manual_seed(7)
    noise = [(torch.empty(B * L, K, device=DEV).exponential_(1, generator=gen),
              torch.zeros(B, L, device=DEV).uniform_(0, 1, generator=gen)) for _ in range(steps)]
    trace = []
    cls = cls0.clone()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        final = m.generate2(class_ids=cls, timesteps=steps, temperature=1.0, _noise=noise, _trace=trace)
    assert torch.equal(cls, cls0 + K) and len(trace) == steps
    assert int(final.min()) >= 0 and int(final.max()) < K
    scal = T.generate2_scalars(cfg, steps, 1.0)
    agree_all, n_all = 0, 0
    for t in trace:
        s = t["step"]
        assert t["mask_len"] == int(scal[s][0]) and abs(t["temperature"] - scal[s][1]) < 1e-12
        q = noise[s][0].view(B, L, K)
        u = noise[s][1]
        # (i) same logits: integer outputs exact
        o = T.generate2_step_teacher_forced(p, cfg, None, t["input_ids"], s, steps, scal, q, u, logits=t["logits"])
        safe = (o["top2"][..., 0] - o["top2"][..., 1]) > 1e-5 * o["top2"][..., 0]
        assert float(safe.float().mean()) > 0.999
        assert torch.equal(t["sampled"][safe], o["sampled"][safe])
        known = ~o["unknown"]
        assert torch.equal(t["sampled"][known], t["input_ids"][known])
        row_ok = (t["sampled"] == o["sampled"]).all(-1)
        near = ((o["conf"] - o["cut"]).abs() < 1e-4).sum(-1) > 1
        rows = row_ok & ~near
        assert int(rows.sum()) >= int(0.9 * B)
        assert torch.equal(t["next_ids"][rows], o["next_ids"][rows])
        assert torch.equal((t["next_ids"][rows] == 2024).sum(-1).float(), o["mask_len"][rows, 0].float())
        # (ii) the oracle's own fp32 forward from the same state
        model_in = torch.cat([cls[:, None], t["input_ids"]], dim=1)
        with torch.no_grad():
            f = T.generate2_step_teacher_forced(p, cfg, model_in, t["input_ids"], s, steps, scal, q, u)
        unk = f["unknown"]
        wide = unk & ((f["top2"][..., 0] - f["top2"][..., 1]) > 0.15 * f["top2"][..., 0])  # bf16 logit noise ~ 1e-2 absolute
        assert torch.equal(t["sampled"][wide], f["sampled"][wide]), s
        agree_all += int((t["sampled"][unk] == f["sampled"][unk]).sum())
        n_all += int(unk.sum())
    print(f"generate2 config 5: sampled ids agree with the fp32 oracle on {agree_all}/{n_all} unknown tokens "
          f"({100.0 * agree_all / max(1, n_all):.2f} %) without any screen; exact on the screened ones and on shared logits")
    assert agree_all > 0.9 * n_all
    # the graph-captured loop consumes the torch generator like the launched loop and gives identical ids
    outs = []
    g2 = torch.Generator(device=DEV)
    for use_graph in (False, True, True):  # the third call replays the graph captured by the second
        g2.manual_seed(11)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            outs.append(m.generate2(class_ids=cls0.clone(), timesteps=steps, generator=g2, use_cuda_graph=use_graph))
        outs.append(g2.get_state().clone())
    assert torch.equal(outs[0], outs[2]) and torch.equal(outs[0], outs[4])
    assert torch.equal(outs[1], outs[3]) and torch.equal(outs[1], outs[5])  # same generator advance
