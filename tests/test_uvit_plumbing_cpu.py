"""Host-logic test (no GPU): the autograd plumbing of MaskGiTUViT_v2 training -- one Function per block -- with the C-ABI
kernels replaced by shape/dtype-checking stand-ins.  Verifies that every parameter receives a
gradient of its own shape, that every op sees the operand shapes / dtypes its kernel contract states (adaLN slices, fp32
accumulators, bf16 GEMM operands), also for norms without elementwise affine.  Numerics are covered by the GPU tests."""
import pytest
import torch

from open_muse_b200 import MaskGiTUViT_v2, ops

BF, F32 = torch.bfloat16, torch.float32


def _fake_ops(mp):
    def lin_fwd(x, w, out_dtype=BF, res=None, n_valid=None):
        assert x.shape[1] == w.shape[1], (x.shape, w.shape)
        return torch.zeros(x.shape[0], w.shape[0], dtype=F32 if res is not None else out_dtype)

    def wgrad(dy, x, dw):
        assert dw.shape == (dy.shape[1], x.shape[1]) and dy.dtype == BF and x.dtype == BF and dw.dtype == F32

    def dgrad_acc(dy, w, acc):
        assert acc.shape == (dy.shape[0], w.shape[1]) and acc.dtype == F32

    def silu_bwd(dy, x, out=None, out_dtype=None):
        assert dy.dtype == BF
        return out if out is not None else torch.zeros(x.shape, dtype=out_dtype or x.dtype)

    def anm(a, w, eps, rms, out_dtype=BF, residual=None, mod=None, rows_per_sample=1, want_residual=True):
        if mod is not None:
            assert mod.shape[1] == 2 * a.shape[1] and mod.dtype == F32
        return (torch.zeros(a.shape) if want_residual else None), torch.zeros(a.shape, dtype=out_dtype)

    def anm_bwd(dy, dr_out, x, w, eps, rms, da_dtype, mod=None, rows_per_sample=1, dw=None, dmod=None, want_dr=True):
        assert dy.shape == x.shape and x.dtype == F32
        if dr_out is not None:
            assert dr_out.dtype == F32 and dr_out.shape == x.shape
        if mod is not None:
            assert dmod.shape == mod.shape
        return torch.zeros(x.shape, dtype=da_dtype), (torch.zeros(x.shape) if want_dr else None)

    def dwb(dy, conv, x, wk, nw, dres, dwk, dnw, B, hh, ww, eps, rms):
        assert dy.dtype == BF and dres.dtype == F32 and dwk.shape == wk.shape
        return torch.zeros(x.shape)

    def grnb(x, dout, stats, gamma, dg, db, B, HW):
        assert dout.dtype == BF and dg.shape == gamma.shape
        return torch.zeros_like(x)

    def adb(dy, x, mod, dmod, B, rps):
        assert dy.dtype == F32 and mod.shape == dmod.shape == (B, 2 * x.shape[1])
        return torch.zeros_like(x)

    def attb(q, k, v, o, do, lse, dq, dk, dv, B, nh, Sq, Skv, sc, head_dim=64):
        assert do.dtype == BF and do.shape == o.shape and dq.shape == q.shape and dk.shape == k.shape

    fakes = dict(
        linear_fwd=lin_fwd, linear_dgrad=lambda dy, w, out_dtype=BF: torch.zeros(dy.shape[0], w.shape[1], dtype=out_dtype),
        linear_wgrad=wgrad, linear_dgrad_acc=dgrad_acc, cast_bf16=lambda x: x.to(BF), silu_bf16=lambda x: x.to(BF),
        silu_bwd=silu_bwd, embed_fwd=lambda ids, w, pos: torch.zeros(ids.numel(), w.shape[1]),
        embed_bwd=lambda ids, dx, dword, dpos: None, add_norm_mod=anm, add_norm_mod_bwd=anm_bwd,
        dwconv3x3_norm=lambda x, wk, nw, B, hh, ww, eps, rms, save_conv=False: (torch.zeros(x.shape, dtype=BF), torch.zeros(x.shape, dtype=BF)),
        dwconv3x3_norm_bwd=dwb, grn=lambda x, g, b, B, HW, save_stats=False: (torch.zeros_like(x), torch.zeros(2, B, x.shape[1])),
        grn_bwd=grnb, adaln_apply=lambda x, mod, B, rps: x.clone(), adaln_bwd=adb,
        attn_fwd=lambda q, k, v, B, nh, Sq, Skv, sc, head_dim=64: (torch.zeros(q.shape[0], nh * head_dim, dtype=BF), torch.zeros(B, nh, Sq)),
        attn_bwd=attb, glu_fwd=lambda ab: torch.zeros(ab.shape[0], ab.shape[1] // 2, dtype=BF), glu_bwd=lambda ab, d: torch.zeros_like(ab),
        ce_fwd=lambda lg, lab, V, ls: (torch.zeros(2), torch.zeros(2, lg.shape[0])),
        ce_bwd=lambda lg, lab, ws, dl, out, V, ls, row_scale=None: torch.zeros_like(lg))
    for k, v in fakes.items():
        mp.setattr(ops, k, v)


CFGS = [
    dict(hidden_size=128, num_attention_heads=2, in_channels=64, block_out_channels=(64,), block_num_heads=1, num_res_blocks=2,
         num_hidden_layers=2, intermediate_size=128, vocab_size=72, codebook_size=64, encoder_hidden_size=32, cond_embed_dim=16,
         micro_cond_encode_dim=8, micro_cond_embed_dim=40),
    dict(hidden_size=64, num_attention_heads=1, in_channels=64, block_out_channels=(64,), block_num_heads=1, num_res_blocks=1,
         num_hidden_layers=1, intermediate_size=64, vocab_size=72, codebook_size=64, encoder_hidden_size=32, cond_embed_dim=16,
         micro_cond_encode_dim=8, micro_cond_embed_dim=40, ln_elementwise_affine=False, norm_type="layernorm"),
]


@pytest.mark.parametrize("cfg", CFGS, ids=["rmsnorm-kvmapper", "layernorm-noaffine"])
def test_uvit_v2_training_plumbing(monkeypatch, cfg):
    import open_muse_b200.uvit_v2_train as T

    _fake_ops(monkeypatch)
    torch.manual_seed(0)
    m = MaskGiTUViT_v2(**cfg).train()
    ids, lab = torch.randint(0, 64, (3, 16)), torch.randint(0, 64, (3, 16))
    enc, ce, mc = torch.randn(3, 5, 32), torch.randn(3, 16), torch.rand(3, 5)
    padded, loss = T.train_forward(m, ids, enc, ce, mc, lab, 0.1, torch.rand(3, 16))
    assert padded.shape == (48, 64)
    (loss + 0 * padded.float().sum()).backward()
    for n, p in m.named_parameters():
        assert p.grad is not None and p.grad.shape == p.shape and p.grad.dtype == torch.float32, n


# ---------------------------------------------------------------------------------------------------------------------
# force_down_up_sample training (uvit_v2_train.ResampleFn): the token permutations around the patch GEMMs and the mapping of
# the GEMM weight gradients back to the Conv2d / ConvTranspose2d parameter layouts, checked NUMERICALLY on the CPU with exact
# fp32 stand-ins for the kernels against torch autograd through F.conv2d / F.conv_transpose2d on the NCHW tensor (what the
# reference computes, muse/modeling_transformer_v2.py:509-513, :555-559).
def _math_ops(mp):
    def norm(x, w, eps, rms):
        x = x.float()
        y = x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps) if rms else torch.nn.functional.layer_norm(x, x.shape[-1:], eps=eps)
        return y if w is None else y * w.float()

    def anm(a, w, eps, rms, out_dtype=BF, residual=None, mod=None, rows_per_sample=1, want_residual=True):
        assert residual is None and mod is None and not want_residual
        return None, norm(a, w, eps, rms)

    def anm_bwd(dy, dr_out, x, w, eps, rms, da_dtype, mod=None, rows_per_sample=1, dw=None, dmod=None, want_dr=True):
        assert dr_out is None and not want_dr and x.dtype == F32 and dy.shape == x.shape
        xx = x.detach().clone().requires_grad_(True)
        ww = None if w is None else w.detach().clone().requires_grad_(True)
        with torch.enable_grad():
            y = norm(xx, ww, eps, rms)
        gs = torch.autograd.grad(y, [xx] + ([] if ww is None else [ww]), dy.float())
        if dw is not None:
            dw += gs[1]
        return gs[0].to(da_dtype), None

    def wgrad(dy, x, dw):
        assert dw.shape == (dy.shape[1], x.shape[1]) and dw.dtype == F32
        dw += dy.float().t() @ x.float()

    mp.setattr(ops, "add_norm_mod", anm)
    mp.setattr(ops, "add_norm_mod_bwd", anm_bwd)
    mp.setattr(ops, "linear_fwd", lambda x, w, out_dtype=BF, res=None, n_valid=None: x.float() @ w.float().t())
    mp.setattr(ops, "linear_dgrad", lambda dy, w, out_dtype=BF: dy.float() @ w.float())
    mp.setattr(ops, "linear_wgrad", wgrad)
    mp.setattr(ops, "cast_bf16", lambda x: x)


@pytest.mark.parametrize("norm_type", ["rmsnorm", "layernorm"])
def test_uvit_v2_resample_functions_match_conv_autograd(monkeypatch, norm_type):
    import open_muse_b200.uvit_v2_train as T

    _math_ops(monkeypatch)
    cfg = dict(CFGS[0], force_down_up_sample=True, norm_type=norm_type)
    torch.manual_seed(1)
    m = MaskGiTUViT_v2(**cfg).train()
    down, up = m.down_blocks[0].downsample, m.up_blocks[0].upsample
    with torch.no_grad():
        for p in (down[0].norm.weight, up[0].norm.weight):
            p.copy_(torch.rand_like(p) + 0.5)
        for p in (down[1].weight, up[1].weight):  # bf16-representable, so the packed bf16 operands are exact
            p.copy_(torch.randn_like(p).to(BF).float())
    W = m._weights()
    B, hw, C = 3, 6, 64
    rms, eps = int(norm_type == "rmsnorm"), m.config.layer_norm_eps

    def norm2d(x, w):  # NCHW, normalised over the channels (Norm2D)
        t = x.permute(0, 2, 3, 1)
        t = t * torch.rsqrt(t.pow(2).mean(-1, keepdim=True) + eps) if rms else torch.nn.functional.layer_norm(t, (C,), eps=eps)
        return (t * w).permute(0, 3, 1, 2)

    to_nchw = lambda t, n: t.view(B, n, n, C).permute(0, 3, 1, 2)
    to_tok = lambda x: x.permute(0, 2, 3, 1).reshape(-1, C)
    for key, seq, n_in, conv in (("ds", down, hw, torch.nn.functional.conv2d), ("us", up, hw // 2, torch.nn.functional.conv_transpose2d)):
        sh = T._Shared(m, W, B, n_in * n_in, 5)
        assert sh.hw == n_in
        h = torch.randn(B * n_in * n_in, C, requires_grad=True)
        out = T.ResampleFn.apply(sh, key, h, seq[0].norm.weight, seq[1].weight)
        n_out = n_in // 2 if key == "ds" else n_in * 2
        assert out.shape == (B * n_out * n_out, C)
        d_out = torch.randn_like(out)
        g_h, g_n, g_w = torch.autograd.grad(out, (h, seq[0].norm.weight, seq[1].weight), d_out)
        h2 = h.detach().clone().requires_grad_(True)
        ref = to_tok(conv(norm2d(to_nchw(h2, n_in), seq[0].norm.weight), seq[1].weight, stride=2))
        r_h, r_n, r_w = torch.autograd.grad(ref, (h2, seq[0].norm.weight, seq[1].weight), d_out)
        for name, a, b in (("out", out, ref), ("dh", g_h, r_h), ("dnorm", g_n, r_n), ("dconv", g_w, r_w)):
            assert a.shape == b.shape, (key, name, a.shape, b.shape)
            err = float((a.detach() - b.detach()).norm() / b.detach().norm())
            assert err < 1e-5, (key, name, err)


def test_uvit_v2_training_plumbing_force_down_up_sample(monkeypatch):
    """whole train_forward with the shape-checking stand-ins: 8x8 tokens outside, 4x4 inside, every parameter (the two
    resampling convolutions and their norms included) receives a gradient of its own shape"""
    import open_muse_b200.uvit_v2_train as T

    _fake_ops(monkeypatch)
    torch.manual_seed(0)
    m = MaskGiTUViT_v2(**dict(CFGS[0], force_down_up_sample=True)).train()
    ids, lab = torch.randint(0, 64, (3, 64)), torch.randint(0, 64, (3, 64))
    enc, ce, mc = torch.randn(3, 5, 32), torch.randn(3, 16), torch.rand(3, 5)
    padded, loss = T.train_forward(m, ids, enc, ce, mc, lab, 0.1, None)
    assert padded.shape == (3 * 64, 64)
    (loss + 0 * padded.float().sum()).backward()
    for n, p in m.named_parameters():
        assert p.grad is not None and p.grad.shape == p.shape and p.grad.dtype == torch.float32, n
