"""Dropout of MaskGitTransformer (hidden_dropout / attention_dropout in training mode) without a GPU.

This file holds the one restatement of the keep-mask generator of csrc/philox.cuh (Philox4x32-10 and the mapping from
(seed, site, coordinates) to keep bits): it is pinned here to the Random123 known answers, the GPU tests
(tests/test_dropout_gpu.py) compare the kernels' stored bits with it, and the dropout-aware CPU stand-ins below draw their
masks from it.  With those stand-ins the product's host code runs in exact mode (tests/cpu_math_ops.py) and is compared
with the UNMODIFIED reference whose three nn.Dropout modules are replaced by modules that apply the recorded masks."""
import numpy as np
import pytest
import torch

from open_muse_b200 import MaskGitTransformer, ops
from tests import cpu_math_ops

# ---------------------------------------------------------------------------------------------------- the generator
_M = np.uint64(0xFFFFFFFF)
_MUL0, _MUL1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Random123 philox4x32_R(10): counters (arrays of 32-bit values), key (k0, k1) -> four arrays of 32-bit words"""
    c = [np.asarray(x, dtype=np.uint64) & _M for x in (c0, c1, c2, c3)]
    c = np.broadcast_arrays(*c)
    k0, k1 = np.uint64(k0) & _M, np.uint64(k1) & _M
    for r in range(10):
        if r:
            k0, k1 = (k0 + _W0) & _M, (k1 + _W1) & _M
        p0, p1 = c[0] * _MUL0, c[2] * _MUL1
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & _M, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & _M]
    return c


def threshold(p):
    """t = round(p * 65536) in fp32 (keep iff the 16-bit uniform >= t)"""
    return int(min(max(np.rint(np.float32(p) * np.float32(65536.0)), 0), 65536))


def keep_scale(p):
    t = threshold(p)
    return 0.0 if t >= 65536 else float(np.float32(65536.0) / np.float32(65536 - t))


def _key(seed):
    s = int(seed.reshape(-1)[0]) if isinstance(seed, torch.Tensor) else int(seed)
    s %= 1 << 64
    return s & 0xFFFFFFFF, s >> 32


def _lane_keep(words, lane, t):
    w = np.choose(lane >> 1, words) if np.ndim(lane) else words[lane >> 1]
    return ((w >> (np.uint64(16) * (np.asarray(lane, dtype=np.uint64) & np.uint64(1)))) & np.uint64(0xFFFF)) >= t


def attn_keep(seed, site, B, nh, Sq, Skv, p):
    """bool [B, nh, Sq, Skv]: counter (call, q, b * nh + h, site), call = (k/64)*8 + ((k%64)/32)*4 + (k%8)/2,
    lane 2 ((k/8) % 4) + k % 2"""
    k = np.arange(Skv, dtype=np.uint64)
    call = (k // 64) * 8 + ((k % 64) // 32) * 4 + (k % 8) // 2
    lane = (2 * ((k // 8) % 4) + k % 2).astype(np.int64)
    bh = np.arange(B * nh, dtype=np.uint64)[:, None, None]
    q = np.arange(Sq, dtype=np.uint64)[None, :, None]
    words = philox4x32_10(call[None, None, :], q, bh, np.uint64(site), *_key(seed))
    lane = np.broadcast_to(lane, words[0].shape)
    return torch.from_numpy(_lane_keep(words, lane, threshold(p)).reshape(B, nh, Sq, Skv))


def elem_keep(seed, site, rows, cols, p):
    """bool [rows, cols]: counter (col / 8, row, 0, site), lane col % 8"""
    col = np.arange(cols, dtype=np.uint64)[None, :]
    row = np.arange(rows, dtype=np.uint64)[:, None]
    words = philox4x32_10(col // 8, row, np.uint64(0), np.uint64(site), *_key(seed))
    lane = np.broadcast_to((col % 8).astype(np.int64), words[0].shape)
    return torch.from_numpy(_lane_keep(words, lane, threshold(p)))


def pack_bits(keep):
    """bool [..., n] -> int32 [..., ceil(n / 32)]: bit k % 32 of word k / 32, pad bits 0"""
    n = keep.shape[-1]
    W = (n + 31) // 32
    k = torch.zeros(*keep.shape[:-1], W * 32, dtype=torch.int64)
    k[..., :n] = keep.long()
    w = (k.view(*keep.shape[:-1], W, 32) << torch.arange(32)).sum(-1)
    return torch.where(w >= 1 << 31, w - (1 << 32), w).to(torch.int32)


def unpack_bits(bits, n):
    b = (bits.long()[..., None] >> torch.arange(32)) & 1
    return b.flatten(-2)[..., :n].bool()


# ------------------------------------------------------------------------------------------- dropout-aware stand-ins
def _dropout_fwd(x, p, seed, site):
    keep = elem_keep(seed, site, x.shape[0], x.shape[1], p)
    x.copy_((x.float() * keep * keep_scale(p)).to(x.dtype))
    bits = pack_bits(keep)
    ops._drop_record(site, bits)
    return x, bits


def _dropout_bwd(dy, bits, p, out=None):
    dx = (dy.float() * unpack_bits(bits, dy.shape[1]) * keep_scale(p)).to(dy.dtype)
    if out is not None:
        out.copy_(dx)
        return out
    return dx


def _attn_z(q, k, v, B, nh, Sq, Skv, scale, hd, z):
    s = (cpu_math_ops._heads(q, B, Sq, nh, hd) @ cpu_math_ops._heads(k, B, Skv, nh, hd).transpose(-1, -2)) * scale
    o = (s.softmax(-1) * z) @ cpu_math_ops._heads(v, B, Skv, nh, hd)
    return o.permute(0, 2, 1, 3).reshape(B * Sq, nh * hd), torch.logsumexp(s, -1)


def _attn_fwd(q, k, v, B, nh, Sq, Skv, scale, head_dim=64, dropout=None):
    if dropout is None:
        return cpu_math_ops.attn_fwd(q, k, v, B, nh, Sq, Skv, scale, head_dim)
    p, seed, site = dropout
    keep = attn_keep(seed, site, B, nh, Sq, Skv, p)
    o, lse = _attn_z(q, k, v, B, nh, Sq, Skv, scale, int(head_dim), keep * keep_scale(p))
    bits = pack_bits(keep)
    ops._drop_record(site, bits)
    return o.to(torch.bfloat16), lse, bits


def _attn_bwd(q, k, v, o, do, lse, dq, dk, dv, B, nh, Sq, Skv, scale, head_dim=64, dropout=None):
    if dropout is None:
        return cpu_math_ops.attn_bwd(q, k, v, o, do, lse, dq, dk, dv, B, nh, Sq, Skv, scale, head_dim)
    p, bits = dropout
    z = unpack_bits(bits, Skv) * keep_scale(p)
    qq, kk, vv = (t.detach().float().clone().requires_grad_(True) for t in (q, k, v))
    with torch.enable_grad():
        out, _ = _attn_z(qq, kk, vv, B, nh, Sq, Skv, scale, int(head_dim), z)
    gq, gk, gv = torch.autograd.grad(out, (qq, kk, vv), do.float())
    dq.copy_(gq), dk.copy_(gk), dv.copy_(gv)


def _norm_fwd(x, w, eps, out_dtype, res=None, act=0, rms=0, save_stats=True, dropout=None):
    if dropout is None:
        return cpu_math_ops.norm_fwd(x, w, eps, out_dtype, res, act, rms, save_stats)
    y, stats = cpu_math_ops.norm_fwd(x, w, eps, torch.float32, res, act, rms, save_stats)
    y, bits = _dropout_fwd(y, *dropout)  # the dropout is applied to the fp32 normalised value, then rounded once
    return y.to(out_dtype), stats, bits


def _norm_bwd(dy, x, w, stats, dx_dtype, dw=None, dres=None, act=0, rms=0, y_fwd=None, want_dw=False, bf16_copy=False,
              dropout=None):
    if dropout is not None:
        assert y_fwd is None
        dy = _dropout_bwd(dy.float(), dropout[1], dropout[0])
    return cpu_math_ops.norm_bwd(dy, x, w, stats, dx_dtype, dw, dres, act, rms, y_fwd, want_dw, bf16_copy)


def _glu_fwd(ab, dropout=None):
    out = cpu_math_ops._act(ab, 2)
    if dropout is None:
        return out.to(torch.bfloat16)
    out, bits = _dropout_fwd(out, *dropout)
    return out.to(torch.bfloat16), bits


def _glu_bwd(ab, dout, dropout=None):
    if dropout is not None:
        dout = _dropout_bwd(dout.float(), dropout[1], dropout[0])
    return cpu_math_ops.glu_bwd(ab, dout)


def install(mp):
    cpu_math_ops.install(mp, exact=True)
    for name, fn in dict(dropout_fwd=_dropout_fwd, dropout_bwd=_dropout_bwd, attn_fwd=_attn_fwd, attn_bwd=_attn_bwd,
                         norm_fwd=_norm_fwd, norm_bwd=_norm_bwd, glu_fwd=_glu_fwd, glu_bwd=_glu_bwd).items():
        mp.setattr(ops, name, fn)


# --------------------------------------------------------------------------------------------------------- tests
def test_philox_matches_the_random123_known_answers():
    def kat(ctr, key):
        return [int(w) for w in philox4x32_10(*[np.uint64(c) for c in ctr], *key)]

    assert kat([0, 0, 0, 0], (0, 0)) == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    f = 0xFFFFFFFF
    assert kat([f, f, f, f], (f, f)) == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]
    assert kat([0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344], (0xA4093822, 0x299F31D0)) == \
        [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1]


def test_threshold_rate_and_bit_layout():
    for p in (0.1, 0.25, 0.5, 0.9):
        assert abs(threshold(p) / 65536 - p) <= 2 ** -17
    keep = torch.rand(5, 77) > 0.3
    bits = pack_bits(keep)
    assert bits.shape == (5, 3) and bits.dtype == torch.int32
    assert torch.equal(unpack_bits(bits, 77), keep)
    assert int(bits[0, 0]) & 1 == int(keep[0, 0]) and (int(bits[0, 2]) >> 13) == 0  # columns 64..76: bits 0..12 of word 2
    # one Philox call covers the 8 columns a wgmma fragment thread owns in one 32-column half: 8g + c, +1, g = 4G..4G+3
    k = np.arange(64)
    call = (k // 64) * 8 + ((k % 64) // 32) * 4 + (k % 8) // 2
    for cidx in range(8):
        cols = k[call == cidx]
        c = 2 * (cidx % 4)
        assert sorted(cols) == sorted([8 * g + c + e for g in range(4 * (cidx // 4), 4 * (cidx // 4) + 4) for e in (0, 1)])


def _case(golden, name, normformer=None):
    g = golden(name)
    cfg = dict(g["config"], hidden_dropout=0.1, attention_dropout=0.1)
    if normformer is not None:
        cfg["use_normformer"] = normformer
    if "batch" in g:
        fwd = dict(input_ids=g["batch"]["input_ids"], labels=g["batch"]["labels"], label_smoothing=g.get("label_smoothing", 0.0))
    else:
        fwd = dict(input_ids=g["input_ids"], labels=g["labels"], encoder_hidden_states=g["encoder_hidden_states"])
    return cfg, fwd


class _Replay(torch.nn.Module):
    """stands in for the reference's nn.Dropout: the recorded mask and the documented scale 1 / (1 - p_eff)"""

    def __init__(self, keep, scale):
        super().__init__()
        self.keep, self.scale = keep, scale

    def forward(self, x):
        if not self.training:
            return x
        return x * (self.keep.reshape(x.shape).to(x.dtype) * self.scale)


def _rel(a, b):
    a, b = a.detach().float(), b.detach().float()
    return float((a - b).norm() / b.norm().clamp_min(1e-20))


CASES = [("micro_transformer.pt", None), ("micro_t2i_transformer.pt", None), ("micro_t2i_proj_transformer.pt", None),
         ("micro_transformer.pt", False)]


@pytest.mark.parametrize("name,normformer", CASES)
def test_training_with_dropout_reproduces_the_reference_given_the_same_masks(golden, name, normformer):
    from oracle.ref_snapshot import import_reference

    cfg, fwd = _case(golden, name, normformer)
    torch.manual_seed(3)
    with pytest.MonkeyPatch.context() as mp:
        install(mp)
        m = MaskGitTransformer(**cfg).train()
        sd = {k: v.clone() for k, v in m.state_dict().items()}
        with ops.dropout_record() as log:
            logits, loss = m(**fwd)
        loss.backward()
        grads = {n: p.grad.clone() for n, p in m.named_parameters()}
    L = cfg["num_hidden_layers"]
    cross = bool(cfg.get("add_cross_attention"))
    expected = [0] + [s for i in range(L) for s in ([1 + 3 * i] + ([2 + 3 * i] if cross else []) + [3 + 3 * i])]
    assert [s for s, _ in log] == expected
    masks = dict(log)
    B, S = fwd["input_ids"].shape
    kept = torch.cat([unpack_bits(masks[3 + 3 * i], cfg["intermediate_size"]).flatten() for i in range(L)])
    assert 0.75 < float(kept.float().mean()) < 0.97  # the masks are not trivially all-kept or all-dropped

    muse = import_reference()
    torch.manual_seed(0)
    ref = muse.MaskGitTransformer(**cfg)
    ref.load_state_dict(sd)
    ref.train()
    sc = keep_scale(0.1)
    H, I = cfg["hidden_size"], cfg["intermediate_size"]
    ref.embed.dropout = _Replay(unpack_bits(masks[0], H), sc)
    for i, layer in enumerate(ref.transformer_layers):
        layer.attention.dropout = _Replay(unpack_bits(masks[1 + 3 * i], S), sc)
        if cross:
            layer.crossattention.dropout = _Replay(unpack_bits(masks[2 + 3 * i], fwd["encoder_hidden_states"].shape[1]), sc)
        layer.ffn.dropout = _Replay(unpack_bits(masks[3 + 3 * i], I), sc)
    r_logits, r_loss = ref(**fwd)
    r_loss.backward()
    assert _rel(logits, r_logits) < 2e-5
    assert abs(float(loss.detach()) - float(r_loss.detach())) < 2e-6 * abs(float(r_loss)) + 1e-7
    for n, p in ref.named_parameters():
        assert _rel(grads[n], p.grad) < 2e-4, (n, _rel(grads[n], p.grad))
    # and the masks did something: without them the reference computes other logits
    with torch.no_grad():
        ref.eval()
        assert _rel(logits, ref(fwd["input_ids"], encoder_hidden_states=fwd.get("encoder_hidden_states"))) > 1e-3


def _op_trace(mp, model, fwd, backward):
    calls = []
    names = [n for n in dir(ops) if callable(getattr(ops, n)) and not n.startswith("_") and n[0].islower()]
    for n in names:
        fn = getattr(ops, n)
        if isinstance(fn, type):
            continue

        def wrap(*a, _fn=fn, _n=n, **k):
            calls.append((_n, tuple(sorted(k))))
            return _fn(*a, **k)

        mp.setattr(ops, n, wrap)
    out = model(**fwd)
    if backward:
        out[1].backward()
    return calls


@pytest.mark.parametrize("name", ["micro_transformer.pt", "micro_t2i_transformer.pt"])
def test_inactive_dropout_leaves_the_op_sequence_alone(golden, name):
    """rate 0.0 in training mode and rate 0.1 in eval mode launch no dropout op and pass no dropout keyword: the same op
    calls, with the same keywords, as a model whose dropout rates are 0.0"""
    cfg, fwd = _case(golden, name)
    traces = {}
    for tag, p, train in (("zero-train", 0.0, True), ("drop-eval", 0.1, False), ("zero-eval", 0.0, False)):
        with pytest.MonkeyPatch.context() as mp:
            install(mp)
            torch.manual_seed(0)
            m = MaskGitTransformer(**dict(cfg, hidden_dropout=p, attention_dropout=p)).train(train)
            traces[tag] = _op_trace(mp, m, fwd, backward=train)
    for calls in traces.values():
        assert not any("dropout" in n or "dropout" in k for n, k in calls)
    assert traces["drop-eval"] == traces["zero-eval"]
    with pytest.MonkeyPatch.context() as mp:
        install(mp)
        m = MaskGitTransformer(**dict(cfg, hidden_dropout=0.1, attention_dropout=0.1)).train()
        drop_train = _op_trace(mp, m, fwd, backward=True)
    # with dropout on, the extra calls are exactly the dropout op of the embedding and the dropout keywords; the GLU /
    # mid-norm backward no longer gets the saved output (it is the dropped one); everything else is unchanged
    def strip(calls):
        return [(n, tuple(x for x in k if x not in ("dropout", "y_fwd"))) for n, k in calls if not n.startswith("dropout_")]

    assert [n for n, _ in drop_train if n.startswith("dropout_")] == ["dropout_fwd", "dropout_bwd"]
    assert strip(drop_train) == strip(traces["zero-train"])


def test_generate2_in_training_mode_with_dropout_raises(golden, monkeypatch):
    g = golden("micro_transformer.pt")
    cpu_math_ops.install(monkeypatch, exact=True)
    m = MaskGitTransformer(**dict(g["config"], hidden_dropout=0.1)).train()
    with pytest.raises(RuntimeError, match="eval"):
        m.generate2(class_ids=torch.tensor([1, 2]), timesteps=2, use_cuda_graph=False)
