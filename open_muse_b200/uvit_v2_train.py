"""Training step (forward with saved activations + hand-written backward) of ``MaskGiTUViT_v2`` on libmuse_b200.

Default path (``train_forward``): one ``torch.autograd.Function`` per block -- conditioning MLP, text-state projection, token
embedding, optional down-sampling convolution (``ResampleFn``), every ResBlock + AttentionBlock2D pair, the two projections,
every transformer layer, optional up-sampling transposed convolution, ConvMlmLayer + cross-entropy.  Each forward is the
inference path of ``modeling_transformer_v2.py`` with the activations its backward kernels need kept alive; each backward
returns the gradients of that block's parameters (reference names, fp32) as soon as it has run, so DDP's bucket all-reduces
overlap the rest of the backward pass.  ``UViTTrainFn`` (private test hook ``model._single_train_function``) is the same
computation as ONE Function for the whole network; the tests pin the two against each other.

All arithmetic is in the C-ABI kernels: wgmma GEMMs for every Linear / 1x1 / patch convolution (dgrad with an MN-major
weight operand, deterministic split-K wgrad), wgmma attention backward, and the U-ViT kernels of csrc/uvit_bwd.cu.  Things
that are single tensors consumed by many blocks get ONE accumulator: the text states (fp32, atomic-accumulating dgrad) and
the stacked adaLN mapper output (each op adds into its own column slice), so no gradient is summed with eager ops.
"""
from __future__ import annotations

import copy

import torch

from . import ops

BF16, F32 = torch.bfloat16, torch.float32


def _z(like, dtype=F32):
    return torch.zeros(like.shape, dtype=dtype, device=like.device)


def _lin_bwd(dy, x, w, g, dx_dtype=BF16, need_dx=True):
    """y = x @ w^T: g (fp32, same shape as w) += dy^T x ; returns dx = dy @ w."""
    ops.linear_wgrad(dy, x, g)
    return ops.linear_dgrad(dy, w, out_dtype=dx_dtype) if need_dx else None


class _G(dict):
    """fp32 gradient buffers mirroring the packed-weight dict W (created on first use)."""

    def __init__(self, W):
        super().__init__()
        self.W = W

    def of(self, key):
        if self.W[key] is None:  # e.g. a norm without elementwise affine
            return None
        if key not in self:
            self[key] = _z(self.W[key])
        return self[key]


def _sub(G, W, key, idx=None):
    """gradient dict for a nested block of W (W[key] is a dict, or a list of dicts when idx is given)."""
    holder = G.setdefault(key, {} if idx is None else {})
    if idx is None:
        if not isinstance(holder, _G):
            holder = G[key] = _G(W[key])
        return holder
    if idx not in holder:
        holder[idx] = _G(W[key][idx])
    return holder[idx]


# ------------------------------------------------------------------------------------------------ attention helper
def _attn_fwd(y, ctx_in, a, B, S, Skv, fused):
    Hc = a["o"].shape[0]
    if fused:
        qkv = ops.linear_fwd(y, a["qkv"])
        q, k, v = qkv[:, :Hc], qkv[:, Hc:2 * Hc], qkv[:, 2 * Hc:]
        saved = qkv
    else:
        q = ops.linear_fwd(y, a["q"])
        kv = ops.linear_fwd(ctx_in, a["kv"])
        k, v = kv[:, :Hc], kv[:, Hc:]
        saved = (q, kv)
    o, lse = ops.attn_fwd(q, k, v, B, a["nh"], S, Skv, a["sc"], head_dim=a["hd"])
    return o, (saved, o, lse)


def _attn_bwd(do, y, ctx_in, a, ga, st, B, S, Skv, fused, d_ctx_acc=None):
    """returns dy (bf16); the context gradient is accumulated into d_ctx_acc (fp32) for cross attention."""
    saved, o, lse = st
    Hc = a["o"].shape[0]
    if fused:
        qkv = saved
        dqkv = torch.empty_like(qkv)
        ops.attn_bwd(qkv[:, :Hc], qkv[:, Hc:2 * Hc], qkv[:, 2 * Hc:], o, do, lse, dqkv[:, :Hc], dqkv[:, Hc:2 * Hc],
                     dqkv[:, 2 * Hc:], B, a["nh"], S, Skv, a["sc"], head_dim=a["hd"])
        return _lin_bwd(dqkv, y, a["qkv"], ga.of("qkv"))
    q, kv = saved
    dq, dkv = torch.empty_like(q), torch.empty_like(kv)
    ops.attn_bwd(q, kv[:, :Hc], kv[:, Hc:], o, do, lse, dq, dkv[:, :Hc], dkv[:, Hc:], B, a["nh"], S, Skv, a["sc"],
                 head_dim=a["hd"])
    ops.linear_wgrad(dkv, ctx_in, ga.of("kv"))
    ops.linear_dgrad_acc(dkv, a["kv"], d_ctx_acc)
    return _lin_bwd(dq, y, a["q"], ga.of("q"))


# ------------------------------------------------------------------------------------------------ blocks
def _res_block_fwd(h, w, mod_all, B, hw, eps, rms):
    d, conv = ops.dwconv3x3_norm(h, w["dw"], w["dw_norm"], B, hw, hw, eps, rms, save_conv=True)
    g1 = ops.linear_fwd(d, w["cw0"])
    g2, stats = ops.grn(g1, w["gamma"], w["beta"], B, hw * hw, save_stats=True)
    h2 = ops.linear_fwd(g2, w["cw4"], res=h)
    o, n = w["mod"]
    h3 = ops.adaln_apply(h2, mod_all[:, o:o + n], B, hw * hw)
    return h3, (h, d, conv, g1, g2, stats, h2)


def _res_block_bwd(dh3, st, w, g, mod_all, d_mod_all, B, hw, eps, rms):
    h, d, conv, g1, g2, stats, h2 = st
    o, n = w["mod"]
    dh2 = ops.adaln_bwd(dh3, h2, mod_all[:, o:o + n], d_mod_all[:, o:o + n], B, hw * hw)
    dg2 = _lin_bwd(ops.cast_bf16(dh2), g2, w["cw4"], g.of("cw4"))
    dg1 = ops.grn_bwd(g1, dg2, stats, w["gamma"], g.of("gamma"), g.of("beta"), B, hw * hw)
    dd = _lin_bwd(dg1, d, w["cw0"], g.of("cw0"))
    return ops.dwconv3x3_norm_bwd(dd, conv, h, w["dw"], w["dw_norm"], dh2, g.of("dw"), g.of("dw_norm"), B, hw, hw, eps, rms)


def _attn_block_fwd(h, enc, w, B, S, Skv, eps, rms):
    se = encb = None
    if w["kvm"] is not None:
        se = ops.silu_bf16(enc)
        encb = ops.linear_fwd(se, w["kvm"])
    ctx_in = enc if encb is None else encb
    _, y1 = ops.add_norm_mod(h, w["ln1"], eps, rms, want_residual=False)
    c1, s1 = _attn_fwd(y1, ctx_in, w["a1"], B, S, Skv, False)
    a1o = ops.linear_fwd(c1, w["a1"]["o"])
    r2, y2 = ops.add_norm_mod(a1o, w["ln2"], eps, rms, residual=h)
    c2, s2 = _attn_fwd(y2, ctx_in, w["a2"], B, S, Skv, False)
    out = ops.linear_fwd(c2, w["a2"]["o"], res=r2)
    return out, (h, se, ctx_in, y1, c1, s1, r2, y2, c2, s2)


def _attn_block_bwd(dout, st, w, g, enc, d_enc, B, S, Skv, eps, rms):
    h, se, ctx_in, y1, c1, s1, r2, y2, c2, s2 = st
    g1, g2 = _sub(g, w, "a1"), _sub(g, w, "a2")
    d_ctx = d_enc if se is None else _z(ctx_in)  # fp32 accumulator of the (mapped) text states of this block
    dc2 = _lin_bwd(ops.cast_bf16(dout), c2, w["a2"]["o"], g2.of("o"))
    dy2 = _attn_bwd(dc2, y2, ctx_in, w["a2"], g2, s2, B, S, Skv, False, d_ctx)
    da1o, dh_res = ops.add_norm_mod_bwd(dy2, dout, r2, w["ln2"], eps, rms, BF16, dw=g.of("ln2"))
    dc1 = _lin_bwd(da1o, c1, w["a1"]["o"], g1.of("o"))
    dy1 = _attn_bwd(dc1, y1, ctx_in, w["a1"], g1, s1, B, S, Skv, False, d_ctx)
    dh, _ = ops.add_norm_mod_bwd(dy1, dh_res, h, w["ln1"], eps, rms, F32, dw=g.of("ln1"), want_dr=False)
    if se is not None:  # kv_mapper(silu(enc))
        d_se = _lin_bwd(ops.cast_bf16(d_ctx), se, w["kvm"], g.of("kvm"))
        ops.silu_bwd(d_se, enc, out=d_enc)
    return dh


def _layer_fwd(x, r, enc, w, mod_all, B, S, Skv, H, eps, rms):
    m = lambda k: mod_all[:, w[k][0]:w[k][0] + w[k][1]]
    r1, y1 = ops.add_norm_mod(x, w["ln1"], eps, rms, residual=r, mod=m("mod1"), rows_per_sample=S)
    c, s_sa = _attn_fwd(y1, None, w["sa"], B, S, S, True)
    a = ops.linear_fwd(c, w["sa"]["o"])
    r2, y2 = ops.add_norm_mod(a, w["ln2"], eps, rms, residual=r1, mod=m("mod2"), rows_per_sample=S)
    cc, s_ca = _attn_fwd(y2, enc, w["ca"], B, S, Skv, False)
    co = ops.linear_fwd(cc, w["ca"]["o"])
    r3, y3 = ops.add_norm_mod(co, w["ln3"], eps, 0, residual=r2, mod=m("mod3"), rows_per_sample=S)
    ab = ops.linear_fwd(y3, w["wi"])
    gl = ops.glu_fwd(ab)
    f = ops.linear_fwd(gl, w["wo"])
    return f, r3, (r is not None, r1, y1, c, s_sa, r2, y2, cc, s_ca, r3, y3, ab, gl)


def _layer_bwd(df, dr3, st, w, g, enc, d_enc, mod_all, d_mod_all, B, S, Skv, eps, rms):
    had_r, r1, y1, c, s_sa, r2, y2, cc, s_ca, r3, y3, ab, gl = st
    m = lambda t, k: t[:, w[k][0]:w[k][0] + w[k][1]]
    gsa, gca = _sub(g, w, "sa"), _sub(g, w, "ca")
    dgl = _lin_bwd(df, gl, w["wo"], g.of("wo"))
    dy3 = _lin_bwd(ops.glu_bwd(ab, dgl), y3, w["wi"], g.of("wi"))
    dco, dr2 = ops.add_norm_mod_bwd(dy3, dr3, r3, w["ln3"], eps, 0, BF16, mod=m(mod_all, "mod3"), rows_per_sample=S,
                                    dw=g.of("ln3"), dmod=m(d_mod_all, "mod3"))
    dcc = _lin_bwd(dco, cc, w["ca"]["o"], gca.of("o"))
    dy2 = _attn_bwd(dcc, y2, enc, w["ca"], gca, s_ca, B, S, Skv, False, d_enc)
    da, dr1 = ops.add_norm_mod_bwd(dy2, dr2, r2, w["ln2"], eps, rms, BF16, mod=m(mod_all, "mod2"), rows_per_sample=S,
                                   dw=g.of("ln2"), dmod=m(d_mod_all, "mod2"))
    dc = _lin_bwd(da, c, w["sa"]["o"], gsa.of("o"))
    dy1 = _attn_bwd(dc, y1, None, w["sa"], gsa, s_sa, B, S, S, True)
    dx, dr = ops.add_norm_mod_bwd(dy1, dr1, r1, w["ln1"], eps, rms, BF16, mod=m(mod_all, "mod1"), rows_per_sample=S,
                                  dw=g.of("ln1"), dmod=m(d_mod_all, "mod1"), want_dr=had_r)
    return dx, dr


# ------------------------------------------------------------------------------------------------ whole network
def forward(model, W, input_ids, encoder_hidden_states, cond_embeds, micro_conds):
    """Inference-identical forward that also returns the saved state for ``backward``."""
    from .modeling_transformer_v2 import sinusoidal_encode

    c = model.config
    B, S = input_ids.shape
    hw = int(S ** 0.5)
    rms, eps, H = (0 if c.norm_type == "layernorm" else 1), c.layer_norm_eps, c.hidden_size
    Skv = encoder_hidden_states.shape[1]
    ehs = encoder_hidden_states.reshape(B * Skv, -1).to(BF16).contiguous()
    r_enc, enc = ops.add_norm_mod(ops.linear_fwd(ehs, W["encoder_proj"]), W["enc_norm"], eps, rms)
    mc = sinusoidal_encode(micro_conds.flatten(), c.micro_cond_encode_dim).reshape(B, -1)
    cond_in = torch.cat([cond_embeds.float(), mc], dim=1).to(BF16).contiguous()
    c1 = ops.linear_fwd(cond_in, W["cond0"])
    c1s = ops.silu_bf16(c1)
    cond = ops.linear_fwd(c1s, W["cond2"])
    sc = ops.silu_bf16(cond)
    mod_all = ops.linear_fwd(sc, W["mappers"], out_dtype=F32)
    ids = input_ids.contiguous().to(torch.int64)
    e = ops.embed_fwd(ids, W["emb"], None)
    _, en = ops.add_norm_mod(e, W["emb_norm"], eps, rms, want_residual=False)
    h = ops.linear_fwd(en, W["emb_conv"], out_dtype=F32)
    blocks = {"down": [], "up": []}
    for w in W["down"]:
        h, s_r = _res_block_fwd(h, w, mod_all, B, hw, eps, rms)
        h, s_a = _attn_block_fwd(h, enc, w, B, S, Skv, eps, rms)
        blocks["down"].append((s_r, s_a))
    h_down = h
    _, y_pth = ops.add_norm_mod(h, W["pth_norm"], eps, rms, want_residual=False)
    x, r, layers = ops.linear_fwd(y_pth, W["pth"]), None, []
    for w in W["layers"]:
        x, r, s_l = _layer_fwd(x, r, enc, w, mod_all, B, S, Skv, H, eps, rms)
        layers.append(s_l)
    r_f, y_f = ops.add_norm_mod(x, W["pfh_norm"], eps, rms, residual=r)
    h = ops.linear_fwd(y_f, W["pfh"], out_dtype=F32)
    for w in W["up"]:
        h, s_r = _res_block_fwd(h, w, mod_all, B, hw, eps, rms)
        h, s_a = _attn_block_fwd(h, enc, w, B, S, Skv, eps, rms)
        blocks["up"].append((s_r, s_a))
    hb = ops.cast_bf16(h)
    y1 = ops.linear_fwd(hb, W["mlm1"])
    r_m, y2 = ops.add_norm_mod(y1, W["mlm_norm"], eps, rms)
    logits = ops.linear_fwd(y2, W["mlm2"])
    saved = dict(B=B, S=S, hw=hw, Skv=Skv, ehs=ehs, r_enc=r_enc, enc=enc, cond_in=cond_in, c1=c1, c1s=c1s, cond=cond, sc=sc,
                 mod_all=mod_all, ids=ids, e=e, en=en, blocks=blocks, h_down=h_down, y_pth=y_pth, layers=layers, r_f=r_f,
                 y_f=y_f, hb=hb, y1=y1, r_m=r_m, y2=y2)
    return logits, saved


def backward(model, W, saved, d_logits):
    """d_logits: bf16 [B*S, vpad].  Returns the nested fp32 gradient dict G mirroring W."""
    c = model.config
    s = saved
    B, S, hw, Skv = s["B"], s["S"], s["hw"], s["Skv"]
    rms, eps = (0 if c.norm_type == "layernorm" else 1), c.layer_norm_eps
    enc, mod_all = s["enc"], s["mod_all"]
    G = _G(W)
    d_enc = _z(enc)          # fp32 accumulator: the text states feed every cross attention
    d_mod = _z(mod_all)      # every adaLN op adds into its own column slice
    # ConvMlmLayer
    dy2 = _lin_bwd(d_logits, s["y2"], W["mlm2"], G.of("mlm2"))
    dy1, _ = ops.add_norm_mod_bwd(dy2, None, s["r_m"], W["mlm_norm"], eps, rms, BF16, dw=G.of("mlm_norm"), want_dr=False)
    dh = _lin_bwd(dy1, s["hb"], W["mlm1"], G.of("mlm1"), dx_dtype=F32)
    for i in reversed(range(len(W["up"]))):
        w, g = W["up"][i], _sub(G, W, "up", i)
        s_r, s_a = s["blocks"]["up"][i]
        dh = _attn_block_bwd(dh, s_a, w, g, enc, d_enc, B, S, Skv, eps, rms)
        dh = _res_block_bwd(dh, s_r, w, g, mod_all, d_mod, B, hw, eps, rms)
    dy_f = _lin_bwd(ops.cast_bf16(dh), s["y_f"], W["pfh"], G.of("pfh"))
    dx, dr = ops.add_norm_mod_bwd(dy_f, None, s["r_f"], W["pfh_norm"], eps, rms, BF16, dw=G.of("pfh_norm"))
    for i in reversed(range(len(W["layers"]))):
        dx, dr = _layer_bwd(dx, dr, s["layers"][i], W["layers"][i], _sub(G, W, "layers", i), enc, d_enc, mod_all, d_mod, B, S,
                            Skv, eps, rms)
    dy_pth = _lin_bwd(dx, s["y_pth"], W["pth"], G.of("pth"))
    dh, _ = ops.add_norm_mod_bwd(dy_pth, None, s["h_down"], W["pth_norm"], eps, rms, F32, dw=G.of("pth_norm"), want_dr=False)
    for i in reversed(range(len(W["down"]))):
        w, g = W["down"][i], _sub(G, W, "down", i)
        s_r, s_a = s["blocks"]["down"][i]
        dh = _attn_block_bwd(dh, s_a, w, g, enc, d_enc, B, S, Skv, eps, rms)
        dh = _res_block_bwd(dh, s_r, w, g, mod_all, d_mod, B, hw, eps, rms)
    # ConvEmbed
    d_en = _lin_bwd(ops.cast_bf16(dh), s["en"], W["emb_conv"], G.of("emb_conv"))
    d_e, _ = ops.add_norm_mod_bwd(d_en, None, s["e"], W["emb_norm"], eps, rms, F32, dw=G.of("emb_norm"), want_dr=False)
    ops.embed_bwd(s["ids"], d_e, G.of("emb"), None)
    # conditioning: stacked adaLN mappers <- SiLU <- cond_embed MLP
    d_sc = _lin_bwd(ops.cast_bf16(d_mod), s["sc"], W["mappers"], G.of("mappers"))
    d_cond = ops.silu_bwd(d_sc, s["cond"])
    d_c1s = _lin_bwd(d_cond, s["c1s"], W["cond2"], G.of("cond2"))
    d_c1 = ops.silu_bwd(d_c1s, s["c1"])
    _lin_bwd(d_c1, s["cond_in"], W["cond0"], G.of("cond0"), need_dx=False)
    # text states: encoder_proj + norm
    d_y0, _ = ops.add_norm_mod_bwd(d_enc, None, s["r_enc"], W["enc_norm"], eps, rms, BF16, dw=G.of("enc_norm"), want_dr=False)
    _lin_bwd(d_y0, s["ehs"], W["encoder_proj"], G.of("encoder_proj"), need_dx=False)
    return G


def param_grads(model, G):
    """Maps the packed gradient buffers back onto the parameters (reference names), in ``model.parameters()`` order."""
    c = model.config
    out = {}

    def put(p, g):
        if p is not None and g is not None:
            out[p] = g.reshape(p.shape)

    def rows(g, *ps):
        o = 0
        for p in ps:
            put(p, g[o:o + p.shape[0]])
            o += p.shape[0]

    def attn(a, g, fused):
        if fused:
            rows(g["qkv"], a.query.weight, a.key.weight, a.value.weight)
        else:
            put(a.query.weight, g["q"])
            rows(g["kv"], a.key.weight, a.value.weight)
        put(a.out.weight, g["o"])

    mappers = []

    def block(blk, gl):
        for i, (rb, ab) in enumerate(zip(blk.res_blocks, blk.attention_blocks)):
            g = gl[i]
            put(rb.depthwise.weight, g["dw"].t().contiguous())
            put(rb.norm.norm.weight, g.get("dw_norm"))
            put(rb.channelwise[0].weight, g["cw0"])
            put(rb.channelwise[2].gamma, g["gamma"])
            put(rb.channelwise[2].beta, g["beta"])
            put(rb.channelwise[4].weight, g["cw4"])
            mappers.append(rb.adaLN_modulation.mapper.weight)
            if ab.kv_mapper is not None:
                put(ab.kv_mapper.weight, g["kvm"])
            put(ab.attn_layer_norm.weight, g.get("ln1"))
            attn(ab.attention, g["a1"], False)
            put(ab.crossattn_layer_norm.weight, g.get("ln2"))
            attn(ab.crossattention, g["a2"], False)

    put(model.encoder_proj.weight, G["encoder_proj"])
    put(model.encoder_proj_layer_norm.weight, G.get("enc_norm"))
    put(model.cond_embed[0].weight, G["cond0"])
    put(model.cond_embed[2].weight, G["cond2"])
    put(model.embed.embeddings.weight, G["emb"])
    put(model.embed.layer_norm.weight, G.get("emb_norm"))
    put(model.embed.conv.weight, G["emb_conv"])
    put(model.project_to_hidden_norm.weight, G.get("pth_norm"))
    put(model.project_to_hidden.weight, G["pth"])
    put(model.project_from_hidden_norm.weight, G.get("pfh_norm"))
    put(model.project_from_hidden.weight, G["pfh"])
    put(model.mlm_layer.conv1.weight, G["mlm1"])
    put(model.mlm_layer.layer_norm.norm.weight, G.get("mlm_norm"))
    put(model.mlm_layer.conv2.weight, G["mlm2"][: c.codebook_size])
    block(model.down_blocks[0], G["down"])  # mapper order must match _weights(): down, layers, up
    for i, l in enumerate(model.transformer_layers):
        g = G["layers"][i]
        put(l.attn_layer_norm.weight, g.get("ln1"))
        mappers.append(l.self_attn_adaLN_modulation.mapper.weight)
        attn(l.attention, g["sa"], True)
        put(l.crossattn_layer_norm.weight, g.get("ln2"))
        attn(l.crossattention, g["ca"], False)
        mappers.append(l.cross_attn_adaLN_modulation.mapper.weight)
        put(l.ffn.pre_mlp_layer_norm.weight, g.get("ln3"))
        mappers.append(l.ffn.adaLN_modulation.mapper.weight)
        rows(g["wi"], l.ffn.wi_0.weight, l.ffn.wi_1.weight)
        put(l.ffn.wo.weight, g["wo"])
    block(model.up_blocks[0], G["up"])
    rows(G["mappers"], *mappers)
    return [out.get(p) for p in model.parameters()]


class UViTTrainFn(torch.autograd.Function):
    """(logits_padded, loss) = f(params...): the whole MaskGiTUViT_v2 training forward; backward returns every gradient."""

    @staticmethod
    def forward(ctx, model, input_ids, encoder_hidden_states, cond_embeds, micro_conds, labels, label_smoothing,
                loss_weight, *params):
        W = model._weights()
        logits, saved = forward(model, W, input_ids, encoder_hidden_states, cond_embeds, micro_conds)
        V = model.config.codebook_size
        ctx.model, ctx.W, ctx.saved, ctx.V, ctx.ls = model, W, saved, V, label_smoothing
        ctx.set_materialize_grads(False)
        if labels is None:
            ctx.ce = None
            return logits, None
        labels = labels.reshape(-1).contiguous().to(torch.int64)
        out, ws = ops.ce_fwd(logits, labels, V, label_smoothing)
        row_scale, loss = None, out[0]
        if loss_weight is not None:  # (sum_r w_r loss_r) / sum_r w_r on the unreduced loss (:305-317)
            lw = loss_weight.reshape(-1).float()
            row_scale = (lw / lw.sum()).contiguous()
            loss = (ws[1] * row_scale).sum()
        ctx.ce = (labels, ws, out, row_scale)
        ctx.save_for_backward(logits)  # an OUTPUT of this Function: as a plain ctx attribute it would form a reference cycle
        return logits, loss

    @staticmethod
    def backward(ctx, d_logits, d_loss):
        dl = None
        if d_loss is not None and ctx.ce is not None:
            labels, ws, out, row_scale = ctx.ce
            dl = ops.ce_bwd(ctx.saved_tensors[0], labels, ws, d_loss.to(F32).reshape(1).contiguous(), out, ctx.V, ctx.ls,
                            row_scale=row_scale)
        if d_logits is not None:
            extra = d_logits.to(BF16).contiguous()
            dl = extra if dl is None else dl + extra
        if dl is None:
            raise RuntimeError("MaskGiTUViT_v2: backward called without any gradient")
        G = backward(ctx.model, ctx.W, ctx.saved, dl)
        grads = param_grads(ctx.model, G)
        ctx.saved = None
        return (None,) * 8 + tuple(grads)


# =================================================================================================================
# Per-block autograd Functions: the same forward / backward helpers as above, cut at the block boundaries so that the
# gradients of a block's parameters exist as soon as its backward has run and DDP's bucket all-reduces overlap the rest
# of the backward pass (the whole-network Function above releases everything at the very end).  Tensors consumed by
# every block enter each Function as fp32 inputs -- the normalised text states ``enc32`` and the SiLU'd conditioning
# vector ``sc32`` -- and autograd sums their per-block gradients; each block computes its own adaLN (scale | shift) rows
# from ``sc`` with its slice of the stacked mapper matrix.
class _Shared:
    """per-forward constants and bf16 operand copies shared by the block Functions"""

    def __init__(self, model, W, B, S, Skv):
        c = model.config
        self.W, self.B, self.S, self.Skv, self.hw = W, B, S, Skv, int(S ** 0.5)
        self.rms, self.eps, self.H = (0 if c.norm_type == "layernorm" else 1), c.layer_norm_eps, c.hidden_size
        self.enc = self.sc = None  # bf16 GEMM operands of enc32 / sc32


def _present(params):
    return [p for p in params if p is not None]


def _align(params, grads):
    """gradients of the non-None parameters, in order"""
    return [g.reshape(p.shape) for p, g in zip(params, grads) if p is not None]


def _local_mods(sh, w, keys):
    """this block's rows of the stacked mapper matrix and its W entry re-based onto the block-local (scale | shift) tensor"""
    base = w[keys[0]][0]
    total = sum(w[k][1] for k in keys)
    wl = dict(w)
    for k in keys:
        wl[k] = (w[k][0] - base, w[k][1])
    return wl, sh.W["mappers"][base:base + total]


def _mapper_bwd(sh, d_mod, w_map):
    g_map = _z(w_map)
    d_sc32 = _lin_bwd(ops.cast_bf16(d_mod), sh.sc, w_map, g_map, dx_dtype=F32)
    return g_map, d_sc32


def _attn_params(a):
    return [a.query.weight, a.key.weight, a.value.weight, a.out.weight]


def _attn_grads(g, a, fused):
    n = a.query.weight.shape[0]
    if fused:
        q, k, v = g["qkv"][:n], g["qkv"][n:2 * n], g["qkv"][2 * n:]
    else:
        q, k, v = g["q"], g["kv"][:n], g["kv"][n:]
    return [q, k, v, g["o"]]


class CondFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, sh, cond_in, w0, w2):
        W = sh.W
        c1 = ops.linear_fwd(cond_in, W["cond0"])
        c1s = ops.silu_bf16(c1)
        cond = ops.linear_fwd(c1s, W["cond2"])
        sh.sc = ops.silu_bf16(cond)
        ctx.sh, ctx.sv = sh, (cond_in, c1, c1s, cond)
        ctx.set_materialize_grads(False)
        return sh.sc.float()

    @staticmethod
    def backward(ctx, d_sc32):
        W, (cond_in, c1, c1s, cond) = ctx.sh.W, ctx.sv
        g0, g2 = _z(W["cond0"]), _z(W["cond2"])
        d_cond = ops.silu_bwd(ops.cast_bf16(d_sc32.contiguous()), cond)
        d_c1 = ops.silu_bwd(_lin_bwd(d_cond, c1s, W["cond2"], g2), c1)
        _lin_bwd(d_c1, cond_in, W["cond0"], g0, need_dx=False)
        ctx.sv = None  # release the block's activations now, not when the graph dies
        return None, None, g0, g2


class EncFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, sh, ehs, w_proj, w_norm):
        W = sh.W
        r_enc, sh.enc = ops.add_norm_mod(ops.linear_fwd(ehs, W["encoder_proj"]), W["enc_norm"], sh.eps, sh.rms)
        ctx.sh, ctx.sv, ctx.has_norm = sh, (ehs, r_enc), w_norm is not None
        ctx.set_materialize_grads(False)
        return sh.enc.float()

    @staticmethod
    def backward(ctx, d_enc32):
        sh, (ehs, r_enc) = ctx.sh, ctx.sv
        W = sh.W
        g_p = _z(W["encoder_proj"])
        g_n = _z(W["enc_norm"]) if ctx.has_norm else None
        d_y0, _ = ops.add_norm_mod_bwd(d_enc32.contiguous(), None, r_enc, W["enc_norm"], sh.eps, sh.rms, BF16, dw=g_n, want_dr=False)
        _lin_bwd(d_y0, ehs, W["encoder_proj"], g_p, need_dx=False)
        ctx.sv = None  # release the block's activations now, not when the graph dies
        return None, None, g_p, g_n


class EmbedFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, sh, ids, w_emb, w_norm, w_conv):
        W = sh.W
        e = ops.embed_fwd(ids, W["emb"], None)
        _, en = ops.add_norm_mod(e, W["emb_norm"], sh.eps, sh.rms, want_residual=False)
        ctx.sh, ctx.sv, ctx.has_norm, ctx.conv_shape = sh, (ids, e, en), w_norm is not None, w_conv.shape
        ctx.set_materialize_grads(False)
        return ops.linear_fwd(en, W["emb_conv"], out_dtype=F32)

    @staticmethod
    def backward(ctx, dh):
        sh, (ids, e, en) = ctx.sh, ctx.sv
        W = sh.W
        g_c, g_e = _z(W["emb_conv"]), _z(W["emb"])
        g_n = _z(W["emb_norm"]) if ctx.has_norm else None
        d_en = _lin_bwd(ops.cast_bf16(dh.contiguous()), en, W["emb_conv"], g_c)
        d_e, _ = ops.add_norm_mod_bwd(d_en, None, e, W["emb_norm"], sh.eps, sh.rms, F32, dw=g_n, want_dr=False)
        ops.embed_bwd(ids, d_e, g_e, None)
        ctx.sv = None  # release the block's activations now, not when the graph dies
        return None, None, g_e, g_n, g_c.reshape(ctx.conv_shape)


def block_params(rb, ab):
    return [rb.depthwise.weight, rb.norm.norm.weight, rb.channelwise[0].weight, rb.channelwise[2].gamma, rb.channelwise[2].beta,
            rb.channelwise[4].weight, rb.adaLN_modulation.mapper.weight, None if ab.kv_mapper is None else ab.kv_mapper.weight,
            ab.attn_layer_norm.weight] + _attn_params(ab.attention) + [ab.crossattn_layer_norm.weight] + _attn_params(ab.crossattention)


class UBlockFn(torch.autograd.Function):
    """ResBlock + AttentionBlock2D pair of the down / up stage"""

    @staticmethod
    def forward(ctx, sh, model, which, idx, h, enc32, sc32, *params):
        w = sh.W[which][idx]
        wl, w_map = _local_mods(sh, w, ["mod"])
        mod = ops.linear_fwd(sh.sc, w_map, out_dtype=F32)
        h, s_r = _res_block_fwd(h, wl, mod, sh.B, sh.hw, sh.eps, sh.rms)
        h, s_a = _attn_block_fwd(h, sh.enc, wl, sh.B, sh.S, sh.Skv, sh.eps, sh.rms)
        ctx.sh, ctx.sv, ctx.key = sh, (wl, w_map, mod, s_r, s_a), (model, which, idx)
        ctx.set_materialize_grads(False)
        return h

    @staticmethod
    def backward(ctx, dh):
        sh, (wl, w_map, mod, s_r, s_a), (model, which, idx) = ctx.sh, ctx.sv, ctx.key
        stage = model.down_blocks[0] if which == "down" else model.up_blocks[0]
        rb, ab = stage.res_blocks[idx], stage.attention_blocks[idx]
        g, d_enc, d_mod = _G(wl), _z(sh.enc), _z(mod)
        dh = _attn_block_bwd(dh.contiguous(), s_a, wl, g, sh.enc, d_enc, sh.B, sh.S, sh.Skv, sh.eps, sh.rms)
        dh = _res_block_bwd(dh, s_r, wl, g, mod, d_mod, sh.B, sh.hw, sh.eps, sh.rms)
        g_map, d_sc32 = _mapper_bwd(sh, d_mod, w_map)
        params = block_params(rb, ab)
        grads = [g["dw"].t().contiguous(), g.get("dw_norm"), g["cw0"], g["gamma"], g["beta"], g["cw4"], g_map, g.get("kvm"),
                 g.get("ln1")] + _attn_grads(g["a1"], ab.attention, False) + [g.get("ln2")] + _attn_grads(g["a2"], ab.crossattention, False)
        ctx.sv = None  # release the block's activations now, not when the graph dies
        return (None, None, None, None, dh, d_enc, d_sc32, *_align(params, grads))


def layer_params(l):
    return [l.attn_layer_norm.weight, l.self_attn_adaLN_modulation.mapper.weight] + _attn_params(l.attention) + \
        [l.crossattn_layer_norm.weight] + _attn_params(l.crossattention) + \
        [l.cross_attn_adaLN_modulation.mapper.weight, l.ffn.pre_mlp_layer_norm.weight, l.ffn.adaLN_modulation.mapper.weight,
         l.ffn.wi_0.weight, l.ffn.wi_1.weight, l.ffn.wo.weight]


class ULayerFn(torch.autograd.Function):
    """one TransformerLayer carrying (hidden, residual)"""

    @staticmethod
    def forward(ctx, sh, model, idx, x, r, enc32, sc32, *params):
        w = sh.W["layers"][idx]
        wl, w_map = _local_mods(sh, w, ["mod1", "mod2", "mod3"])
        mod = ops.linear_fwd(sh.sc, w_map, out_dtype=F32)
        f, r3, s_l = _layer_fwd(x, r, sh.enc, wl, mod, sh.B, sh.S, sh.Skv, sh.H, sh.eps, sh.rms)
        s_l = list(s_l)
        assert s_l[9] is r3
        s_l[9] = None  # r3 is an OUTPUT of this Function: held through save_for_backward, a ctx attribute would be a cycle
        ctx.save_for_backward(r3)
        ctx.sh, ctx.sv, ctx.key = sh, (wl, w_map, mod, s_l), (model, idx)
        ctx.set_materialize_grads(False)
        return f, r3

    @staticmethod
    def backward(ctx, df, dr3):
        sh, (wl, w_map, mod, s_l), (model, idx) = ctx.sh, ctx.sv, ctx.key
        s_l = list(s_l)
        s_l[9] = ctx.saved_tensors[0]
        l = model.transformer_layers[idx]
        g, d_enc, d_mod = _G(wl), _z(sh.enc), _z(mod)
        if df is None:
            df = torch.zeros(s_l[1].shape, dtype=BF16, device=s_l[1].device)
        dx, dr = _layer_bwd(df.contiguous(), None if dr3 is None else dr3.contiguous(), s_l, wl, g, sh.enc, d_enc, mod, d_mod,
                            sh.B, sh.S, sh.Skv, sh.eps, sh.rms)
        g_map, d_sc32 = _mapper_bwd(sh, d_mod, w_map)
        H2 = 2 * sh.H
        I = l.ffn.wi_0.weight.shape[0]
        params = layer_params(l)
        grads = [g.get("ln1"), g_map[:H2]] + _attn_grads(g["sa"], l.attention, True) + [g.get("ln2")] + \
            _attn_grads(g["ca"], l.crossattention, False) + [g_map[H2:2 * H2], g.get("ln3"), g_map[2 * H2:], g["wi"][:I], g["wi"][I:],
                                                             g["wo"]]
        ctx.sv = None  # release the block's activations now, not when the graph dies
        return (None, None, None, dx, dr, d_enc, d_sc32, *_align(params, grads))


class ProjFn(torch.autograd.Function):
    """project_to_hidden (norm + Linear, residual=None) and project_from_hidden ((x + residual) -> norm + Linear)"""

    @staticmethod
    def forward(ctx, sh, key, x, r, w_norm, w_lin):
        W = sh.W
        r_out, y = ops.add_norm_mod(x, W[key + "_norm"], sh.eps, sh.rms, residual=r)
        ctx.sh, ctx.sv, ctx.key, ctx.has_norm = sh, (r_out, y, x.dtype, r is not None), key, w_norm is not None
        ctx.set_materialize_grads(False)
        return ops.linear_fwd(y, W[key], out_dtype=BF16 if key == "pth" else F32)

    @staticmethod
    def backward(ctx, d_out):
        sh, (r_out, y, x_dtype, had_r), key = ctx.sh, ctx.sv, ctx.key
        W = sh.W
        g_l = _z(W[key])
        g_n = _z(W[key + "_norm"]) if ctx.has_norm else None
        d = d_out.contiguous()
        dy = _lin_bwd(d if d.dtype == BF16 else ops.cast_bf16(d), y, W[key], g_l)
        dx, dr = ops.add_norm_mod_bwd(dy, None, r_out, W[key + "_norm"], sh.eps, sh.rms, x_dtype, dw=g_n, want_dr=had_r)
        ctx.sv = None  # release the block's activations now, not when the graph dies
        return None, None, dx, dr, g_n, g_l


class ResampleFn(torch.autograd.Function):
    """force_down_up_sample (reference :509-513, :555-559): ``ds`` = Norm2D + Conv2d(k=2, s=2) in front of the down stage,
    ``us`` = Norm2D + ConvTranspose2d(k=2, s=2) behind the up stage.  Both are ONE GEMM on the token-major layout: the
    strided conv reads 2x2 patches ``[B*S/4, (dy, dx, ci)]``, the transposed conv writes ``[B*S, (dy, dx, co)]`` followed
    by depth-to-space; the backward is the same GEMM's dgrad / wgrad with the inverse token permutation around it.
    ``sh`` describes the grid this op READS (hw x hw tokens per sample)."""

    @staticmethod
    def forward(ctx, sh, key, h, w_norm, w_conv):
        W, B, hw = sh.W, sh.B, sh.hw
        C = h.shape[1]
        if h.dtype != F32 or h.shape[0] != B * hw * hw:
            raise ValueError(f"ResampleFn: expected fp32 [{B * hw * hw}, C] tokens, got {h.dtype} {tuple(h.shape)}")
        h = h.contiguous()
        _, y = ops.add_norm_mod(h, W[key + "_norm"], sh.eps, sh.rms, want_residual=False)
        if key == "ds":
            a = y.view(B, hw // 2, 2, hw // 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(B * hw * hw // 4, 4 * C)
            out = ops.linear_fwd(a, W["ds"], out_dtype=F32)
        else:
            a = y
            t = ops.linear_fwd(y, W["us"], out_dtype=F32)
            out = t.view(B, hw, hw, 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(B * hw * hw * 4, C)
        ctx.sh, ctx.sv, ctx.key = sh, (h, a), key
        ctx.has_norm, ctx.conv_shape = w_norm is not None, w_conv.shape
        ctx.set_materialize_grads(False)
        return out

    @staticmethod
    def backward(ctx, d_out):
        sh, (h, a), key = ctx.sh, ctx.sv, ctx.key
        W, B, hw = sh.W, sh.B, sh.hw
        C = h.shape[1]
        g_w = _z(W[key])
        g_n = _z(W[key + "_norm"]) if ctx.has_norm else None
        d = d_out.contiguous()
        if key == "ds":  # d: [B*S/4, co] -> patches [B*S/4, (dy, dx, ci)] -> tokens [B*S, ci]
            dp = _lin_bwd(d if d.dtype == BF16 else ops.cast_bf16(d), a, W["ds"], g_w)
            dy = dp.view(B, hw // 2, hw // 2, 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(B * hw * hw, C)
            g_conv = g_w.view(C, 2, 2, C).permute(0, 3, 1, 2)  # [co, (dy, dx, ci)] -> Conv2d weight [co, ci, dy, dx]
        else:            # d: [B*S*4, co] -> space-to-depth [B*S, (dy, dx, co)] -> tokens [B*S, ci]
            dt = d.view(B, hw, 2, hw, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(B * hw * hw, 4 * C)
            dy = _lin_bwd(dt if dt.dtype == BF16 else ops.cast_bf16(dt), a, W["us"], g_w)
            g_conv = g_w.view(2, 2, C, C).permute(3, 2, 0, 1)  # [(dy, dx, co), ci] -> ConvTranspose2d weight [ci, co, dy, dx]
        dh, _ = ops.add_norm_mod_bwd(dy, None, h, W[key + "_norm"], sh.eps, sh.rms, F32, dw=g_n, want_dr=False)
        ctx.sv = None  # release the activations now, not when the graph dies
        return None, None, dh, g_n, g_conv.reshape(ctx.conv_shape)


class TailFn(torch.autograd.Function):
    """ConvMlmLayer + cross-entropy"""

    @staticmethod
    def forward(ctx, sh, V, h, labels, label_smoothing, loss_weight, w1, w_norm, w2):
        W = sh.W
        hb = ops.cast_bf16(h)
        y1 = ops.linear_fwd(hb, W["mlm1"])
        r_m, y2 = ops.add_norm_mod(y1, W["mlm_norm"], sh.eps, sh.rms)
        logits = ops.linear_fwd(y2, W["mlm2"])
        ctx.sh, ctx.sv, ctx.V, ctx.ls = sh, (hb, r_m, y2), V, label_smoothing
        ctx.save_for_backward(logits)  # output of this Function (see ULayerFn)
        ctx.has_norm, ctx.shapes = w_norm is not None, (w1.shape, w2.shape)
        ctx.set_materialize_grads(False)
        if labels is None:
            ctx.ce = None
            return logits, None
        labels = labels.reshape(-1).contiguous().to(torch.int64)
        out, ws = ops.ce_fwd(logits, labels, V, label_smoothing)
        row_scale, loss = None, out[0]
        if loss_weight is not None:
            lw = loss_weight.reshape(-1).float()
            row_scale = (lw / lw.sum()).contiguous()
            loss = (ws[1] * row_scale).sum()
        ctx.ce = (labels, ws, out, row_scale)
        return logits, loss

    @staticmethod
    def backward(ctx, d_logits, d_loss):
        sh, (hb, r_m, y2) = ctx.sh, ctx.sv
        logits = ctx.saved_tensors[0]
        W = sh.W
        dl = None
        if d_loss is not None and ctx.ce is not None:
            labels, ws, out, row_scale = ctx.ce
            dl = ops.ce_bwd(logits, labels, ws, d_loss.to(F32).reshape(1).contiguous(), out, ctx.V, ctx.ls, row_scale=row_scale)
        if d_logits is not None:
            extra = d_logits.to(BF16).contiguous()
            dl = extra if dl is None else dl + extra
        if dl is None:
            raise RuntimeError("MaskGiTUViT_v2: backward called without any gradient")
        g1, g2 = _z(W["mlm1"]), _z(W["mlm2"])
        g_n = _z(W["mlm_norm"]) if ctx.has_norm else None
        dy2 = _lin_bwd(dl, y2, W["mlm2"], g2)
        dy1, _ = ops.add_norm_mod_bwd(dy2, None, r_m, W["mlm_norm"], sh.eps, sh.rms, BF16, dw=g_n, want_dr=False)
        dh = _lin_bwd(dy1, hb, W["mlm1"], g1, dx_dtype=F32)
        ctx.sv = None  # release the block's activations now, not when the graph dies
        return None, None, dh, None, None, None, g1.reshape(ctx.shapes[0]), g_n, g2[: ctx.V].reshape(ctx.shapes[1])


def train_forward(model, input_ids, encoder_hidden_states, cond_embeds, micro_conds, labels, label_smoothing, loss_weight):
    """(logits_padded, loss) through the per-block Functions."""
    from .modeling_transformer_v2 import sinusoidal_encode

    c = model.config
    W = model._weights()
    B, S = input_ids.shape
    Skv = encoder_hidden_states.shape[1]
    sh = _Shared(model, W, B, S, Skv)
    ehs = encoder_hidden_states.reshape(B * Skv, -1).to(BF16).contiguous()
    mc = sinusoidal_encode(micro_conds.flatten(), c.micro_cond_encode_dim).reshape(B, -1)
    cond_in = torch.cat([cond_embeds.float(), mc], dim=1).to(BF16).contiguous()
    sc32 = CondFn.apply(sh, cond_in, model.cond_embed[0].weight, model.cond_embed[2].weight)
    enc32 = EncFn.apply(sh, ehs, model.encoder_proj.weight, model.encoder_proj_layer_norm.weight)
    h = EmbedFn.apply(sh, input_ids.contiguous().to(torch.int64), model.embed.embeddings.weight, model.embed.layer_norm.weight,
                      model.embed.conv.weight)
    down, up = model.down_blocks[0], model.up_blocks[0]
    sh_full = sh
    if c.force_down_up_sample:  # the stages and the transformer layers run on the (hw/2)^2 grid (reference :509-513)
        if sh.hw % 2:
            raise ValueError(f"force_down_up_sample needs an even token grid, got {sh.hw}x{sh.hw}")
        h = ResampleFn.apply(sh_full, "ds", h, down.downsample[0].norm.weight, down.downsample[1].weight)
        sh = copy.copy(sh_full)  # same operand caches (W, enc, sc), coarse grid
        sh.S, sh.hw = S // 4, sh_full.hw // 2
    for i, (rb, ab) in enumerate(zip(down.res_blocks, down.attention_blocks)):
        h = UBlockFn.apply(sh, model, "down", i, h, enc32, sc32, *_present(block_params(rb, ab)))
    x = ProjFn.apply(sh, "pth", h, None, model.project_to_hidden_norm.weight, model.project_to_hidden.weight)
    r = None
    for i, l in enumerate(model.transformer_layers):
        x, r = ULayerFn.apply(sh, model, i, x, r, enc32, sc32, *_present(layer_params(l)))
    h = ProjFn.apply(sh, "pfh", x, r, model.project_from_hidden_norm.weight, model.project_from_hidden.weight)
    for i, (rb, ab) in enumerate(zip(up.res_blocks, up.attention_blocks)):
        h = UBlockFn.apply(sh, model, "up", i, h, enc32, sc32, *_present(block_params(rb, ab)))
    if c.force_down_up_sample:  # back to the full grid (:555-559); sh still describes the coarse grid this op reads
        h = ResampleFn.apply(sh, "us", h, up.upsample[0].norm.weight, up.upsample[1].weight)
        sh = sh_full
    return TailFn.apply(sh, c.codebook_size, h, labels, label_smoothing, loss_weight, model.mlm_layer.conv1.weight,
                        model.mlm_layer.layer_norm.norm.weight, model.mlm_layer.conv2.weight)
