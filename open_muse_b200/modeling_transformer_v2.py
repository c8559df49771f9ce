"""``MaskGiTUViT_v2`` -- the U-ViT text-to-image transformer of the reference (muse/modeling_transformer_v2.py) behind the
reference's surface: same constructor keys (``MaskGiTUViT_v2Config`` :79-123, unknown keys dropped like
``config_from_legacy_kwargs`` :126-147), same parameter names / shapes / construction order (so ``torch.manual_seed(s);
MaskGiTUViT_v2(**cfg)`` reproduces the reference's initial weights, including the special initialisations of :206-223),
``forward(input_ids, encoder_hidden_states, cond_embeds, micro_conds, labels=, label_smoothing=, loss_weight=)`` and the
classifier-free-guidance ``generate2`` (:330-479).

Everything runs on libmuse_b200: wgmma GEMMs for every Linear / 1x1 conv, wgmma attention, fused prenorm-residual
norm + adaLN modulation, depthwise-conv + Norm2D, GELU + GlobalResponseNorm, the fused decode step.  The block forwards
(ResBlock, AttentionBlock2D, TransformerLayer, the force_down_up_sample resampling) are defined once in ``uvit_v2_train.py``
next to their hand-written backwards; inference (``_forward_tokens``) calls them without keeping their saved state, training
runs them inside one autograd Function per block.  The modules below are parameter containers.
Activations are token-major ``[B*h*w, C]`` throughout -- the NCHW <-> NHWC permutes of the reference disappear.
"""
from __future__ import annotations

import math
from functools import partial
from typing import Tuple

import numpy as np
import torch
from torch import nn

from . import ops
from . import uvit_v2_train as T
from .modeling_utils import ConfigMixin, ModelMixin
from .sampling import cosine_schedule

_CONFIG_DEFAULTS = dict(
    hidden_size=1024, use_bias=False, hidden_dropout=0.0, cond_embed_dim=768, micro_cond_encode_dim=256,
    micro_cond_embed_dim=1280, encoder_hidden_size=768, vocab_size=8256, mask_token_id=8255, codebook_size=8192,
    in_channels=768, block_out_channels=(768,), num_res_blocks=3, force_down_up_sample=False, block_num_heads=12,
    num_hidden_layers=22, num_attention_heads=16, attention_dropout=0.0, intermediate_size=2816, use_fused_mlp=False,
    norm_type="rmsnorm", layer_norm_eps=1e-6, ln_elementwise_affine=True, use_fused_residual_norm=False,
    add_cond_embeds=True, add_micro_cond_embeds=True)


def sinusoidal_encode(features, embedding_dim, max_positions=10000):
    """[cos(f w_k), sin(f w_k)], w_k = max_positions^(-k / (dim/2)) (reference :59-76); a few hundred values per sample."""
    half = embedding_dim // 2
    w = torch.exp(torch.arange(half, device=features.device, dtype=torch.float32) * (-math.log(max_positions) / half))
    emb = features[:, None].float() * w[None, :]
    emb = torch.cat([emb.cos(), emb.sin()], dim=1)
    if embedding_dim % 2 == 1:
        emb = nn.functional.pad(emb, (0, 1))
    return emb


# ---------------------------------------------------------------------------------------------- parameter containers
class _NormP(nn.Module):
    """LayerNorm / RMSNorm parameter holder (weight only: use_bias=False everywhere)."""

    def __init__(self, dim, affine):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(dim)) if affine else None


class LayerNorm(_NormP):
    pass


class RMSNorm(_NormP):
    pass


def _norm(dim, cfg, kind=None):
    return (LayerNorm if (kind or cfg["norm_type"]) == "layernorm" else RMSNorm)(dim, cfg["ln_elementwise_affine"])


class Norm2D(nn.Module):
    def __init__(self, dim, cfg):
        super().__init__()
        self.norm = _norm(dim, cfg)


class GlobalResponseNorm(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.gamma = nn.Parameter(torch.zeros(1, 1, 1, dim))
        self.beta = nn.Parameter(torch.zeros(1, 1, 1, dim))


class AdaLNModulation(nn.Module):
    def __init__(self, hidden_size, cfg):
        super().__init__()
        self.mapper = nn.Linear(cfg["hidden_size"], hidden_size * 2, bias=False)


class Attention(nn.Module):
    def __init__(self, hidden_size, context_dim, num_heads, cfg):
        super().__init__()
        if hidden_size % num_heads != 0:
            raise ValueError(f"self.hidden_size: {hidden_size} must be divisible by self.num_heads: {num_heads}")
        if hidden_size // num_heads not in (48, 64, 96, 128):
            raise NotImplementedError("open_muse_b200.MaskGiTUViT_v2: head_dim must be 48, 64, 96 or 128 (every U-ViT config "
                                      "of the reference uses 64); the attention kernels are built for these four widths")
        self.num_heads = num_heads
        self.query = nn.Linear(hidden_size, hidden_size, bias=False)
        self.key = nn.Linear(context_dim, hidden_size, bias=False)
        self.value = nn.Linear(context_dim, hidden_size, bias=False)
        self.out = nn.Linear(hidden_size, hidden_size, bias=False)
        self.dropout = nn.Dropout(cfg["attention_dropout"])


class ResBlock(nn.Module):
    def __init__(self, channels, cfg, res_ffn_factor=4):
        super().__init__()
        self.depthwise = nn.Conv2d(channels, channels, kernel_size=3, padding=1, groups=channels, bias=False)
        self.norm = Norm2D(channels, cfg)
        self.channelwise = nn.Sequential(
            nn.Linear(channels, int(channels * res_ffn_factor), bias=False),
            nn.GELU(),
            GlobalResponseNorm(int(channels * res_ffn_factor)),
            nn.Dropout(cfg["hidden_dropout"]),
            nn.Linear(int(channels * res_ffn_factor), channels, bias=False),
        )
        self.adaLN_modulation = AdaLNModulation(channels, cfg)


class AttentionBlock2D(nn.Module):
    def __init__(self, hidden_size, cfg):
        super().__init__()
        self.kv_mapper = nn.Linear(cfg["hidden_size"], hidden_size, bias=False) if cfg["hidden_size"] != hidden_size else None
        self.attn_layer_norm = _norm(hidden_size, cfg)
        self.attention = Attention(hidden_size, hidden_size, cfg["block_num_heads"], cfg)
        self.crossattn_layer_norm = _norm(hidden_size, cfg)
        self.crossattention = Attention(hidden_size, hidden_size, cfg["block_num_heads"], cfg)


class DownsampleBlock(nn.Module):
    """(:505-523) optional Norm2D + Conv2d(k=2, s=2) in front of the res/attention blocks; module order == reference."""

    def __init__(self, channels, cfg):
        super().__init__()
        self.downsample = (nn.Sequential(Norm2D(channels, cfg), nn.Conv2d(channels, channels, kernel_size=2, stride=2, bias=False))
                           if cfg["force_down_up_sample"] else None)
        self.res_blocks = nn.ModuleList([ResBlock(channels, cfg) for _ in range(cfg["num_res_blocks"])])
        self.attention_blocks = nn.ModuleList([AttentionBlock2D(channels, cfg) for _ in range(cfg["num_res_blocks"])])
        self.gradient_checkpointing = False


class UpsampleBlock(nn.Module):
    """(:543-565) res/attention blocks followed by an optional Norm2D + ConvTranspose2d(k=2, s=2)."""

    def __init__(self, channels, cfg):
        super().__init__()
        self.res_blocks = nn.ModuleList([ResBlock(channels, cfg) for _ in range(cfg["num_res_blocks"])])
        self.attention_blocks = nn.ModuleList([AttentionBlock2D(channels, cfg) for _ in range(cfg["num_res_blocks"])])
        self.upsample = (nn.Sequential(Norm2D(channels, cfg), nn.ConvTranspose2d(channels, channels, kernel_size=2, stride=2, bias=False))
                         if cfg["force_down_up_sample"] else None)
        self.gradient_checkpointing = False


class GLUFeedForward(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.pre_mlp_layer_norm = LayerNorm(cfg["hidden_size"], cfg["ln_elementwise_affine"])  # always LayerNorm (:929)
        self.adaLN_modulation = AdaLNModulation(cfg["hidden_size"], cfg)
        self.wi_0 = nn.Linear(cfg["hidden_size"], cfg["intermediate_size"], bias=False)
        self.wi_1 = nn.Linear(cfg["hidden_size"], cfg["intermediate_size"], bias=False)
        self.dropout = nn.Dropout(cfg["hidden_dropout"])
        self.wo = nn.Linear(cfg["intermediate_size"], cfg["hidden_size"], bias=False)


class FusedGeLUFeedForward(nn.Module):
    """use_fused_mlp (:954-996): wo(gelu_tanh(wi_0(x))), no gate.  ``dropout`` is constructed (it fixes the module order)
    but, as in the reference, never applied."""

    def __init__(self, cfg):
        super().__init__()
        self.pre_mlp_layer_norm = LayerNorm(cfg["hidden_size"], cfg["ln_elementwise_affine"])  # always LayerNorm (:957)
        self.adaLN_modulation = AdaLNModulation(cfg["hidden_size"], cfg)
        self.wi_0 = nn.Linear(cfg["hidden_size"], cfg["intermediate_size"], bias=False)
        self.dropout = nn.Dropout(cfg["hidden_dropout"])
        self.wo = nn.Linear(cfg["intermediate_size"], cfg["hidden_size"], bias=False)


class TransformerLayer(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        H, nh = cfg["hidden_size"], cfg["num_attention_heads"]
        self.attn_layer_norm = _norm(H, cfg)
        self.self_attn_adaLN_modulation = AdaLNModulation(H, cfg)
        self.attention = Attention(H, H, nh, cfg)
        self.crossattn_layer_norm = _norm(H, cfg)
        self.crossattention = Attention(H, H, nh, cfg)
        self.cross_attn_adaLN_modulation = AdaLNModulation(H, cfg)
        self.ffn = (FusedGeLUFeedForward if cfg["use_fused_mlp"] else GLUFeedForward)(cfg)  # FeedForward (:919-923)


class ConvEmbed(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.embeddings = nn.Embedding(cfg["vocab_size"], cfg["in_channels"])
        self.layer_norm = _norm(cfg["in_channels"], cfg)
        self.conv = nn.Conv2d(cfg["in_channels"], cfg["block_out_channels"][0], kernel_size=1, bias=False)


class ConvMlmLayer(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.conv1 = nn.Conv2d(cfg["block_out_channels"][0], cfg["in_channels"], kernel_size=1, bias=False)
        self.layer_norm = Norm2D(cfg["in_channels"], cfg)
        self.conv2 = nn.Conv2d(cfg["in_channels"], cfg["codebook_size"], kernel_size=1, bias=False)


# ---------------------------------------------------------------------------------------------------------- the model
class _OperandCache:
    """The fused optimizers' view of ``MaskGiTUViT_v2._weights()``, the same protocol as ``MaskGitTransformer._packed``:
    ``refresh()`` brings the cache up to date and returns an object whose ``dst_of`` maps a parameter's data_ptr to its bf16
    copy, which the optimizer's pass writes; after the step ``sync()`` recomputes the few operands that are not such a copy
    (``derived``: the transposed depthwise weights, the permuted down / up-sample weights) in place -- graph-capturable
    copies -- and moves the cache's key to the parameters' new version counters, so the next forward rebuilds nothing.
    In FP8 mode it also re-quantizes the e4m3 weight operands (``quantized``: (bf16 operand, its F8 copy)) from the bf16
    operands the step has just written, so no FP8 copy is left stale by a step that moves the key without a rebuild."""

    def __init__(self, model):
        self.model = model
        self.dst_of, self.derived, self.quantized = {}, [], []

    def refresh(self):
        self.model._weights()
        return self

    def sync(self):
        m = self.model
        if m._cache_key is None:
            return
        for dst, src in self.derived:
            dst.copy_(src())
        for src, dst in self.quantized:
            ops.quantize_rows_e4m3(src, out=dst)
        m._cache_key = m._weights_key()


class MaskGiTUViT_v2(ModelMixin, ConfigMixin):
    _supports_gradient_checkpointing = True

    def __init__(self, **kwargs):
        super().__init__()
        cfg = dict(_CONFIG_DEFAULTS)
        if isinstance(kwargs.get("block_num_heads"), (tuple, list)):
            assert len(kwargs["block_num_heads"]) == 1
            kwargs["block_num_heads"] = kwargs["block_num_heads"][0]
        cfg.update({k: v for k, v in kwargs.items() if k in _CONFIG_DEFAULTS})  # unknown keys are dropped (:126-147)
        cfg["block_out_channels"] = list(cfg["block_out_channels"])
        self.register_to_config(**cfg)
        self.register_to_config(mask_token_id=cfg["vocab_size"] - 1)
        assert len(cfg["block_out_channels"]) == 1
        if cfg["use_bias"]:
            raise NotImplementedError("open_muse_b200.MaskGiTUViT_v2: use_bias=True is not supported")
        self.output_size = cfg["codebook_size"]
        H, C = cfg["hidden_size"], cfg["block_out_channels"][0]

        # construction order == reference (:169-203) so that seeded initialisation is identical
        self.encoder_proj = nn.Linear(cfg["encoder_hidden_size"], H, bias=False)
        self.encoder_proj_layer_norm = _norm(H, cfg)
        self.embed = ConvEmbed(cfg)
        self.cond_embed = nn.Sequential(
            nn.Linear(cfg["micro_cond_embed_dim"] + cfg["cond_embed_dim"], H, bias=False),
            nn.SiLU(),
            nn.Linear(H, H, bias=False),
        )
        self.down_blocks = nn.ModuleList([DownsampleBlock(C, cfg)])
        self.project_to_hidden_norm = _norm(C, cfg)
        self.project_to_hidden = nn.Linear(C, H, bias=False)
        self.transformer_layers = nn.ModuleList([TransformerLayer(cfg) for _ in range(cfg["num_hidden_layers"])])
        self.project_from_hidden_norm = _norm(H, cfg)
        self.project_from_hidden = nn.Linear(H, C, bias=False)
        self.up_blocks = nn.ModuleList([UpsampleBlock(C, cfg)])
        self.mlm_layer = ConvMlmLayer(cfg)
        self.gradient_checkpointing = False

        # weight init, same calls in the same order as the reference (:206-223)
        self.apply(self._init_weights)
        nn.init.xavier_uniform_(self.embed.conv.weight, 0.02)
        nn.init.normal_(self.embed.embeddings.weight, std=np.sqrt(1 / cfg["vocab_size"]))
        nn.init.constant_(self.mlm_layer.conv1.weight, 0)
        self.mlm_layer.conv2.weight.data = self.embed.embeddings.weight.data[: cfg["codebook_size"], :, None, None].clone()
        for m in self.modules():
            if isinstance(m, AdaLNModulation):
                nn.init.constant_(m.mapper.weight, 0)
        self._cache_key, self._cache = None, None
        self._gemm_precision = "bf16"
        self._packed = _OperandCache(self)  # the fused optimizers' handle on the cache (model=)
        self._debug_stages = None  # tests set this to a dict to receive the block-boundary activations
        self._graph = None         # CUDA graph of one decode-step forward (generate2), keyed by shapes and weight versions

    def _init_weights(self, module):
        if isinstance(module, (nn.Linear, nn.Conv2d)):
            nn.init.trunc_normal_(module.weight, std=0.02)
        elif isinstance(module, nn.Embedding):
            nn.init.trunc_normal_(module.weight, std=0.02)
        elif isinstance(module, (LayerNorm, RMSNorm)):
            if module.weight is not None:
                module.weight.data.fill_(1.0)

    def _set_gradient_checkpointing(self, module, value=False):
        self.gradient_checkpointing = value
        if isinstance(module, (DownsampleBlock, UpsampleBlock)):
            module.gradient_checkpointing = value

    def enable_gradient_checkpointing(self):
        """Recompute activations in the backward instead of keeping them: every transformer layer, and the res + attention
        pairs of the down / up stages (each stage's own flag, as the reference's ``_set_gradient_checkpointing`` sets them).
        The recomputed activations are bit-identical to the saved ones, so the gradients equal those without it (up to the
        fp32-atomic summation order of the weight gradients, as between any two runs); only training forwards that a
        backward can follow recompute."""
        self.apply(partial(self._set_gradient_checkpointing, value=True))

    def disable_gradient_checkpointing(self):
        self.apply(partial(self._set_gradient_checkpointing, value=False))

    def generate(self):
        assert False  # (reference :326-328)

    # ------------------------------------------------------------------------------------ GEMM precision
    def set_gemm_precision(self, mode: str):
        """"bf16" (default: the reference's autocast recipe) or "fp8": inference only -- forward under torch.no_grad() in
        eval mode, and generate2 -- with the e4m3 tensor cores for the transformer layers' [q;k;v], cross-attention q,
        [wi_0;wi_1] (wi_0 with use_fused_mlp) and wo GEMMs and the ResBlock / AttentionBlock2D channelwise[0] and q GEMMs.
        Their activations come out of the passes that produce them as e4m3 with one scale per row, the weights are
        quantized per output row; every other GEMM stays bf16 (DESIGN.md section 5).  Not a config key: save_pretrained /
        from_pretrained do not see it.
        "fp8" needs hidden_size, block_out_channels[0] and intermediate_size to be multiples of 16 (the e4m3 rows are fed
        by TMA, whose row pitches are multiples of 16 bytes); bf16 needs multiples of 8."""
        if mode not in ("bf16", "fp8"):
            raise ValueError(f"gemm precision must be 'bf16' or 'fp8', got {mode!r}")
        c = self.config
        widths = dict(hidden_size=c.hidden_size, block_out_channels=c.block_out_channels[0],
                      intermediate_size=c.intermediate_size)
        bad = {k: v for k, v in widths.items() if v % 16}
        if mode == "fp8" and bad:
            raise ValueError(f"gemm precision 'fp8' needs widths that are multiples of 16, got {bad}")
        self._gemm_precision = mode  # part of the operand cache key: the next forward rebuilds the operands
        return self

    @property
    def gemm_precision(self) -> str:
        return self._gemm_precision

    def _check_fp8_inference(self):
        if self._gemm_precision == "fp8" and (self.training or torch.is_grad_enabled()):
            raise RuntimeError("MaskGiTUViT_v2 in FP8 GEMM precision is inference only: call model.eval() and run under "
                               "torch.no_grad(), or set_gemm_precision('bf16') to train")

    # ------------------------------------------------------------------------------------ bf16 operand cache
    def _weights_key(self):
        return (self._gemm_precision,) + tuple((p.data_ptr(), p._version) for p in self.parameters())

    def _weights(self):
        """bf16 GEMM operands (fused [k;v], [q;k;v], [wi_0;wi_1] (wi_0 alone with use_fused_mlp), all adaLN mappers
        stacked into one matrix, logits rows padded to 64), rebuilt only when a parameter changes -- never inside
        generate2, and not after a fused optimizer step with ``model=``, which writes them itself (``_packed``)."""
        key = self._weights_key()
        if key == self._cache_key:
            return self._cache
        W, self._packed.dst_of, self._packed.derived, self._packed.quantized = self._build_weights()
        self._cache_key, self._cache = key, W
        return W

    def _build_weights(self):
        """(W, dst_of, derived, quantized): the operand dict; parameter data_ptr -> address of its bf16 copy, for every
        parameter whose operand is a plain row block of one bf16 matrix; (destination, source view) of the operands that
        are not: the transposed fp32 depthwise weights and the permuted down / up-sample weights; and in FP8 mode
        (bf16 operand, F8 copy) of the FP8 sites, whose W entries are then the F8 copies (the bf16 operands stay, as the
        fused optimizers' destinations)."""
        dev = next(self.parameters()).device
        dst_of, derived = {}, []

        def bf(*ws):
            out = torch.cat([w.detach().reshape(w.shape[0], -1) for w in ws], dim=0).to(torch.bfloat16).contiguous()
            r = 0
            for w in ws:
                dst_of[w.data_ptr()] = out[r: r + w.shape[0]].data_ptr()
                r += w.shape[0]
            return out

        def derive(dtype, shape, src):  # src() is a view of the parameter laid out as the operand viewed as `shape`
            out = torch.empty(shape, dtype=dtype, device=dev)
            view = out.view(src().shape)
            view.copy_(src())
            derived.append((view, src))
            return out

        # fp32 operands of contiguous fp32 parameters are the parameters themselves (no copy to keep current)
        f32 = lambda w: None if w is None else w.detach().float().contiguous()
        W = {"encoder_proj": bf(self.encoder_proj.weight), "enc_norm": f32(self.encoder_proj_layer_norm.weight),
             "cond0": bf(self.cond_embed[0].weight), "cond2": bf(self.cond_embed[2].weight),
             "emb": f32(self.embed.embeddings.weight), "emb_norm": f32(self.embed.layer_norm.weight),
             "emb_conv": bf(self.embed.conv.weight), "pth_norm": f32(self.project_to_hidden_norm.weight),
             "pth": bf(self.project_to_hidden.weight), "pfh_norm": f32(self.project_from_hidden_norm.weight),
             "pfh": bf(self.project_from_hidden.weight), "mlm1": bf(self.mlm_layer.conv1.weight),
             "mlm_norm": f32(self.mlm_layer.layer_norm.norm.weight)}
        V = self.config.codebook_size
        vpad = ((V + 63) // 64) * 64
        w2 = torch.zeros(vpad, self.config.in_channels, dtype=torch.bfloat16, device=dev)
        w2[:V] = self.mlm_layer.conv2.weight.detach().reshape(V, -1).to(torch.bfloat16)
        dst_of[self.mlm_layer.conv2.weight.data_ptr()] = w2[:V].data_ptr()  # the padding rows stay zero
        W["mlm2"], W["vpad"] = w2, vpad
        mappers, off = [], 0

        def mapper(m):
            nonlocal off
            mappers.append(m.mapper.weight)
            o = (off, m.mapper.weight.shape[0])
            off += m.mapper.weight.shape[0]
            return o

        def attn(a, fuse_q):
            hd = a.out.weight.shape[0] // a.num_heads  # 64: scale 0.125 exactly; 48, 96 or 128 otherwise
            d = {"o": bf(a.out.weight), "nh": a.num_heads, "hd": hd, "sc": 1.0 / math.sqrt(hd)}
            if fuse_q:  # self-attention reads k and v from [q;k;v] only: no separate [k;v] copy of the same weights
                d["qkv"] = bf(a.query.weight, a.key.weight, a.value.weight)
            else:
                d["q"], d["kv"] = bf(a.query.weight), bf(a.key.weight, a.value.weight)
            return d

        def block(blk):
            out = []
            for rb, ab in zip(blk.res_blocks, blk.attention_blocks):
                dw = rb.depthwise.weight
                out.append({
                    "dw": derive(torch.float32, (9, dw.shape[0]), lambda dw=dw: dw.detach().reshape(dw.shape[0], 9).t()),
                    "dw_norm": f32(rb.norm.norm.weight), "cw0": bf(rb.channelwise[0].weight),
                    "gamma": f32(rb.channelwise[2].gamma.reshape(-1)), "beta": f32(rb.channelwise[2].beta.reshape(-1)),
                    "cw4": bf(rb.channelwise[4].weight), "mod": mapper(rb.adaLN_modulation),
                    "kvm": None if ab.kv_mapper is None else bf(ab.kv_mapper.weight),
                    "ln1": f32(ab.attn_layer_norm.weight), "a1": attn(ab.attention, False),
                    "ln2": f32(ab.crossattn_layer_norm.weight), "a2": attn(ab.crossattention, False)})
            return out

        if c_down := self.down_blocks[0].downsample:  # [co, ci, dy, dx] -> [co, (dy, dx, ci)]: a GEMM over 2x2 patches
            W["ds_norm"] = f32(c_down[0].norm.weight)
            wd = c_down[1].weight
            W["ds"] = derive(torch.bfloat16, (wd.shape[0], wd[0].numel()), lambda: wd.detach().permute(0, 2, 3, 1))
            c_up = self.up_blocks[0].upsample  # ConvTranspose2d weight [ci, co, dy, dx] -> [(dy, dx, co), ci]
            W["us_norm"] = f32(c_up[0].norm.weight)
            wu = c_up[1].weight
            W["us"] = derive(torch.bfloat16, (wu[0].numel(), wu.shape[0]), lambda: wu.detach().permute(2, 3, 1, 0))
        W["down"] = block(self.down_blocks[0])
        W["layers"] = []
        for l in self.transformer_layers:
            W["layers"].append({
                "ln1": f32(l.attn_layer_norm.weight), "mod1": mapper(l.self_attn_adaLN_modulation),
                "sa": attn(l.attention, True), "ln2": f32(l.crossattn_layer_norm.weight), "ca": attn(l.crossattention, False),
                "mod2": mapper(l.cross_attn_adaLN_modulation), "ln3": f32(l.ffn.pre_mlp_layer_norm.weight),
                "mod3": mapper(l.ffn.adaLN_modulation), "wi": bf(*T._ffn_wi(l.ffn)),
                "glu": isinstance(l.ffn, GLUFeedForward),  # else FusedGeLUFeedForward: "wi" is wi_0 alone, no gate
                "wo": bf(l.ffn.wo.weight)})
        W["up"] = block(self.up_blocks[0])
        W["mappers"] = bf(*mappers)
        quantized = []
        if self._gemm_precision == "fp8":
            def f8(d, k):
                quantized.append((d[k], ops.quantize_rows_e4m3(d[k])))
                d[k] = quantized[-1][1]

            for w in W["down"] + W["up"]:
                f8(w, "cw0"), f8(w["a1"], "q"), f8(w["a2"], "q")
            for w in W["layers"]:
                f8(w["sa"], "qkv"), f8(w["ca"], "q"), f8(w, "wi"), f8(w, "wo")
        return W, dst_of, derived, quantized

    # ------------------------------------------------------------------------------------------- forward
    def _forward_tokens(self, input_ids, encoder_hidden_states, cond_embeds, micro_conds, drop=None):
        """drop: the forward's dropout (p_hidden, p_attn, seed) in training mode, else None (uvit_v2_train.unit_drop)"""
        c = self.config
        if not input_ids.is_cuda:
            raise RuntimeError("open_muse_b200.MaskGiTUViT_v2 runs on CUDA (sm_90a) only; move inputs to the GPU")
        B, S = input_ids.shape
        hw = int(S ** 0.5)
        if hw * hw != S:
            raise ValueError(f"sequence length {S} is not a square token grid")
        W = self._weights()
        rms, eps = (0 if c.norm_type == "layernorm" else 1), c.layer_norm_eps
        Skv = encoder_hidden_states.shape[1]
        ehs = encoder_hidden_states.reshape(B * Skv, -1).to(torch.bfloat16).contiguous()
        _, enc = ops.add_norm_mod(ops.linear_fwd(ehs, W["encoder_proj"]), W["enc_norm"], eps, rms, want_residual=False)
        mc = sinusoidal_encode(micro_conds.flatten(), c.micro_cond_encode_dim).reshape(B, -1)
        cond_in = torch.cat([cond_embeds.float(), mc], dim=1).to(torch.bfloat16).contiguous()
        cond = ops.linear_fwd(ops.silu_bf16(ops.linear_fwd(cond_in, W["cond0"])), W["cond2"])
        mod_all = ops.linear_fwd(ops.silu_bf16(cond), W["mappers"], out_dtype=torch.float32)  # every adaLN (scale | shift)
        # ConvEmbed: gather -> norm -> 1x1 conv
        e = ops.embed_fwd(input_ids.contiguous().to(torch.int64), W["emb"], None)
        _, en = ops.add_norm_mod(e, W["emb_norm"], eps, rms, want_residual=False)
        h = ops.linear_fwd(en, W["emb_conv"], out_dtype=torch.float32)
        dbg = self._debug_stages
        if dbg is not None:
            dbg.update(enc=enc.float().view(B, Skv, -1), cond=cond.float(), embed=h.view(B, S, -1).clone())
        if "ds" in W:  # force_down_up_sample (:509-513)
            h, _ = T._resample_fwd(h, W, "ds", B, hw, eps, rms)
            hw, S = hw // 2, S // 4
            if dbg is not None:
                dbg["downsample"] = h.view(B, hw, hw, -1).permute(0, 3, 1, 2).clone()
        R, L = len(W["down"]), len(W["layers"])
        for j, w in enumerate(W["down"]):
            dj = T.unit_drop(drop, j)
            h, _ = T._res_block_fwd(h, w, mod_all, B, hw, eps, rms, save=False, drop=dj)
            h, _ = T._attn_block_fwd(h, enc, w, B, S, Skv, eps, rms, drop=dj)
        if dbg is not None:
            dbg["down"] = h.view(B, S, -1).clone()
        _, y = ops.add_norm_mod(h, W["pth_norm"], eps, rms, want_residual=False)
        x, r = ops.linear_fwd(y, W["pth"]), None
        if dbg is not None:
            dbg["hidden0"] = x.float().view(B, S, -1)
        for i, w in enumerate(W["layers"]):
            x, r, _ = T._layer_fwd(x, r, enc, w, mod_all, B, S, Skv, eps, rms, drop=T.unit_drop(drop, R + i))
            if dbg is not None:
                dbg[f"layer{i}"] = (x.float() + r).view(B, S, -1)
        _, y = ops.add_norm_mod(x, W["pfh_norm"], eps, rms, residual=r, want_residual=False)  # (x + residual) -> norm (:289-291)
        h = ops.linear_fwd(y, W["pfh"], out_dtype=torch.float32)
        if dbg is not None:
            dbg["from_hidden"] = h.view(B, S, -1).clone()
        for j, w in enumerate(W["up"]):
            dj = T.unit_drop(drop, R + L + j)
            h, _ = T._res_block_fwd(h, w, mod_all, B, hw, eps, rms, save=False, drop=dj)
            h, _ = T._attn_block_fwd(h, enc, w, B, S, Skv, eps, rms, drop=dj)
        if dbg is not None:
            dbg["up"] = h.view(B, S, -1).clone()
        if "us" in W:  # (:555-559)
            h, _ = T._resample_fwd(h, W, "us", B, hw, eps, rms)
            hw, S = hw * 2, S * 4
            if dbg is not None:
                dbg["upsample"] = h.view(B, hw, hw, -1).permute(0, 3, 1, 2).clone()
        # ConvMlmLayer: 1x1 conv -> Norm2D -> 1x1 conv
        y1 = ops.linear_fwd(ops.cast_bf16(h), W["mlm1"])
        _, y2 = ops.add_norm_mod(y1, W["mlm_norm"], eps, rms, want_residual=False)
        return ops.linear_fwd(y2, W["mlm2"])  # bf16 [B*S, vpad]

    def forward(self, input_ids, encoder_hidden_states, cond_embeds, micro_conds, labels=None, label_smoothing=0.0,
                loss_weight=None, _raw_bf16=False):
        c = self.config
        B, S = input_ids.shape
        self._check_fp8_inference()
        # nn.Dropout is active iff the module is in training mode (also under no_grad), each rate gating its own sites.
        # One seed per forward, drawn on the device from torch's default generator as MaskGitTransformer does:
        # torch.manual_seed reproduces the masks.  Site ids: uvit_v2_train.unit_drop.
        drop = None
        if self.training and (c.hidden_dropout > 0.0 or c.attention_dropout > 0.0):
            seed = torch.randint(-2 ** 63, 2 ** 63 - 1, (1,), dtype=torch.int64, device=input_ids.device)
            drop = (float(c.hidden_dropout), float(c.attention_dropout), seed)
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            # training: one autograd Function per block, so parameter gradients appear during backward (DDP overlap)
            padded, loss = T.train_forward(self, input_ids, encoder_hidden_states, cond_embeds, micro_conds, labels,
                                           label_smoothing, loss_weight, drop=drop)
            logits = padded.view(B, S, -1)[:, :, : c.codebook_size]
            if not (_raw_bf16 or torch.is_autocast_enabled()):
                logits = logits.float()
            return logits if labels is None else (logits, loss)
        with torch.no_grad():
            padded = self._forward_tokens(input_ids, encoder_hidden_states, cond_embeds, micro_conds, drop=drop)
            V = c.codebook_size
            logits = padded.view(B, S, -1)[:, :, :V]
            if not (_raw_bf16 or torch.is_autocast_enabled()):
                logits = logits.float()
            if labels is None:
                return logits
            out, ws = ops.ce_fwd(padded, labels.reshape(-1).contiguous().to(torch.int64), V, label_smoothing)
            if loss_weight is not None:  # per-token weighting of the unreduced loss (:305-317)
                lw = loss_weight.reshape(-1).float()
                loss = (ws[1] * lw).sum() / lw.sum()
            else:
                loss = out[0]
            return logits, loss

    # ------------------------------------------------------------------------------------------- CUDA graph of one forward
    def _graphed_forward(self, model_in, enc, cond, micro):
        """Replays a captured CUDA graph of ``_forward_tokens`` (≈420 kernel launches per decode step, which at small batch
        are bound by launch latency, not by the GPU).  Captured once per (shapes, weight versions); inputs are copied into
        the graph's static buffers.  Returns the static logits buffer, valid until the next replay."""
        self._weights()  # make sure the operand cache is built outside the capture
        key = (tuple(model_in.shape), tuple(enc.shape), tuple(cond.shape), enc.dtype, cond.dtype, model_in.device, self._cache_key)
        st = self._graph
        if st is None or st["key"] != key:
            bufs = [t.clone() for t in (model_in, enc, cond, micro)]
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):  # warm-up off the capture: lazy attribute / cache initialisation
                self._forward_tokens(*bufs)
            torch.cuda.current_stream().wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                out = self._forward_tokens(*bufs)
            st = self._graph = dict(key=key, graph=graph, bufs=bufs, out=out)
        for dst, src in zip(st["bufs"], (model_in, enc, cond, micro)):
            dst.copy_(src)
        st["graph"].replay()
        return st["out"]

    # ------------------------------------------------------------------------------------------- generate2
    @torch.no_grad()
    def generate2(self, encoder_hidden_states, cond_embeds, micro_conds, empty_embeds, empty_cond_embeds, input_ids=None,
                  negative_embeds=None, negative_cond_embeds=None, temperature=1.0, timesteps=18, guidance_scale=0,
                  guidance_schedule=None, noise_schedule=cosine_schedule, generator=None, return_intermediate=False,
                  seq_len=None, use_tqdm=None, topk_filter_thres=None, noise_type=None, predict_all_tokens=None,
                  use_cuda_graph=None):
        """MaskGIT parallel decoding with classifier-free guidance, semantics of the reference (:330-479); per step one
        doubled-batch forward and ONE fused kernel (guidance mix, categorical sample, confidence, k-th cut, re-mask)."""
        c = self.config
        self._check_fp8_inference()
        if self.training and (c.hidden_dropout > 0.0 or c.attention_dropout > 0.0):
            # the reference would sample with dropout applied to every forward of the decode loop
            raise RuntimeError("generate2 on a MaskGiTUViT_v2 in training mode would sample with dropout > 0 active; "
                               "call model.eval() first")
        B = encoder_hidden_states.shape[0]
        seq_len = 256 if seq_len is None else seq_len
        mask_id, K = c.mask_token_id, c.codebook_size
        temps = torch.linspace(temperature[0], temperature[1], timesteps) if isinstance(temperature, tuple) else \
            torch.linspace(temperature, 0.01, timesteps)
        if input_ids is None:
            input_ids = torch.full((B, seq_len), mask_id, dtype=torch.long, device=self.device)
        if guidance_schedule == "linear":
            scales = torch.linspace(0, guidance_scale, timesteps)
        elif guidance_schedule == "cosine":
            scales = torch.tensor([float((cosine_schedule(torch.tensor(1 - (s + 1) / timesteps)) * guidance_scale).floor())
                                   for s in range(timesteps)])
        else:
            scales = torch.ones(timesteps) * guidance_scale
        if micro_conds.shape[0] == 1:
            micro_conds = micro_conds.repeat(B, 1).to(input_ids.device)
        use_cfg = guidance_scale > 0
        if use_cfg:
            unc_e = empty_embeds if negative_embeds is None else negative_embeds
            unc_c = empty_cond_embeds if negative_cond_embeds is None else negative_cond_embeds
            unc_e = unc_e.expand(B, -1, -1) if unc_e.shape[0] == 1 else unc_e
            unc_c = unc_c.expand(B, -1) if unc_c.shape[0] == 1 else unc_c
            encoder_hidden_states = torch.cat([encoder_hidden_states, unc_e])
            cond_embeds = torch.cat([cond_embeds, unc_c])
            micro_conds = torch.cat([micro_conds, micro_conds], dim=0)
        intermediate = []
        sampled = input_ids
        input_ids = input_ids.contiguous()
        if use_cuda_graph is None:
            import os

            use_cuda_graph = os.environ.get("MUSE_B200_CUDA_GRAPH", "1") != "0" and self._debug_stages is None
        for step in range(timesteps):
            model_in = torch.cat([input_ids] * 2) if use_cfg else input_ids
            if use_cuda_graph:
                padded = self._graphed_forward(model_in, encoder_hidden_states, cond_embeds, micro_conds)
            else:
                padded = self._forward_tokens(model_in, encoder_hidden_states, cond_embeds, micro_conds)
            # tensor shapes follow the ids (inpainting passes its own); ``seq_len`` only enters the mask_len schedule below,
            # as in the reference (:330-479)
            L = input_ids.shape[1]
            lg = padded.view(model_in.shape[0], L, -1)
            logits, logits_unc = (lg[:B], lg[B:]) if use_cfg else (lg, None)
            # generator consumed like the reference: multinomial(n=1) draws Exp(1) noise of the probabilities' shape,
            # mask_by_random_topk one uniform per token
            q_exp = torch.empty(B * L, K, dtype=torch.float32, device=lg.device).exponential_(1, generator=generator)
            u = torch.zeros(B, L, dtype=torch.float32, device=lg.device).uniform_(0, 1, generator=generator)
            ratio = 1.0 * (step + 1) / timesteps
            mask_len = int((seq_len * noise_schedule(torch.tensor(ratio))).floor())
            prev_ids = input_ids
            sampled, input_ids = ops.sample_step(logits, input_ids, q_exp, u, K, mask_id, mask_len, float(temps[step]),
                                                 logits_unc=logits_unc, guidance=float(scales[step]))
            if return_intermediate:
                # the reference collects the RAW multinomial sample, before the known tokens are re-inserted (:446-449).  The
                # fused kernel emits the re-inserted ids; at the already-decoded positions the raw draw is recomputed here
                # from the same logits and the same Exp(1) noise (argmax p / q) -- a debugging output, off the hot path
                x = logits[..., :K].float()
                if logits_unc is not None:
                    xu = logits_unc[..., :K].float()
                    x = xu + float(scales[step]) * (x - xu)
                raw = (torch.softmax(x, dim=-1) / q_exp.view(B, L, K)).argmax(dim=-1)
                intermediate.append(torch.where(prev_ids == mask_id, sampled, raw))
        return (sampled, intermediate) if return_intermediate else sampled
