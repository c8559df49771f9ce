#!/usr/bin/env python
"""Cost of ``MaskGiTUViT_v2(use_fused_mlp=True)`` (FusedGeLUFeedForward: wo(gelu_tanh(wi_0 x)), no gate) against the GLU
FFN, at the class defaults (22 layers x 1024, 768 block channels) on 256 tokens, in three variants:

  * ``glu_2816``: GLUFeedForward, intermediate_size 2816 (the default);
  * ``fused_2816``: FusedGeLUFeedForward at the same width (2/3 of the FFN GEMM FLOPs);
  * ``fused_4096``: FusedGeLUFeedForward at 4096, about the GLU's parameter count.

For each, with the variants alternated within the call after a warm-up of each, medians over --rounds rounds:

  * ``ffn_fwd_us`` / ``ffn_bwd_us``: one layer's FFN kernels (wi GEMM, activation pass, wo GEMM; and their backward:
    wo wgrad + dgrad, activation backward, wi wgrad + dgrad) on batch x 256 rows, CUDA events over --iters calls;
  * ``act_fwd_us`` / ``act_bwd_us`` and their achieved bytes/s as a fraction of 3.35 TB/s (HBM3 data-sheet bandwidth): the
    bytes the pass must move (fwd: read pre, write out; bwd: read pre and dout, write dpre; the GLU's pre is [a | b], twice
    as wide, and so is its gradient), over its kernel time;
  * ``train_step_ms`` and ``peak_gib``: one eager training forward + backward of the whole model at --batch, and its
    max_memory_allocated.  The default batch is 64: at 16 the eager step is bound by the host's launches and its time
    varies by tens of percent between rounds on a shared machine, which hides the FFN's share;
  * ``generate2_steps_per_s``: decode steps per second of ``generate2`` with classifier-free guidance (CUDA graph), at
    batch 8 and 64, in bf16 and with ``set_gemm_precision("fp8")``.

The card name and power limit are read in the same call.

    python tools/bench_fused_mlp.py [--rounds 3] [--iters 50] [--steps 5] [--batch 64] [--json OUT.json]"""
import argparse
import gc
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, ROOT)
from bench_gemm import card  # noqa: E402
from open_muse_b200 import MaskGiTUViT_v2, ops  # noqa: E402

HBM_BPS = 3.35e12
VARIANTS = {"glu_2816": dict(use_fused_mlp=False, intermediate_size=2816),
            "fused_2816": dict(use_fused_mlp=True, intermediate_size=2816),
            "fused_4096": dict(use_fused_mlp=True, intermediate_size=4096)}
S = 256


def events(fn, iters):
    """mean ms of fn over iters calls, CUDA events, ending in a device synchronise"""
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def ffn_ops(glu, rows, H, I):
    """closures of one layer's FFN forward / backward and of its activation pass alone, on random operands"""
    g = torch.Generator(device="cuda").manual_seed(0)
    bf = dict(dtype=torch.bfloat16, device="cuda")
    y = torch.randn(rows, H, generator=g, **bf)
    wi = torch.randn((2 if glu else 1) * I, H, generator=g, **bf) * 0.02
    wo = torch.randn(H, I, generator=g, **bf) * 0.02
    df = torch.randn(rows, H, generator=g, **bf)
    gwi, gwo = torch.zeros(wi.shape, device="cuda"), torch.zeros(wo.shape, device="cuda")
    act_f = ops.glu_fwd if glu else ops.gelu_tanh_fwd
    act_b = ops.glu_bwd if glu else ops.gelu_tanh_bwd
    pre = ops.linear_fwd(y, wi)
    h = act_f(pre)
    dh = torch.randn(rows, I, generator=g, **bf)

    def fwd():
        ops.linear_fwd(act_f(ops.linear_fwd(y, wi)), wo)

    def bwd():
        ops.linear_wgrad(df, h, gwo)
        d = act_b(pre, ops.linear_dgrad(df, wo))
        ops.linear_wgrad(d, y, gwi)
        ops.linear_dgrad(d, wi)

    act_bytes_f = 2 * rows * ((2 if glu else 1) * I + I)
    act_bytes_b = 2 * rows * (2 * (2 if glu else 1) * I + I)
    return fwd, bwd, (lambda: act_f(pre)), (lambda: act_b(pre, dh)), act_bytes_f, act_bytes_b


def model_inputs(m, B, seed=1):
    c = m.config
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, c.codebook_size, (B, S), generator=g)
    mask = torch.rand(B, S, generator=g) < 0.5
    inp = torch.where(mask, c.mask_token_id, ids)
    lab = torch.where(mask, ids, -100)
    ehs = torch.randn(B, 77, c.encoder_hidden_size, generator=g)
    cond = torch.randn(B, c.cond_embed_dim, generator=g)
    micro = torch.tensor([[512.0, 512.0, 0.0, 0.0, 6.0]]).repeat(B, 1)
    return [t.cuda() for t in (inp, ehs, cond, micro)], lab.cuda()


def train_step(m, args, lab):
    m.zero_grad(set_to_none=True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        _, loss = m(*args, labels=lab)
    loss.backward()


def generate_rate(m, B, steps=12):
    c = m.config
    g = torch.Generator().manual_seed(2)
    kw = dict(encoder_hidden_states=torch.randn(B, 77, c.encoder_hidden_size, generator=g).cuda(),
              cond_embeds=torch.randn(B, c.cond_embed_dim, generator=g).cuda(),
              micro_conds=torch.tensor([[512.0, 512.0, 0.0, 0.0, 6.0]]).cuda(),
              empty_embeds=torch.zeros(1, 77, c.encoder_hidden_size).cuda(), empty_cond_embeds=torch.zeros(1, c.cond_embed_dim).cuda(),
              timesteps=steps, guidance_scale=5.0)
    with torch.no_grad():
        return steps / (events(lambda: m.generate2(**kw, generator=torch.Generator(device="cuda").manual_seed(3)), 2) / 1e3)


def measure(over, a):
    torch.manual_seed(0)
    with torch.device("cuda"):
        m = MaskGiTUViT_v2(**over)
    H, I, L = m.config.hidden_size, m.config.intermediate_size, m.config.num_hidden_layers
    out = dict(params_m=sum(p.numel() for p in m.parameters()) / 1e6, I=I)
    fwd, bwd, af, ab, bf_, bb = ffn_ops(not over["use_fused_mlp"], a.batch * S, H, I)
    out["ffn_fwd_us"] = 1e3 * events(fwd, a.iters)
    out["ffn_bwd_us"] = 1e3 * events(bwd, a.iters)
    out["act_fwd_us"], out["act_bwd_us"] = 1e3 * events(af, a.iters), 1e3 * events(ab, a.iters)
    out["act_fwd_of_peak"] = bf_ / (out["act_fwd_us"] * 1e-6) / HBM_BPS
    out["act_bwd_of_peak"] = bb / (out["act_bwd_us"] * 1e-6) / HBM_BPS
    out["ffn_layer_total_ms"] = L * (out["ffn_fwd_us"] + out["ffn_bwd_us"]) / 1e3
    m.train()
    args, lab = model_inputs(m, a.batch)
    train_step(m, args, lab)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    out["train_step_ms"] = events(lambda: train_step(m, args, lab), a.steps)
    out["peak_gib"] = torch.cuda.max_memory_allocated() / 2 ** 30
    m.zero_grad(set_to_none=True)
    m.eval()
    for prec in ("bf16", "fp8"):
        m.set_gemm_precision(prec)
        for B in (8, 64):
            out[f"generate2_{prec}_b{B}_steps_per_s"] = generate_rate(m, B)
    del m, args, lab
    gc.collect()
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--json", default=os.path.join(os.path.dirname(ROOT), "profiles", "h100_bench_fused_mlp.json"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fused_mlp needs a CUDA device")
    runs = {k: [] for k in VARIANTS}
    for r in range(a.rounds + 1):  # round 0 warms every shape up and is dropped
        for name, over in VARIANTS.items():
            res = measure(over, a)
            if r:
                runs[name].append(res)
            print(name, "round", r, json.dumps({k: round(v, 3) for k, v in res.items()}), flush=True)
    med = {name: {k: statistics.median(x[k] for x in rs) for k in rs[0]} for name, rs in runs.items()}
    result = dict(card=card(), batch=a.batch, tokens=S, rounds=a.rounds, iters=a.iters, steps=a.steps, median=med, runs=runs)
    print(json.dumps(result["median"], indent=1))
    with open(a.json, "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
