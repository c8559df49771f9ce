#!/usr/bin/env python
"""Cost of dropout: the CUDA-graphed base-256 train step (B=256, S=257, H=512, I=2048, 8 layers, AdamW) at dropout 0 / 0
against 0.1 / 0.1, and the three attention kernels at that shape (B=256, 8 heads, S=257, head_dim 64) with and without
the DROP instantiation.  Variants alternate within one call: each round times every variant once.  To keep one step's
memory at a time, a train-step variant is built (model, optimizer, captured graph), timed and released within its round.
Attention kernels are timed per kernel from torch.profiler device events.  The card name and power limit are printed
with the numbers.

    python tools/bench_dropout.py [--rounds 3] [--steps 10] [--batch 256] [--json OUT.json]"""
import argparse
import gc
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_gemm import card  # noqa: E402
from open_muse_b200 import MaskGitTransformer, ops  # noqa: E402
from open_muse_b200.graphs import GraphedStep  # noqa: E402

CFG = dict(vocab_size=2025, max_position_embeddings=257, hidden_size=512, num_hidden_layers=8, num_attention_heads=8,
           intermediate_size=2048, codebook_size=1024, num_vq_tokens=256, num_classes=1000)
KERNELS = ("attn_fwd_tc_kernel", "attn_bwd_dq_tc_kernel", "attn_bwd_dkdv_tc_kernel")


def step_ms(p, B, steps):
    """builds the graphed train step at dropout p / p, returns ms per replay, releases everything"""
    torch.manual_seed(0)
    m = MaskGitTransformer(**CFG, hidden_dropout=p, attention_dropout=p).cuda().train()
    opt = torch.optim.AdamW(m.parameters(), lr=1e-4, weight_decay=0.01, fused=True, capturable=True)
    g = torch.Generator().manual_seed(1)
    tokens = torch.randint(0, 1024, (B, 256), generator=g)
    cls = torch.randint(0, 1000, (B,), generator=g)
    mask = torch.rand(B, 256, generator=g) < 0.5
    inp = torch.cat([(cls + 1024)[:, None], torch.where(mask, 2024, tokens)], 1).cuda()
    lab = torch.cat([torch.full((B, 1), -100), torch.where(mask, tokens, -100)], 1).cuda()

    def step(i, l_):
        with torch.autocast("cuda", dtype=torch.bfloat16):
            _, loss = m(i, labels=l_)
        loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
        return loss

    graphed = GraphedStep(step, (inp, lab), warmup=2)
    graphed(inp, lab)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        graphed(inp, lab)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    del graphed, opt, m
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return ms


def attention_us(drop, B, steps):
    """device time per call of each attention kernel (us) for one forward + backward at the bench shape"""
    nh, S, H = 8, 257, 512
    gen = torch.Generator(device="cuda").manual_seed(2)
    qkv = torch.randn(B * S, 3 * H, generator=gen, device="cuda").to(torch.bfloat16)
    q, k, v = qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:]
    do = torch.randn(B * S, H, generator=gen, device="cuda").to(torch.bfloat16)
    dqkv = torch.empty_like(qkv)
    seed = torch.tensor([5], dtype=torch.int64, device="cuda")

    def once():
        out = ops.attn_fwd(q, k, v, B, nh, S, S, 0.125, **({"dropout": (0.1, seed, 1)} if drop else {}))
        ops.attn_bwd(q, k, v, out[0], do, out[1], dqkv[:, :H], dqkv[:, H:2 * H], dqkv[:, 2 * H:], B, nh, S, S, 0.125,
                     **({"dropout": (0.1, out[2])} if drop else {}))

    once()
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            once()
        torch.cuda.synchronize()
    tot = {kn: 0.0 for kn in KERNELS}
    for ev in prof.events():
        for kn in KERNELS:
            if kn in ev.name and ev.device_type == torch.autograd.DeviceType.CUDA:
                tot[kn] += ev.device_time
    return {kn: t / steps for kn, t in tot.items()}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--json")
    args = ap.parse_args()
    dev_card = card()
    print(f"card: {dev_card}", flush=True)
    rows = {}
    for r in range(args.rounds):
        for p in (0.0, 0.1):
            rows.setdefault(f"train step ms, dropout {p}/{p}", []).append(step_ms(p, args.batch, args.steps))
        for drop in (False, True):
            for kn, us in attention_us(drop, args.batch, args.steps).items():
                rows.setdefault(f"{kn} us, {'DROP' if drop else 'no dropout'}", []).append(us)
        print(f"round {r + 1} of {args.rounds} done", flush=True)
    result = {"card": dev_card, "batch": args.batch, "rounds": args.rounds, "steps": args.steps, "median": {}, "all": rows}
    for name, xs in rows.items():
        result["median"][name] = statistics.median(xs)
        print(f"{name:48s} median {statistics.median(xs):9.3f}  (min {min(xs):.3f}, max {max(xs):.3f})")
    med = result["median"]
    pairs = [("train step ms, dropout 0.0/0.0", "train step ms, dropout 0.1/0.1")]
    pairs += [(f"{kn} us, no dropout", f"{kn} us, DROP") for kn in KERNELS]
    for a, b in pairs:
        print(f"{b}: {100 * (med[b] / med[a] - 1):+.1f} % vs no dropout")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
