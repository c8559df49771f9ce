#!/usr/bin/env python
"""Attention at equal hidden width, 16 heads of 64 against 8 heads of 128 (hidden 1024): the forward, dQ and dK/dV
kernels timed per kernel from torch.profiler device events, for self-attention over 256 tokens and cross-attention from
256 tokens to 77 text states, batch 32, with and without dropout on the probabilities.  Widths alternate within each
round.  TFLOP/s counts the products each kernel must form, 2 B nh Sq Skv hd FLOPs each: the forward Q K^T and P V
(2 products), dQ Q K^T, dO V^T and dS K (3; the kernel forms the two score products in both of its sweeps, which is not
counted), dK/dV K Q^T, V dO^T, P^T dO and dS^T Q (4).  The fraction is of the H100 SXM data-sheet 989 dense BF16 TFLOP/s.
The card name and power limit are printed with the numbers.

    python tools/bench_attention_heads.py [--rounds 3] [--steps 20] [--batch 32] [--json OUT.json]"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_gemm import card  # noqa: E402
from open_muse_b200 import ops  # noqa: E402

HIDDEN, S, TEXT = 1024, 256, 77
PEAK = 989e12
KERNELS = {"attn_fwd_tc_kernel": 2, "attn_bwd_dq_tc_kernel": 3, "attn_bwd_dkdv_tc_kernel": 4}  # products per kernel


def kernel_us(B, hd, Skv, drop, steps):
    """device time per call (us) of each attention kernel for one forward + backward"""
    nh = HIDDEN // hd
    scale = hd ** -0.5
    gen = torch.Generator(device="cuda").manual_seed(2)
    if Skv == S:  # q / k / v: column slices of one [T, 3H] projection
        qkv = torch.randn(B * S, 3 * HIDDEN, generator=gen, device="cuda").to(torch.bfloat16)
        q, k, v = qkv[:, :HIDDEN], qkv[:, HIDDEN:2 * HIDDEN], qkv[:, 2 * HIDDEN:]
    else:  # cross-attention: q of its own, k / v slices of one [T_text, 2H] projection
        q = torch.randn(B * S, HIDDEN, generator=gen, device="cuda").to(torch.bfloat16)
        kv = torch.randn(B * Skv, 2 * HIDDEN, generator=gen, device="cuda").to(torch.bfloat16)
        k, v = kv[:, :HIDDEN], kv[:, HIDDEN:]
    do = torch.randn(B * S, HIDDEN, generator=gen, device="cuda").to(torch.bfloat16)
    dq = torch.empty(B * S, HIDDEN, dtype=torch.bfloat16, device="cuda")
    dk = torch.empty(B * Skv, HIDDEN, dtype=torch.bfloat16, device="cuda")
    dv = torch.empty_like(dk)
    seed = torch.tensor([5], dtype=torch.int64, device="cuda")

    def once():
        out = ops.attn_fwd(q, k, v, B, nh, S, Skv, scale, head_dim=hd, **({"dropout": (0.1, seed, 1)} if drop else {}))
        ops.attn_bwd(q, k, v, out[0], do, out[1], dq, dk, dv, B, nh, S, Skv, scale, head_dim=hd,
                     **({"dropout": (0.1, out[2])} if drop else {}))

    for _ in range(3):
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
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_attention_heads.py needs a GPU: nothing is timed without one")
    dev_card = card()
    print(f"card: {dev_card}", flush=True)
    B = args.batch
    variants = [(hd, Skv, drop) for Skv in (S, TEXT) for drop in (False, True) for hd in (64, 128)]
    samples = {}
    for r in range(args.rounds):
        for hd, Skv, drop in variants:
            for kn, us in kernel_us(B, hd, Skv, drop, args.steps).items():
                samples.setdefault((hd, Skv, drop, kn), []).append(us)
        print(f"round {r + 1} done", flush=True)
    rows = []
    for (hd, Skv, drop, kn), us in samples.items():
        med = statistics.median(us)
        flops = KERNELS[kn] * 2.0 * B * (HIDDEN // hd) * S * Skv * hd
        tflops = flops / (med * 1e-6) / 1e12
        rows.append(dict(kernel=kn, head_dim=hd, heads=HIDDEN // hd, Sq=S, Skv=Skv, dropout=drop, batch=B,
                         us_median=round(med, 2), us_rounds=[round(x, 2) for x in us], tflops=round(tflops, 1),
                         fraction_of_989=round(tflops * 1e12 / PEAK, 3)))
        print(f"{kn:26s} hd {hd:3d} x {HIDDEN // hd:2d} heads, Skv {Skv:3d}, {'DROP' if drop else 'no dropout':10s}: "
              f"{med:8.1f} us  {tflops:6.1f} TFLOP/s  {tflops * 1e12 / PEAK:.3f} of 989", flush=True)
    if args.json:
        with open(args.json, "w") as f:
            # the settings that shape the numbers, not where the file was written
            command = f"python tools/bench_attention_heads.py --rounds {args.rounds} --steps {args.steps} --batch {B}"
            json.dump(dict(card=dev_card, command=command, hidden=HIDDEN, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
