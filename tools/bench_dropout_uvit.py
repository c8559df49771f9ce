#!/usr/bin/env python
"""Cost of dropout in MaskGiTUViT_v2: the eager train step at the reference defaults (603 M parameters: hidden 1024, 22
layers, 3 ResBlock + AttentionBlock2D pairs per stage at 768 channels; 256 tokens, 77 text states; AdamW) at dropout
0 / 0 against 0.1 / 0.1, and the six GELU + GRN kernels at the default width (C = 4 x 768 = 3072, 256 tokens) with and
without the dropout instantiation.  Variants alternate within one call: each round times every variant once.

  * step: CUDA events around --steps steps after a warm-up step, each step ending in a device synchronise; both models
    live through the whole run (same initial weights), so a round only switches which one steps.
  * device-time breakdown: one extra profiled step per variant (torch.profiler, CUDA activities) after the timed rounds,
    summed by kernel family, so the cost of each dropout site shows up where it is paid.
  * GRN kernels: device time per call from torch.profiler over --steps forward + backward calls.

The card name and power limit are printed with the numbers.

    python tools/bench_dropout_uvit.py [--rounds 3] [--steps 10] [--batch 16] [--json OUT.json]"""
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
from open_muse_b200 import MaskGiTUViT_v2, ops  # noqa: E402

GRN_KERNELS = ("grn_stats_kernel", "grn_finalize_kernel", "grn_apply_kernel", "grn_bwd_stats_kernel",
               "grn_bwd_finalize_kernel", "grn_bwd_apply_kernel")
FAMILIES = (("attention fwd", ("attn_fwd",)), ("attention bwd", ("attn_bwd",)), ("GRN", ("grn_",)),
            ("GLU", ("glu_",)), ("GEMM", ("gemm",)))


def make_model(p):
    torch.manual_seed(0)
    m = MaskGiTUViT_v2(hidden_dropout=p, attention_dropout=p).cuda().train()
    opt = torch.optim.AdamW(m.parameters(), lr=1e-4, weight_decay=0.01, fused=True)
    return m, opt


def make_batch(B):
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(0, 8192, (B, 256), generator=g)
    mask = torch.rand(B, 256, generator=g) < 0.5
    inp, lab = torch.where(mask, 8255, ids).cuda(), torch.where(mask, ids, -100).cuda()
    enc = torch.randn(B, 77, 768, generator=g).cuda()
    ce = torch.randn(B, 768, generator=g).cuda()
    mc = torch.tensor([[1024.0, 1024.0, 0.0, 0.0, 6.0]]).repeat(B, 1).cuda()
    return inp, enc, ce, mc, lab


def train_step(m, opt, batch):
    inp, enc, ce, mc, lab = batch
    with torch.autocast("cuda", dtype=torch.bfloat16):
        _, loss = m(inp, enc, ce, mc, labels=lab)
    loss.backward()
    opt.step()
    opt.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    return loss


def step_ms(m, opt, batch, steps):
    train_step(m, opt, batch)  # warm-up
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        train_step(m, opt, batch)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def _device_events(prof):
    return [ev for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA]


def step_breakdown(m, opt, batch):
    """device time (ms) of one train step by kernel family"""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        train_step(m, opt, batch)
    out = {name: 0.0 for name, _ in FAMILIES}
    out["other"] = out["total"] = 0.0
    for ev in _device_events(prof):
        t = ev.device_time / 1000.0
        out["total"] += t
        fam = next((name for name, keys in FAMILIES if any(k in ev.name for k in keys)), "other")
        out[fam] += t
    return out


def grn_us(drop, B, steps):
    """device time per call of each GELU + GRN kernel (us) for one forward + backward at the default width"""
    HW, C = 256, 3072
    gen = torch.Generator(device="cuda").manual_seed(2)
    x = torch.randn(B * HW, C, generator=gen, device="cuda").to(torch.bfloat16)
    dout = torch.randn(B * HW, C, generator=gen, device="cuda").to(torch.bfloat16)
    gamma = torch.randn(C, generator=gen, device="cuda") * 0.1
    beta = torch.randn(C, generator=gen, device="cuda") * 0.1
    dg, db = torch.zeros(C, device="cuda"), torch.zeros(C, device="cuda")
    seed = torch.tensor([5], dtype=torch.int64, device="cuda")

    def once():
        if drop:
            _, st, bits = ops.grn(x, gamma, beta, B, HW, save_stats=True, dropout=(0.1, seed, 0))
            ops.grn_bwd(x, dout, st, gamma, dg, db, B, HW, dropout=(0.1, bits))
        else:
            _, st = ops.grn(x, gamma, beta, B, HW, save_stats=True)
            ops.grn_bwd(x, dout, st, gamma, dg, db, B, HW)

    once()
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            once()
        torch.cuda.synchronize()
    tot = {kn: 0.0 for kn in GRN_KERNELS}
    for ev in _device_events(prof):
        for kn in GRN_KERNELS:
            if kn + "<" in ev.name or kn + "(" in ev.name:
                tot[kn] += ev.device_time
    return {kn: t / steps for kn, t in tot.items()}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--json")
    args = ap.parse_args()
    dev_card = card()
    print(f"card: {dev_card}", flush=True)
    batch = make_batch(args.batch)
    models = {p: make_model(p) for p in (0.0, 0.1)}
    n_params = sum(p.numel() for p in models[0.0][0].parameters())
    print(f"MaskGiTUViT_v2 reference defaults: {n_params / 1e6:.1f} M parameters, batch {args.batch}", flush=True)
    rows = {}
    for r in range(args.rounds):
        for p, (m, opt) in models.items():
            rows.setdefault(f"train step ms, dropout {p}/{p}", []).append(step_ms(m, opt, batch, args.steps))
        for drop in (False, True):
            for kn, us in grn_us(drop, args.batch, args.steps).items():
                rows.setdefault(f"{kn} us, {'dropout' if drop else 'no dropout'}", []).append(us)
        print(f"round {r + 1} of {args.rounds} done", flush=True)
    result = {"card": dev_card, "batch": args.batch, "params": n_params, "rounds": args.rounds, "steps": args.steps,
              "median": {}, "all": rows, "step_device_ms_by_family": {}}
    for name, xs in rows.items():
        result["median"][name] = statistics.median(xs)
        print(f"{name:48s} median {statistics.median(xs):9.3f}  (min {min(xs):.3f}, max {max(xs):.3f})")
    med = result["median"]
    pairs = [("train step ms, dropout 0.0/0.0", "train step ms, dropout 0.1/0.1")]
    pairs += [(f"{kn} us, no dropout", f"{kn} us, dropout") for kn in GRN_KERNELS]
    for a, b in pairs:
        print(f"{b}: {100 * (med[b] / med[a] - 1):+.1f} % vs no dropout")
    for p, (m, opt) in models.items():
        bd = step_breakdown(m, opt, batch)
        result["step_device_ms_by_family"][f"dropout {p}/{p}"] = bd
        print(f"device ms of one step, dropout {p}/{p}: " + ", ".join(f"{k} {v:.1f}" for k, v in bd.items()))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
