#!/usr/bin/env python
"""Cost and memory of gradient checkpointing (``enable_gradient_checkpointing()``) on the reference's training workloads:

  * MaskGitTransformer at configs/imagenet.yaml widths (24 x 768, I 3072, 257 tokens), batch 192;
  * MaskGitTransformer at configs/cc12m.yaml widths (24 x 1024, I 4096, RMSNorm, cross-attention) on 77 x 768 text
    states, batch 64;
  * MaskGiTUViT_v2 of configs/research_run_512.yaml at 512 px (1024 tokens), batch 32;
  * the same with force_down_up_sample (research_run_512_with_downsample.yaml), batch 64.

The model widths come from tests/golden/configs.json (the parsed reference configs).  For each workload one model (same
weights) trains with FusedAdamW(model=); checkpointing is switched off and on between steps, alternating within the call
after a warm-up step of each:

  * step ms: CUDA events around --steps train steps, each ending in a device synchronise; median over --rounds rounds;
  * peak max_memory_allocated of a train step;
  * held: memory_allocated after the forward minus before (what lives until the backward);
  * activation bytes per sample: the slope of ``held`` between the batch and half of it;
  * the largest batch that slope of the PEAK predicts for the card's memory (computed, never tried);
  * the no-grad forward time of the same batch: the recompute is one forward without its last GEMMs, so the step time
    checkpointing adds should stay below it.

The card name and power limit are read in the same call.

    python tools/bench_recompute.py [--rounds 3] [--steps 3] [--only NAME] [--json OUT.json]"""
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
from open_muse_b200 import FusedAdamW, MaskGitTransformer, MaskGiTUViT_v2  # noqa: E402

CONFIGS = json.load(open(os.path.join(ROOT, "tests", "golden", "configs.json")))


def _cfg(name):
    return {k: v for k, v in CONFIGS[name]["transformer"].items()}


def imagenet(B):
    c = _cfg("imagenet.yaml")
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(0, 1024, (B, 256), generator=g)
    mask = torch.rand(B, 256, generator=g) < 0.5
    cls = torch.randint(0, 1000, (B, 1), generator=g) + 1024
    inp = torch.cat([cls, torch.where(mask, c["vocab_size"] - 1, ids)], 1)
    lab = torch.cat([torch.full((B, 1), -100), torch.where(mask, ids, -100)], 1)
    return MaskGitTransformer, c, dict(input_ids=inp.cuda(), labels=lab.cuda())


def cc12m(B):
    c = dict(_cfg("cc12m.yaml"), encoder_hidden_size=768)  # 77 x 768 CLIP text states, no projection
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(0, 8192, (B, 256), generator=g)
    mask = torch.rand(B, 256, generator=g) < 0.5
    return MaskGitTransformer, c, dict(input_ids=torch.where(mask, c["vocab_size"] - 1, ids).cuda(),
                                       labels=torch.where(mask, ids, -100).cuda(),
                                       encoder_hidden_states=torch.randn(B, 77, 768, generator=g).cuda())


def _uvit(name, B):
    c = _cfg(name)
    S = 1024  # 512 px through the f16 VQGAN: 32 x 32 tokens
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(0, 8192, (B, S), generator=g)
    mask = torch.rand(B, S, generator=g) < 0.5
    mc = torch.tensor([[512.0, 512.0, 0.0, 0.0, 6.0]]).repeat(B, 1)
    return MaskGiTUViT_v2, c, dict(input_ids=torch.where(mask, c["vocab_size"] - 1, ids).cuda(),
                                   encoder_hidden_states=torch.randn(B, 77, 768, generator=g).cuda(),
                                   cond_embeds=torch.randn(B, 768, generator=g).cuda(), micro_conds=mc.cuda(),
                                   labels=torch.where(mask, ids, -100).cuda())


WORKLOADS = {
    "v1 imagenet.yaml": (imagenet, 192),
    "v1 cc12m.yaml t2i": (cc12m, 64),
    "uvit research_run_512.yaml": (lambda B: _uvit("research_run_512.yaml", B), 32),
    "uvit research_run_512_with_downsample.yaml": (lambda B: _uvit("research_run_512_with_downsample.yaml", B), 64),
}


def set_ckpt(m, on):
    (m.enable_gradient_checkpointing if on else m.disable_gradient_checkpointing)()


def train_step(m, opt, fwd):
    with torch.autocast("cuda", dtype=torch.bfloat16):
        _, loss = m(**fwd)
    loss.backward()
    opt.step()
    opt.zero_grad(set_to_none=True)
    torch.cuda.synchronize()


def step_ms(m, opt, fwd, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        train_step(m, opt, fwd)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def memory(m, opt, fwd):
    """(held after the forward, peak of the step) in bytes"""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        _, loss = m(**fwd)
    torch.cuda.synchronize()
    held = torch.cuda.memory_allocated() - base
    loss.backward()
    opt.step()
    opt.zero_grad(set_to_none=True)
    del loss
    torch.cuda.synchronize()
    return held, torch.cuda.max_memory_allocated()


def nograd_forward_ms(m, fwd, steps):
    args = {k: v for k, v in fwd.items() if k != "labels"}
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        m(**args)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            m(**args)
        e1.record()
        torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def run(name, rounds, steps, total_mem):
    make, B = WORKLOADS[name]
    cls, cfg, fwd = make(B)
    _, _, half = make(B // 2)
    torch.manual_seed(0)
    with torch.device("cuda"):
        m = cls(**cfg)
    m.train()
    opt = FusedAdamW(m.parameters(), lr=1e-4, weight_decay=0.01, model=m)
    out = {"batch": B, "params": sum(p.numel() for p in m.parameters())}
    for on in (False, True):  # warm-up, then the memory of each variant at both batch sizes
        set_ckpt(m, on)
        train_step(m, opt, fwd)
        held_b, peak_b = memory(m, opt, fwd)
        held_h, peak_h = memory(m, opt, half)
        slope = (held_b - held_h) / (B - B // 2)
        peak_slope = (peak_b - peak_h) / (B - B // 2)
        key = "on" if on else "off"
        out[key] = {"held_after_forward_GiB": held_b / 2 ** 30, "peak_GiB": peak_b / 2 ** 30,
                    "activation_MiB_per_sample": slope / 2 ** 20, "peak_MiB_per_sample": peak_slope / 2 ** 20,
                    "predicted_max_batch": int((total_mem - (peak_b - peak_slope * B)) // peak_slope)}
    times = {False: [], True: []}
    for _ in range(rounds):
        for on in (False, True):
            set_ckpt(m, on)
            times[on].append(step_ms(m, opt, fwd, steps))
    for on in (False, True):
        out["on" if on else "off"]["step_ms"] = statistics.median(times[on])
        out["on" if on else "off"]["step_ms_all"] = times[on]
    set_ckpt(m, False)
    out["nograd_forward_ms"] = nograd_forward_ms(m.train(), fwd, steps)
    out["overhead_ms"] = out["on"]["step_ms"] - out["off"]["step_ms"]
    del m, opt
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--only", choices=list(WORKLOADS))
    ap.add_argument("--json")
    args = ap.parse_args()
    dev_card = card()
    total = torch.cuda.get_device_properties(0).total_memory
    print(f"card: {dev_card}, {total / 2 ** 30:.1f} GiB", flush=True)
    result = {"card": dev_card, "total_memory_GiB": total / 2 ** 30, "rounds": args.rounds, "steps": args.steps,
              "workloads": {}}
    for name in ([args.only] if args.only else WORKLOADS):
        r = run(name, args.rounds, args.steps, total)
        result["workloads"][name] = r
        print(f"{name} (batch {r['batch']}, {r['params'] / 1e6:.0f} M parameters): no-grad forward "
              f"{r['nograd_forward_ms']:.1f} ms, checkpointing adds {r['overhead_ms']:.1f} ms", flush=True)
        for k in ("off", "on"):
            v = r[k]
            print(f"  {k:3s}: step {v['step_ms']:8.1f} ms, peak {v['peak_GiB']:6.2f} GiB, held {v['held_after_forward_GiB']:6.2f}"
                  f" GiB, {v['activation_MiB_per_sample']:8.1f} MiB/sample, predicted max batch {v['predicted_max_batch']}",
                  flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
