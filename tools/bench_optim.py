#!/usr/bin/env python
"""One optimizer step, timed: the reference Lion (training/optimizer.py, from the oracle snapshot), FusedLion without EMA,
FusedLion with EMA and model=, torch.optim.AdamW(fused=True), FusedAdamW(model=) and FusedAdamW8bit(model=) each without
and with EMA, at the v1 base-256 size (36 M parameters) and the MaskGiTUViT_v2 default (603 M).  Then one eager
U-ViT train step (forward, backward, step) with FusedAdamW(model=) against torch AdamW(fused=True), whose step is followed
by the full operand rebuild of the next forward, and FusedAdamW8bit(model=); and the peak memory of that train step after a
warm-up step with FusedAdamW(model=) and FusedAdamW8bit(model=), each model and optimizer alone on the card.

  * CUDA events around --steps steps after --warmup steps; variants alternate within each of --rounds rounds, and the
    median over rounds is reported.
  * GB/s from the bytes each algorithm needs per parameter: Lion reads p, g, m and writes p, m (20 B); + EMA shadow read
    and write + bf16 copy (30 B); AdamW 28 B, + bf16 copy 30 B, + EMA 38 B; AdamW with 8-bit moments reads p, g and two
    codes and writes p, two codes and the bf16 copy (18 B), + EMA shadow read and write (26 B).  Share of the H100 SXM
    data-sheet 3.35 TB/s.  The optimizer-state bytes of each variant are reported beside it.
  * The card's name and power limit are read in the same run.

    python tools/bench_optim.py [--rounds 3] [--steps 10] [--warmup 2] [--batch 16] [--json OUT.json]"""
import argparse
import gc
import importlib.util
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_gemm import card  # noqa: E402
from oracle import ref_snapshot  # noqa: E402
from open_muse_b200 import EMAModel, FusedAdamW, FusedAdamW8bit, FusedLion, MaskGitTransformer, MaskGiTUViT_v2  # noqa: E402,E501

PEAK_BW = 3.35e12  # H100 SXM data sheet, HBM3
BASE_CFG = dict(vocab_size=2025, max_position_embeddings=257, hidden_size=512, num_hidden_layers=8, num_attention_heads=8,
                intermediate_size=2048, codebook_size=1024, num_vq_tokens=256, num_classes=1000, hidden_dropout=0.0,
                attention_dropout=0.0)


def ref_lion():
    path = os.path.join(ref_snapshot.DEST, "training", "optimizer.py")
    spec = importlib.util.spec_from_file_location("_ref_training_optimizer", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.Lion


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def state_bytes(opt):
    """bytes of every tensor in the optimizer's per-parameter state (a group's shared step counter counted once)"""
    seen = {}
    for st in opt.state.values():
        for t in st.values():
            if torch.is_tensor(t):
                seen[t.data_ptr()] = t.numel() * t.element_size()
    return sum(seen.values())


def optimizer_steps(name, model, args):
    params = list(model.parameters())
    n = sum(p.numel() for p in params)
    g = torch.Generator(device="cuda").manual_seed(0)
    for p in params:
        p.grad = torch.randn(p.shape, generator=g, device="cuda") * 1e-3
    kw = dict(lr=1e-4, weight_decay=0.01)
    variants = {  # name -> (optimizer, bytes per parameter)
        "reference Lion": (ref_lion()(params, **kw), 20),
        "FusedLion": (FusedLion(params, **kw), 20),
        "FusedLion ema+model": (FusedLion(params, ema=EMAModel(params, decay=0.9999), model=model, **kw), 30),
        "torch AdamW fused": (torch.optim.AdamW(params, fused=True, **kw), 28),
        "FusedAdamW model": (FusedAdamW(params, model=model, **kw), 30),
        "FusedAdamW ema+model": (FusedAdamW(params, ema=EMAModel(params, decay=0.9999), model=model, **kw), 38),
        "FusedAdamW8bit model": (FusedAdamW8bit(params, model=model, **kw), 18),
        "FusedAdamW8bit ema+model": (FusedAdamW8bit(params, ema=EMAModel(params, decay=0.9999), model=model, **kw), 26),
    }
    model._packed.refresh()
    ms = {k: [] for k in variants}
    for _ in range(args.rounds):
        for k, (opt, _) in variants.items():
            ms[k].append(timed(opt.step, args.steps, args.warmup))
    out = []
    for k, (_, bpp) in variants.items():
        t = statistics.median(ms[k])
        gbs = bpp * n / (t * 1e-3) / 1e9
        out.append(dict(model=name, params=n, variant=k, ms=round(t, 4), ms_rounds=[round(x, 4) for x in ms[k]],
                        bytes_per_param=bpp, GBps=round(gbs, 1), share_of_3_35_TBps=round(gbs * 1e9 / PEAK_BW, 3),
                        state_bytes=state_bytes(variants[k][0])))
    del variants
    for p in params:
        p.grad = None
    free()
    return out


def uvit_batch(B):
    gen = torch.Generator().manual_seed(1)
    ids = torch.randint(0, 8192, (B, 256), generator=gen)
    mask = torch.rand(B, 256, generator=gen) < 0.5
    batch = (torch.where(mask, 8255, ids).cuda(), torch.randn(B, 77, 768, generator=gen).cuda(),
             torch.randn(B, 768, generator=gen).cuda(), torch.tensor([[1024.0, 1024.0, 0.0, 0.0, 6.0]]).repeat(B, 1).cuda())
    return batch, torch.where(mask, ids, -100).cuda()


def train_step(m, opt, batch, labels):
    with torch.autocast("cuda", dtype=torch.bfloat16):
        _, loss = m(*batch, labels=labels)
    loss.backward()
    opt.step()
    opt.zero_grad(set_to_none=True)


def uvit_train_steps(args):
    torch.manual_seed(0)
    names = ("torch AdamW fused + operand rebuild", "FusedAdamW model", "FusedAdamW8bit model")
    models = {k: MaskGiTUViT_v2().cuda().train() for k in names}
    a, b, c = models.values()
    b.load_state_dict(a.state_dict())
    c.load_state_dict(a.state_dict())
    opts = {"torch AdamW fused + operand rebuild": torch.optim.AdamW(a.parameters(), lr=1e-4, weight_decay=0.01, fused=True),
            "FusedAdamW model": FusedAdamW(b.parameters(), lr=1e-4, weight_decay=0.01, model=b),
            "FusedAdamW8bit model": FusedAdamW8bit(c.parameters(), lr=1e-4, weight_decay=0.01, model=c)}
    batch, labels = uvit_batch(args.batch)

    def step(m, opt):
        train_step(m, opt, batch, labels)

    ms = {k: [] for k in models}
    for _ in range(args.rounds):
        for k in models:
            ms[k].append(timed(lambda: step(models[k], opts[k]), args.steps, args.warmup))
    return [dict(model="MaskGiTUViT_v2 default", batch=args.batch, variant=k, step_ms=round(statistics.median(v), 3),
                 ms_rounds=[round(x, 3) for x in v]) for k, v in ms.items()]


def free():
    """the fused optimizers and the models they pack operands for hold reference cycles (model._packed.model is the
    model), so `del` alone leaves their tensors allocated until the cyclic collector runs"""
    gc.collect()
    torch.cuda.empty_cache()


def uvit_train_memory(args):
    """torch.cuda.max_memory_allocated over two eager train steps of the U-ViT default after one warm-up step (which
    creates the optimizer state and the operand cache), each optimizer with its own model alone on the card.  Memory is
    reported above what was allocated before the model was built, and the run stops if a variant leaves memory behind."""
    out = []
    batch, labels = uvit_batch(args.batch)
    free()
    base = torch.cuda.memory_allocated()
    for name, cls in (("FusedAdamW model", FusedAdamW), ("FusedAdamW8bit model", FusedAdamW8bit)):
        torch.manual_seed(0)
        m = MaskGiTUViT_v2().cuda().train()
        opt = cls(m.parameters(), lr=1e-4, weight_decay=0.01, model=m)
        train_step(m, opt, batch, labels)
        torch.cuda.synchronize()
        resident = torch.cuda.memory_allocated() - base
        torch.cuda.reset_peak_memory_stats()
        for _ in range(2):
            train_step(m, opt, batch, labels)
        torch.cuda.synchronize()
        out.append(dict(model="MaskGiTUViT_v2 default", batch=args.batch, variant=name,
                        max_memory_allocated_GB=round((torch.cuda.max_memory_allocated() - base) / 1e9, 3),
                        resident_between_steps_GB=round(resident / 1e9, 3), state_bytes=state_bytes(opt)))
        del m, opt
        free()
        left = torch.cuda.memory_allocated() - base
        if left > 2 ** 20:
            raise SystemExit(f"{name}: {left} bytes still allocated after the variant was released")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_optim.py times the GPU: no CUDA device")
    res = dict(card=card(), rounds=args.rounds, steps=args.steps, warmup=args.warmup, optimizer_step=[])
    torch.manual_seed(0)
    res["optimizer_step"] += optimizer_steps("MaskGitTransformer base-256", MaskGitTransformer(**BASE_CFG).cuda(), args)
    torch.manual_seed(0)
    uvit = MaskGiTUViT_v2().cuda()
    res["optimizer_step"] += optimizer_steps("MaskGiTUViT_v2 default", uvit, args)
    del uvit
    free()
    res["uvit_train_step"] = uvit_train_steps(args)
    free()
    res["uvit_train_memory"] = uvit_train_memory(args)
    for r in res["optimizer_step"] + res["uvit_train_step"] + res["uvit_train_memory"]:
        print(json.dumps(r))
    line = json.dumps(res)
    print(line)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
