#!/usr/bin/env python
"""FP8 inference of MaskGiTUViT_v2 (set_gemm_precision("fp8")) against the bf16 default, in one run on one card.

  * generate2 steps per second at the class defaults (hidden 1024, 22 layers, blocks 768 wide, 3 res blocks) with
    classifier-free guidance, batch 1 / 8 / 64: 256 px (16 x 16 tokens) and 512 px with force_down_up_sample
    (32 x 32 tokens, the stages at 16 x 16).  CUDA graphs on (the default), --timesteps steps per call.  Each precision
    has its own copy of the model, so the timed calls replay the graphs and operands an untimed round built; the two
    precisions alternate within each of --rounds rounds and the median is reported.
  * PipelineMuse latency at bench.py's t2i_pipeline_latency settings (12 steps, CFG, taming decode and PIL; the text
    encoder's states precomputed), batch 1 and 8, both resolutions, timed the same way.
  * Each FP8 GEMM site at the class defaults, batch 8 with CFG (4096 token rows), against the same product in bf16: CUDA
    events over --iters launches, TFLOP/s from 2 M N K, and the share of the data-sheet dense peaks (1,979 TFLOP/s FP8,
    989 bf16, H100 SXM at up to 700 W).
  * The card's name and power limit are read in the same run.

    python tools/bench_fp8.py [--rounds 3] [--timesteps 12] [--iters 50] [--json OUT.json]"""
import argparse
import copy
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_gemm import card, timeit  # noqa: E402
from open_muse_b200 import MaskGiTUViT_v2, ops  # noqa: E402
from open_muse_b200.modeling_taming_vqgan import VQGANModel  # noqa: E402

PEAK_FP8, PEAK_BF16 = 1979e12, 989e12  # H100 SXM data sheet, dense
DEV = "cuda"

# (site, N, K) of the FP8 GEMMs at the class defaults; M = tokens
SITES = [("layer [q;k;v]", 3072, 1024), ("layer cross-attention q", 1024, 1024), ("layer [wi_0;wi_1]", 5632, 1024),
         ("layer wo", 1024, 2816), ("ResBlock channelwise[0]", 3072, 768), ("AttentionBlock2D q", 768, 768)]


def gemm_sites(M, iters):
    out = []
    g = torch.Generator(device=DEV).manual_seed(0)
    for name, N, K in SITES:
        x = torch.randn(M, K, device=DEV, generator=g).to(torch.bfloat16)
        w = (torch.randn(N, K, device=DEV, generator=g) * 0.02).to(torch.bfloat16)
        x8, w8 = ops.quantize_rows_e4m3(x), ops.quantize_rows_e4m3(w)
        t8 = timeit(lambda: ops.linear_fwd(x8, w8), iters, 5)
        tb = timeit(lambda: ops.linear_fwd(x, w), iters, 5)
        fl = 2.0 * M * N * K
        out.append(dict(site=name, M=M, N=N, K=K, fp8_us=t8 * 1e3, bf16_us=tb * 1e3, fp8_tflops=fl / t8 / 1e9,
                        bf16_tflops=fl / tb / 1e9, fp8_peak_frac=fl / t8 / 1e-3 / PEAK_FP8,
                        bf16_peak_frac=fl / tb / 1e-3 / PEAK_BF16, speedup=tb / t8))
        print(f"{name:26s} M={M} N={N} K={K}: fp8 {t8 * 1e3:8.1f} us ({fl / t8 / 1e9:6.1f} TFLOP/s) | bf16 {tb * 1e3:8.1f} us "
              f"({fl / tb / 1e9:6.1f} TFLOP/s) | x{tb / t8:.2f}", flush=True)
    return out


def _alternate(fns, rounds):
    """{name: median ms} of the calls fns[name]() (each ending in a device synchronise), the names alternating within
    each of `rounds` rounds after one untimed round.  Each precision has its own model, so no call rebuilds an operand
    cache or recaptures a CUDA graph: the timed calls replay what the untimed round built (checked by the caller)."""
    t = {k: [] for k in fns}
    for r in range(rounds + 1):
        for k, fn in fns.items():
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            if r:
                t[k].append(e0.elapsed_time(e1))
    return {k: statistics.median(v) for k, v in t.items()}


def generate_rates(models, res, batches, timesteps, rounds):
    c = models["bf16"].config
    S = (res // 16) ** 2
    rows = []
    for B in batches:
        g = torch.Generator().manual_seed(B)
        kw = dict(encoder_hidden_states=torch.randn(B, 77, c.encoder_hidden_size, generator=g).to(DEV),
                  cond_embeds=torch.randn(B, c.cond_embed_dim, generator=g).to(DEV),
                  micro_conds=torch.tensor([[res, res, 0.0, 0.0, 6.0]]).to(DEV),
                  empty_embeds=torch.randn(1, 77, c.encoder_hidden_size, generator=g).to(DEV),
                  empty_cond_embeds=torch.randn(1, c.cond_embed_dim, generator=g).to(DEV),
                  guidance_scale=8.0, timesteps=timesteps, seq_len=S)
        graphs = {}

        def call(prec):
            m = models[prec]
            m.generate2(**kw, generator=torch.Generator(device=DEV).manual_seed(1))
            if prec in graphs:  # the timed calls replay the graph the untimed round captured
                assert m._graph is graphs[prec], "a timed generate2 call recaptured its CUDA graph"
            graphs[prec] = m._graph

        ms = _alternate({p: (lambda p=p: call(p)) for p in models}, rounds)
        mb, mf = ms["bf16"], ms["fp8"]
        row = dict(res=res, batch=B, tokens=S, timesteps=timesteps, bf16_ms=mb, fp8_ms=mf,
                   bf16_steps_per_s=timesteps / mb * 1e3, fp8_steps_per_s=timesteps / mf * 1e3, speedup=mb / mf)
        print(f"generate2 {res} px batch {B:3d} (CFG): bf16 {row['bf16_steps_per_s']:7.2f} steps/s | fp8 "
              f"{row['fp8_steps_per_s']:7.2f} steps/s | x{mb / mf:.3f}", flush=True)
        rows.append(row)
    return rows


def pipeline_latency(models, vae, res, rounds):
    """PipelineMuse at bench.py's t2i_pipeline_latency settings (12 steps, CFG, precomputed text states, taming decode,
    PIL), batch 1 and 8"""
    from open_muse_b200 import PipelineMuse

    g = torch.Generator(device=DEV).manual_seed(3)
    emb = lambda *s: torch.randn(*s, device=DEV, generator=g)  # noqa: E731
    kw = dict(prompt_embeds=emb(1, 77, 768), pooled_embeds=emb(1, 768), negative_prompt_embeds=emb(1, 77, 768),
              negative_pooled_embeds=emb(1, 768), timesteps=12, transformer_seq_len=(res // 16) ** 2)
    pipes = {p: PipelineMuse(vae=vae, transformer=m, is_class_conditioned=False).to(DEV) for p, m in models.items()}
    rows = []
    for bs in (1, 8):
        ms = _alternate({p: (lambda p=p: pipes[p](**kw, num_images_per_prompt=bs, generator=g)) for p in pipes}, rounds)
        row = dict(res=res, batch=bs, bf16_ms=ms["bf16"], fp8_ms=ms["fp8"], speedup=ms["bf16"] / ms["fp8"])
        print(f"PipelineMuse {res} px batch {bs}: bf16 {ms['bf16']:7.1f} ms | fp8 {ms['fp8']:7.1f} ms | "
              f"x{row['speedup']:.3f}", flush=True)
        rows.append(row)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--timesteps", type=int, default=12)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--batches", default="1,8,64")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8 needs a GPU")
    info = dict(card=card(), torch=torch.__version__)
    print(info["card"], flush=True)
    gemms = gemm_sites(16 * 256, a.iters)
    torch.manual_seed(2)
    vae = VQGANModel(num_embeddings=8192).to(DEV).eval()
    gen, pipe = [], []
    for res in (256, 512):
        torch.manual_seed(4)
        with torch.device(DEV):
            m = MaskGiTUViT_v2(force_down_up_sample=(res == 512))
            with torch.no_grad():  # the zero-initialised output conv would make every logit equal (as bench.py)
                torch.nn.init.trunc_normal_(m.mlm_layer.conv1.weight, std=0.02)
        # one model per precision, same weights: switching one model's precision would rebuild its operands and
        # recapture its graph inside the timed calls
        models = {"bf16": m.eval(), "fp8": copy.deepcopy(m).set_gemm_precision("fp8").eval()}
        gen += generate_rates(models, res, [int(b) for b in a.batches.split(",")], a.timesteps, a.rounds)
        pipe += pipeline_latency(models, vae, res, a.rounds)
        del m, models
        torch.cuda.empty_cache()
    info["card_after"] = card()
    res = dict(info, gemm_sites=gemms, generate2=gen, pipeline=pipe)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(dict(card=info["card"], gemm_speedups=[round(r["speedup"], 3) for r in gemms],
                          generate2_speedups=[round(r["speedup"], 3) for r in gen],
                          pipeline_speedups=[round(r["speedup"], 3) for r in pipe])))


if __name__ == "__main__":
    main()
