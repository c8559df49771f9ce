#!/usr/bin/env python
"""FP8 against bf16 GEMM precision of ``MaskGitTransformer`` (``set_gemm_precision``), alternated within one call after a
warm-up of each, medians over --rounds rounds; one model per precision:

  * ``sites``: each FP8 GEMM site of a layer against its bf16 GEMM, CUDA events over --iters calls: ``qkv``, ``cq``
    (cross-attention q, text-conditional only), ``wi`` ([wi_0;wi_1]) and ``wo`` with its fp32 residual add, at the base
    widths (H 512, I 2048, 64 x 257 tokens) and the cc12m widths (H 1024, I 4096, 256 tokens, batch 8 and 64 x 2 for
    classifier-free guidance).  The FP8 operands come from the e4m3 passes, so only the GEMM is timed on either side;
  * ``generate2_steps_per_s``: decode steps per second of ``generate2`` (CUDA graph, 12 steps): the class-conditional
    base model at batch 64 (BASELINE config 5), and a 24-layer cc12m.yaml-width text-conditional model with guidance
    3 at batch 8 and 64 (random encoder states);
  * ``pipeline_ms``: ``PipelineMuse`` latency, class-conditional base model + MaskGitVQGAN decode + PIL, 12 steps, batch
    1 and 8.

Random weights.  The card name and power limit are read in the same call.

    python tools/bench_fp8_transformer.py [--rounds 3] [--iters 50] [--json OUT.json]"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, ROOT)
from bench_gemm import card  # noqa: E402
from open_muse_b200 import MaskGitTransformer, MaskGitVQGAN, PipelineMuse, ops  # noqa: E402

DEV = "cuda"
BASE = dict(vocab_size=2025, max_position_embeddings=257, hidden_size=512, num_hidden_layers=8, num_attention_heads=8,
            intermediate_size=2048, codebook_size=1024, num_vq_tokens=256, num_classes=1000, hidden_dropout=0.0,
            attention_dropout=0.0)
CC12M = dict(add_cross_attention=True, codebook_size=8192, encoder_hidden_size=1024, hidden_size=1024,
             intermediate_size=4096, layer_norm_eps=1e-6, max_position_embeddings=256, norm_type="rmsnorm",
             num_attention_heads=16, num_hidden_layers=24, num_vq_tokens=256, use_codebook_size_for_output=True,
             use_normformer=False, vocab_size=8256, hidden_dropout=0.0, attention_dropout=0.0)
PRECISIONS = ("bf16", "fp8")


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


def site_calls(T, H, I, cross, g):
    """{site: {precision: zero-argument GEMM call}} on random operands of one layer"""
    r = lambda *s: torch.randn(*s, device=DEV, generator=g)  # noqa: E731
    shapes = {"qkv": (H, 3 * H), "wi": (H, 2 * I), "wo": (I, H)}
    if cross:
        shapes["cq"] = (H, H)
    res = r(T, H)
    out = {}
    for site, (K, N) in shapes.items():
        x = r(T, K).to(torch.bfloat16)
        w = (r(N, K) * 0.02).to(torch.bfloat16)
        x8, w8 = ops.quantize_rows_e4m3(x), ops.quantize_rows_e4m3(w)
        kw = {"res": res} if site == "wo" else {}
        out[site] = {"bf16": (lambda x=x, w=w, kw=kw: ops.linear_fwd(x, w, **kw)),
                     "fp8": (lambda x8=x8, w8=w8, kw=kw: ops.linear_fwd(x8, w8, **kw))}
    return out


def models(cfg):
    out = {}
    for prec in PRECISIONS:
        torch.manual_seed(0)
        out[prec] = MaskGitTransformer(**cfg).to(DEV).eval().set_gemm_precision(prec)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark measures the H100: no GPU found"
    result = {"card": card(), "rounds": a.rounds, "iters": a.iters}
    g = torch.Generator(device=DEV).manual_seed(0)

    # ---- GEMM sites
    workloads = {"base H512 I2048 64x257": (64 * 257, 512, 2048, False),
                 "cc12m H1024 I4096 8x256": (8 * 256, 1024, 4096, True),
                 "cc12m H1024 I4096 64x256 cfg": (128 * 256, 1024, 4096, True)}
    sites = {}
    for wl, (T, H, I, cross) in workloads.items():
        calls = site_calls(T, H, I, cross, g)
        times = {s: {p: [] for p in PRECISIONS} for s in calls}
        for s in calls:
            for p in PRECISIONS:
                events(calls[s][p], 5)  # warm-up
        for _ in range(a.rounds):
            for s in calls:
                for p in PRECISIONS:
                    times[s][p].append(events(calls[s][p], a.iters) * 1e3)
        sites[wl] = {s: {"bf16_us": statistics.median(t["bf16"]), "fp8_us": statistics.median(t["fp8"]),
                         "speedup": statistics.median(t["bf16"]) / statistics.median(t["fp8"]),
                         "bf16_rounds_us": t["bf16"], "fp8_rounds_us": t["fp8"]} for s, t in times.items()}
        del calls
    result["sites"] = sites
    print(json.dumps({"sites": {wl: {s: round(v["speedup"], 3) for s, v in d.items()} for wl, d in sites.items()}}),
          flush=True)

    # ---- generate2
    gen = {}

    def decode(ms, kw, name, steps=12):
        calls = {p: (lambda p=p: ms[p].generate2(**{k: (v.clone() if torch.is_tensor(v) else v) for k, v in kw.items()},
                                                 timesteps=steps, generator=torch.Generator(device=DEV).manual_seed(1)))
                 for p in PRECISIONS}
        for p in PRECISIONS:
            calls[p]()
        t = {p: [] for p in PRECISIONS}
        for _ in range(a.rounds):
            for p in PRECISIONS:
                t[p].append(steps / (events(calls[p], 3) * 1e-3))
        gen[name] = {f"{p}_steps_per_s": statistics.median(t[p]) for p in PRECISIONS}
        gen[name]["speedup"] = gen[name]["fp8_steps_per_s"] / gen[name]["bf16_steps_per_s"]
        gen[name].update({f"{p}_rounds": t[p] for p in PRECISIONS})
        print(json.dumps({name: round(gen[name]["speedup"], 3)}), flush=True)

    base = models(BASE)
    decode(base, dict(class_ids=torch.randint(0, 1000, (64,), device=DEV, generator=g)), "base class-cond B=64 (config 5)")
    big = models(CC12M)
    for B in (8, 64):
        ehs = torch.randn(B, 77, 1024, device=DEV, generator=g)
        decode(big, dict(encoder_hidden_states=ehs, negative_embeds=torch.zeros_like(ehs), guidance_scale=3.0),
               f"cc12m widths 24 layers, CFG 3, B={B}")
    del big
    torch.cuda.empty_cache()
    result["generate2"] = gen

    # ---- PipelineMuse
    torch.manual_seed(2)
    vae = MaskGitVQGAN().to(DEV).eval()
    pipes = {p: PipelineMuse(vae=vae, transformer=base[p], is_class_conditioned=True).to(DEV) for p in PRECISIONS}
    pipe_ms = {}
    for bs in (1, 8):
        run = {p: (lambda p=p: pipes[p](class_ids=[207], num_images_per_prompt=bs, timesteps=12,
                                        generator=torch.Generator(device=DEV).manual_seed(3))) for p in PRECISIONS}
        t = {p: [] for p in PRECISIONS}
        for p in PRECISIONS:
            imgs = run[p]()
            assert len(imgs) == bs
        for _ in range(a.rounds):
            for p in PRECISIONS:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                run[p]()
                torch.cuda.synchronize()
                t[p].append((time.perf_counter() - t0) * 1e3)
        pipe_ms[f"bs{bs}"] = {f"{p}_ms": statistics.median(t[p]) for p in PRECISIONS}
        pipe_ms[f"bs{bs}"].update({f"{p}_rounds_ms": t[p] for p in PRECISIONS})
    result["pipeline_ms"] = pipe_ms
    result["card_after"] = card()
    print(json.dumps(result, indent=1))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
