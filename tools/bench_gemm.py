#!/usr/bin/env python
"""Times every GEMM role of the base-256 train step (B=256, S=257 -> T=65792 tokens, H=512, I=2048) alone, with CUDA
events after a warm-up, and reports us, TFLOP/s and the fraction of the H100 SXM data-sheet dense BF16 peak
(989 TFLOP/s at 700 W).  The card name, power limit and SM clock are read in the same run and printed with the numbers.

    python tools/bench_gemm.py [--iters 20] [--warmup 5] [--json OUT.json] [--dump DIR]

--dump DIR writes, per role, the SHA-256 of the output bytes computed on seeded inputs (DIR/gemm_outputs.json), so
two builds can be compared bit for bit without moving gigabytes of outputs around."""
import argparse
import hashlib
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from open_muse_b200 import ops  # noqa: E402

PEAK_BF16_TFLOPS = 989.0  # H100 SXM data sheet, dense BF16, 700 W
B, S, H, I = 256, 257, 512, 2048
T = B * S
# (role, N, K, residual epilogue in forward): the Linear layers of one transformer layer and of the head
LAYERS = [("qkv", 3 * H, H, False), ("attn-out", H, H, True), ("wi", 2 * I, H, False), ("wo", H, I, True),
          ("head dense", H, H, False), ("logits", 2048, H, False)]


def card():
    q = "name,power.limit,clocks.max.sm,clocks_throttle_reasons.active"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        out = torch.cuda.get_device_name()
    return out


def timeit(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--json", help="write the rows as JSON to this file")
    ap.add_argument("--dump", help="directory for the SHA-256 digests of every output on seeded inputs")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_gemm needs a GPU")
    dev = "cuda"
    gen = torch.Generator(device=dev)

    def rnd(seed, *shape, dtype=torch.bfloat16):
        gen.manual_seed(seed)
        return torch.randn(*shape, device=dev, generator=gen).to(dtype)

    info = card()
    print(f"# {info}", flush=True)
    rows, digests = [], {}
    for li, (name, N, K, has_res) in enumerate(LAYERS):
        x, w, dy = rnd(10 * li + 1, T, K), rnd(10 * li + 2, N, K), rnd(10 * li + 3, T, N)
        res = rnd(10 * li + 4, T, N, dtype=torch.float32) if has_res else None
        flops = 2.0 * T * N * K
        # role, majors (A, B: 0 = K-major, 1 = MN-major), epilogue, M, N, K, call
        cases = [(f"fwd {name}" + (" +residual" if has_res else ""), "K,K", "resadd_f32" if has_res else "bf16",
                  T, N, K, lambda: ops.linear_fwd(x, w, res=res)),
                 (f"dgrad {name}", "K,MN", "bf16", T, K, N, lambda: ops.linear_dgrad(dy, w)),
                 (f"wgrad {name}", "MN,MN", "splitk_f32", N, K, T, lambda: ops.linear_wgrad_det(dy, x))]
        if name == "logits":  # the fp32 epilogue at a bench shape (the head's fp32-logits variant)
            cases.append(("fwd logits fp32", "K,K", "f32", T, N, K, lambda: ops.linear_fwd(x, w, out_dtype=torch.float32)))
        for role, majors, epi, m, n, k, fn in cases:
            ms = timeit(fn, args.iters, args.warmup)
            tf = flops / (ms * 1e-3) / 1e12
            row = {"role": role, "M": m, "N": n, "K": k, "majors": majors, "epilogue": epi, "us": ms * 1e3,
                   "tflops": tf, "frac_of_peak": tf / PEAK_BF16_TFLOPS}
            rows.append(row)
            print(f"{role:24s} M={m:6d} N={n:6d} K={k:6d} {majors:6s} {epi:11s} {ms * 1e3:9.1f} us "
                  f"{tf:7.1f} TFLOP/s {tf / PEAK_BF16_TFLOPS:5.3f} of peak", flush=True)
            if args.dump:
                out = fn()
                torch.cuda.synchronize()
                digests[role] = hashlib.sha256(out.contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest()
            del fn
        del x, w, dy, res, cases
        torch.cuda.empty_cache()
    total_us = sum(r["us"] for r in rows)
    total_tf = sum(2.0 * r["M"] * r["N"] * r["K"] for r in rows) / (total_us * 1e-6) / 1e12
    print(f"# all roles: {total_us:.1f} us, {total_tf:.1f} TFLOP/s, {total_tf / PEAK_BF16_TFLOPS:.3f} of peak "
          f"(data-sheet peak {PEAK_BF16_TFLOPS} TFLOP/s at 700 W)")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": info, "peak_tflops": PEAK_BF16_TFLOPS, "rows": rows}, f, indent=1)
    if args.dump:
        os.makedirs(args.dump, exist_ok=True)
        with open(os.path.join(args.dump, "gemm_outputs.json"), "w") as f:
            json.dump(digests, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
