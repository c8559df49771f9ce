#!/usr/bin/env python
"""The three norm backward passes of a base-256 train step at batch 256 (T = 65 792 rows), on the row-ring kernels and
on the register-path kernels they replace (MUSE_NORM_BWD_RING=0), alternated within each round; medians of the rounds.
Each call is timed with CUDA events over --iters launches, the ordered column sum of dw included.  Bytes are what the
pass must move (inputs read once, outputs written once); the fraction is of the H100 SXM data-sheet 3.35 TB/s.
The card name and power limit are read in the same call and printed with the numbers.

    python tools/bench_norm_bwd.py [--rounds 3] [--iters 20] [--json OUT.json]"""
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

T, H, I = 65792, 512, 2048
PEAK = 3.35e12
BF = torch.bfloat16


def cases():
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(0)
    rnd = lambda *s, dt=BF: torch.randn(*s, device=dev, generator=g).to(dt)  # noqa: E731
    w, wI = 1 + 0.1 * rnd(H, dt=torch.float32), 1 + 0.1 * rnd(I, dt=torch.float32)
    x, dres, a = rnd(T, H, dt=torch.float32), rnd(T, H, dt=torch.float32), rnd(T, H)
    dy = rnd(T, H)
    _, st = ops.norm_fwd(x, w, 1e-6, BF)
    x2, _, st2 = ops.norm2_fwd(a, dres, w, w, 1e-6)
    ab, dyI = rnd(T, 2 * I), rnd(T, I)
    y, st4 = ops.norm_fwd(ab, wI, 1e-6, BF, act=2)
    seed = torch.tensor([7], dtype=torch.int64, device=dev)
    _, st4d, bits = ops.norm_fwd(ab, wI, 1e-6, BF, act=2, dropout=(0.1, seed, 3))
    e = T * H
    return [
        # bf16 dy + fp32 x + fp32 dres in, fp32 dx + its bf16 copy out
        ("norm_bwd_warp_kernel bf16 dy, fp32 x, +dres, bf16 copy of dx [T,512]", 16 * e,
         lambda: ops.take_bf16_copy(ops.norm_bwd(dy, x, w, st, torch.float32, dres=dres, want_dw=True, bf16_copy=True)[0])),
        # bf16 d_h2 + fp32 x2 + fp32 dres + bf16 a in, fp32 dx2 + bf16 d_a out
        ("norm2_bwd_warp_kernel [T,512]", 18 * e, lambda: ops.norm2_bwd(dy, x2, w, dres, a, w, st2)),
        # bf16 dy + y + [a | b] in, bf16 d[a | b] out
        ("glu_norm_bwd_kernel saved y [T,2x2048]->[T,2048]", 12 * T * I,
         lambda: ops.norm_bwd(dyI, ab, wI, st4, BF, act=2, y_fwd=y, want_dw=True)),
        # bf16 dy + [a | b] + keep bits in, bf16 d[a | b] out
        ("glu_norm_bwd_kernel dropout [T,2x2048]->[T,2048]", 10 * T * I + T * I // 8,
         lambda: ops.norm_bwd(dyI, ab, wI, st4d, BF, act=2, want_dw=True, dropout=(0.1, bits))),
    ]


def time_us(fn, setting, iters):
    os.environ["MUSE_NORM_BWD_RING"] = setting
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    settings = {"register path": "0", "ring": ""}
    gpu = card()
    print(f"# {gpu}")
    rows = []
    for name, nbytes, fn in cases():
        times = {k: [] for k in settings}
        for _ in range(args.rounds):
            for k, v in settings.items():
                times[k].append(time_us(fn, v, args.iters))
        row = {"kernel": name, "algorithmic_bytes": nbytes}
        for k in settings:
            us = statistics.median(times[k])
            row[k] = {"us": us, "GB_per_s": nbytes / us / 1e3, "frac_of_3350_GBps": nbytes / us * 1e6 / PEAK,
                      "rounds_us": times[k]}
            print(f"{name:70s} {k:18s} {nbytes / 1e6:8.1f} MB {us:8.1f} us {nbytes / us / 1e3:7.0f} GB/s "
                  f"{row[k]['frac_of_3350_GBps']:.2f}")
        rows.append(row)
    os.environ.pop("MUSE_NORM_BWD_RING", None)
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"gpu": gpu, "rows": T, "rounds": args.rounds, "iters": args.iters, "peak_GBps": 3350,
                       "peak_source": "H100 SXM data sheet, not measured", "kernels": rows}, f, indent=1)


if __name__ == "__main__":
    main()
