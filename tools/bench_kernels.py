#!/usr/bin/env python
"""Per-kernel timings at the base-256 shapes (B=256, T=65792, H=512, I=2048) with CUDA events.
Prints achieved GB/s (algorithmic bytes) or TFLOP/s per op -- the inner optimisation loop of the round.

    python tools/bench_kernels.py [GROUP ...] [--dump DIR]

GROUP selects the groups whose name contains it (glu, rownorm, norm, attn, gemm, resgemm; default all).  rownorm times every entry
point of the warp-per-row LayerNorm / RMSNorm kernels at the shapes training runs, on seeded inputs; with --dump DIR it
also writes DIR/rownorm_outputs.json, the SHA-256 of every run-to-run deterministic output, and DIR/rownorm_atomic.pt,
the weight gradients accumulated with atomics (order-dependent, so two builds are compared with a tolerance)."""
import argparse
import hashlib
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from open_muse_b200 import ops  # noqa: E402

dev = "cuda"
B, S, H, I, nh = 256, 257, 512, 2048, 8
T = B * S


def timeit(fn, n=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def report(name, ms, gbytes=None, gflop=None):
    s = f"{name:34s} {ms*1e3:9.1f} us"
    if gbytes is not None:
        s += f"  {gbytes/ms:8.1f} GB/s"
    if gflop is not None:
        s += f"  {gflop/ms:8.1f} TFLOP/s"
    print(s, flush=True)


def bf(*shape):
    return torch.randn(*shape, device=dev).to(torch.bfloat16)


ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
ap.add_argument("groups", nargs="*")
ap.add_argument("--dump", help="directory for the digests / tensors of the rownorm outputs")
args = ap.parse_args()
only = args.groups or None


def want(tag):
    return only is None or any(o in tag for o in only)


def rownorm(dump):
    """(name, call, atomic) for each entry point of the warp-per-row norm kernels: call() returns the outputs as a dict,
    atomic names the outputs that accumulate with atomics (zeroed before the dumped call)."""
    gen = torch.Generator(device=dev)

    def rnd(seed, *shape, dtype=torch.float32):
        gen.manual_seed(seed)
        return torch.randn(*shape, device=dev, generator=gen).to(dtype)

    cases = []
    for Hn in (512, 1024):  # base-256 width; cc12m width (4 chunks of 256 columns per lane)
        x, xb, res, dres = rnd(1, T, Hn), rnd(2, T, Hn, dtype=torch.bfloat16), rnd(3, T, Hn), rnd(4, T, Hn)
        dyb, w, w2 = rnd(5, T, Hn, dtype=torch.bfloat16), 1 + 0.1 * rnd(6, Hn), 1 + 0.1 * rnd(7, Hn)
        st = ops.norm_fwd(x, w, 1e-6, torch.bfloat16)[1]
        dw = torch.zeros(Hn, device=dev)
        x2, _, st2 = ops.norm2_fwd(xb, res, w, w2, 1e-6)

        def bwd_copy(x=x, w=w, st=st, dyb=dyb, dres=dres):
            dx, dwo = ops.norm_bwd(dyb, x, w, st, torch.float32, dres=dres, want_dw=True, bf16_copy=True)
            return {"dx": dx, "dx_copy": ops.take_bf16_copy(dx), "dw": dwo}

        def bwd_atomic(x=x, w=w, st=st, dyb=dyb, dres=dres, dw=dw):
            return {"dx": ops.norm_bwd(dyb, x, w, st, torch.float32, dw=dw, dres=dres), "dw": dw}

        cases += [
            (f"norm_fwd fp32->bf16 H={Hn}", lambda x=x, w=w: dict(zip(("y", "stats"), ops.norm_fwd(x, w, 1e-6, torch.bfloat16))), ()),
            (f"norm_fwd bf16->fp32 +res H={Hn}",
             lambda xb=xb, w=w, res=res: dict(zip(("y", "stats"), ops.norm_fwd(xb, w, 1e-6, torch.float32, res=res))), ()),
            (f"norm_bwd +dres, bf16 copy, ordered dw H={Hn}", bwd_copy, ()),
            (f"norm_bwd +dres, atomic dw H={Hn}", bwd_atomic, ("dw",)),
            (f"norm2_fwd H={Hn}", lambda xb=xb, res=res, w=w, w2=w2: dict(zip(("x2", "h2", "stats"), ops.norm2_fwd(xb, res, w, w2, 1e-6))), ()),
            (f"norm2_bwd H={Hn}", lambda dyb=dyb, x2=x2, w2=w2, dres=dres, xb=xb, w=w, st2=st2: dict(zip(
                ("dx2", "d_a", "dw1", "dw2"), ops.norm2_bwd(dyb, x2, w2, dres, xb, w, st2))), ()),
        ]
    Bu, S = 32, 256  # MaskGiTUViT_v2 defaults: batch 32, 16 x 16 = 256 tokens
    for Hn, with_mod, rms in ((1024, True, 1), (768, False, 0)):
        a, r, w = rnd(11, Bu * S, Hn, dtype=torch.bfloat16), rnd(12, Bu * S, Hn), 1 + 0.1 * rnd(13, Hn)
        mod = 0.1 * rnd(14, Bu, 2 * Hn) if with_mod else None
        dy, dr_out = rnd(15, Bu * S, Hn, dtype=torch.bfloat16), rnd(16, Bu * S, Hn)
        r_out = ops.add_norm_mod(a, w, 1e-6, rms, residual=r, mod=mod, rows_per_sample=S)[0]
        dw = torch.zeros(Hn, device=dev)
        dmod = torch.zeros(Bu, 2 * Hn, device=dev) if with_mod else None
        tag = f"H={Hn}" + (" +mod" if with_mod else "")

        def anm_bwd(dy=dy, dr_out=dr_out, r_out=r_out, w=w, rms=rms, mod=mod, dw=dw, dmod=dmod):
            da, dr = ops.add_norm_mod_bwd(dy, dr_out, r_out, w, 1e-6, rms, torch.bfloat16, mod=mod, rows_per_sample=S, dw=dw,
                                          dmod=dmod)
            return {"da": da, "dr": dr, "dw": dw, **({"dmod": dmod} if dmod is not None else {})}

        cases += [
            (f"add_norm_mod {tag}", lambda a=a, w=w, rms=rms, r=r, mod=mod: dict(zip(("r_out", "y"), ops.add_norm_mod(
                a, w, 1e-6, rms, residual=r, mod=mod, rows_per_sample=S))), ()),
            (f"add_norm_mod_bwd {tag}", anm_bwd, ("dw", "dmod")),
        ]
    C, hw = 768, 16
    xd, wk, nw = rnd(21, Bu * hw * hw, C), 0.3 * rnd(22, 9, C), 1 + 0.1 * rnd(23, C)
    dyd, dresd = rnd(24, Bu * hw * hw, C, dtype=torch.bfloat16), rnd(25, Bu * hw * hw, C)
    conv = ops.dwconv3x3_norm(xd, wk, nw, Bu, hw, hw, 1e-6, 0, save_conv=True)[1]
    dwk, dnw = torch.zeros(9, C, device=dev), torch.zeros(C, device=dev)
    cases += [
        (f"dwconv3x3_norm C={C}", lambda: dict(zip(("y", "conv"), ops.dwconv3x3_norm(xd, wk, nw, Bu, hw, hw, 1e-6, 0, save_conv=True))), ()),
        (f"dwconv3x3_norm_bwd C={C}", lambda: {"dx": ops.dwconv3x3_norm_bwd(dyd, conv, xd, wk, nw, dresd, dwk, dnw, Bu, hw, hw, 1e-6, 0),
                                               "dwk": dwk, "dnw": dnw}, ("dwk", "dnw")),
    ]
    digests, atomic = {}, {}
    for name, call, acc in cases:
        report(name, timeit(call, n=20, warm=5))
        if dump:
            outs = call()  # the buffers to zero are the ones this call returns
            for k in acc:
                if k in outs:
                    outs[k].zero_()
            outs = call()
            torch.cuda.synchronize()
            for k, t in outs.items():
                if k in acc:
                    atomic[f"{name}/{k}"] = t.cpu()
                else:
                    digests[f"{name}/{k}"] = hashlib.sha256(t.contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest()
    if dump:
        os.makedirs(dump, exist_ok=True)
        with open(os.path.join(dump, "rownorm_outputs.json"), "w") as f:
            json.dump(digests, f, indent=1, sort_keys=True)
        torch.save(atomic, os.path.join(dump, "rownorm_atomic.pt"))


u = T * H * 2 / 1e6  # MB of one bf16 [T,H]
if want("glu"):
    ab = bf(T, 2 * I)
    w = torch.ones(I, device=dev)
    dy = bf(T, I)
    dw = torch.zeros(I, device=dev)
    y, st = ops.norm_fwd(ab, w, 1e-6, torch.bfloat16, act=2)
    report("glu+LN fwd (fused)", timeit(lambda: ops.norm_fwd(ab, w, 1e-6, torch.bfloat16, act=2)), 12 * u)
    report("glu+LN bwd (fused)", timeit(lambda: ops.norm_bwd(dy, ab, w, st, torch.bfloat16, dw=dw, act=2)), 20 * u)
    report("glu+LN bwd (fused, saved y)", timeit(lambda: ops.norm_bwd(dy, ab, w, st, torch.bfloat16, dw=dw, act=2, y_fwd=y)), 24 * u)
    report("glu fwd (plain)", timeit(lambda: ops.glu_fwd(ab)), 12 * u)
    report("glu bwd (plain)", timeit(lambda: ops.glu_bwd(ab, dy)), 20 * u)
    gl = ops.glu_fwd(ab)
    y2, st2 = ops.norm_fwd(gl, w, 1e-6, torch.bfloat16)
    report("LN fwd [T,2048] bf16->bf16", timeit(lambda: ops.norm_fwd(gl, w, 1e-6, torch.bfloat16)), 8 * u)
    report("LN bwd [T,2048] bf16", timeit(lambda: ops.norm_bwd(dy, gl, w, st2, torch.bfloat16, dw=dw)), 12 * u)
    del ab, dy, gl, y, y2
if want("rownorm"):
    rownorm(args.dump)
if want("norm"):
    x = torch.randn(T, H, device=dev)
    w = torch.ones(H, device=dev)
    xb = bf(T, H)
    dres = torch.randn(T, H, device=dev)
    dw = torch.zeros(H, device=dev)
    y, st = ops.norm_fwd(x, w, 1e-6, torch.bfloat16)
    report("LN fwd fp32->bf16 [T,512]", timeit(lambda: ops.norm_fwd(x, w, 1e-6, torch.bfloat16)), 3 * u)
    report("LN fwd bf16->fp32 +res", timeit(lambda: ops.norm_fwd(xb, w, 1e-6, torch.float32, res=x)), 5 * u)
    report("LN bwd bf16 dy, fp32 x, +dres", timeit(lambda: ops.norm_bwd(xb, x, w, st, torch.float32, dw=dw, dres=dres)), 7 * u)
    report("LN bwd fp32 dy, bf16 x -> bf16", timeit(lambda: ops.norm_bwd(x, xb, w, st, torch.bfloat16, dw=dw)), 4 * u)
    report("cast fp32->bf16", timeit(lambda: ops.cast_bf16(x)), 3 * u)
    ids_e = torch.randint(0, 1024, (256, 257), device=dev)
    ids_e[torch.rand(256, 257, device=dev) < 0.5] = 2024
    dword, dpos = torch.zeros(2025, H, device=dev), torch.zeros(257, H, device=dev)
    report("embed bwd (half of the tokens = mask id)", timeit(lambda: ops.embed_bwd(ids_e, x, dword, dpos)), 2 * u)
if want("attn"):
    qkv = bf(T, 3 * H)
    scale = 0.125
    o, lse = ops.attn_fwd(qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:], B, nh, S, S, scale)
    do = bf(T, H)
    dqkv = torch.empty_like(qkv)
    fl = 4 * S * S * 64 * B * nh / 1e9
    report("attn fwd", timeit(lambda: ops.attn_fwd(qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:], B, nh, S, S, scale)), gflop=fl)
    report("attn bwd", timeit(lambda: ops.attn_bwd(qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:], o, do, lse, dqkv[:, :H],
                                                   dqkv[:, H:2 * H], dqkv[:, 2 * H:], B, nh, S, S, scale)), gflop=2.5 * fl)
if want("gemm"):
    x = bf(T, H)
    for name, N, K in [("qkv", 3 * H, H), ("out", H, H), ("wi", 2 * I, H), ("wo", H, I), ("logits", 2048, H)]:
        w = bf(N, K)
        xin = bf(T, K)
        fl = 2 * T * N * K / 1e9
        report(f"gemm fwd {name} [T,{K}]x[{N},{K}]", timeit(lambda: ops.linear_fwd(xin, w)), gflop=fl)
        dyy = bf(T, N)
        report(f"gemm dgrad {name}", timeit(lambda: ops.linear_dgrad(dyy, w)), gflop=fl)
        dwt = torch.zeros(N, K, device=dev)
        report(f"gemm wgrad {name}", timeit(lambda: ops.linear_wgrad(dyy, xin, dwt)), gflop=fl)
    res = torch.randn(T, H, device=dev)
    w = bf(H, I)
    xin = bf(T, I)
    report("gemm wo + residual (fp32 out)", timeit(lambda: ops.linear_fwd(xin, w, res=res)), gflop=2 * T * H * I / 1e9)
if want("resgemm"):  # the two residual-epilogue GEMMs of a layer (attention out-projection, FFN wo)
    res = torch.randn(T, H, device=dev)
    for name, K in [("attn out", H), ("wo", I)]:
        w = bf(H, K)
        xin = bf(T, K)
        report(f"gemm {name} + residual (fp32 out)", timeit(lambda: ops.linear_fwd(xin, w, res=res), n=20), gbytes=(T * K * 2 + 2 * T * H * 4) / 1e6,
               gflop=2 * T * H * K / 1e9)
