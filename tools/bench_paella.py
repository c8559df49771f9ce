#!/usr/bin/env python
"""PaellaVQModel throughput: get_code (pixels -> ids) and decode_code (ids -> pixels) at 256 px, batch 64, for the default
f4 architecture (levels=2, c_hidden=384, 12 bottleneck blocks) in both tensor-core precisions, the unmodified reference
(oracle/_ref, fp32 eager with torch's default TF32 settings) on the same GPU when the snapshot is present, and an ASSUMED f8
shape (levels=3, c_hidden=384: the f8 checkpoint's config.json is not available offline, so its widths are a guess).

  * CUDA events around --steps calls after --warmup calls, per variant; variants alternate within each of --rounds rounds
    and the median is reported.
  * Roofline: FLOPs and bytes are counted here from the layer shapes, as the kernels run them (bf16x3 = three tensor-core
    passes; the 4x4 strided conv as the 3x3 space-to-depth form it runs as, 2.25x its MACs; ResBlocks as their four
    launches; SIMT layers at the FP32 rate).  The least time is the larger of FLOPs over the data-sheet peak and bytes over
    3.35 TB/s; the fraction is that over the measured time, and the bound that sets it is named.
  * Also: the share of get_code time in the 4x4 strided convolutions, and the token-id agreement of "bf16" with "bf16x3".
  * The card's name and power limit are read in the same run.

    python tools/bench_paella.py [--batch 64] [--res 256] [--rounds 2] [--steps 3] [--warmup 1] [--json OUT.json]"""
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
from oracle import ref_snapshot  # noqa: E402
from open_muse_b200 import PaellaVQModel, ops  # noqa: E402

PEAK_BF16, PEAK_FP32, PEAK_BW = 989e12, 67e12, 3.35e12  # H100 SXM data sheet (dense), HBM3


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


def tc_ok(c):
    return c % 64 == 0


def cost(cfg, res, batch, half):
    """(tensor-core FLOPs, SIMT FLOPs, bytes) of get_code (half="enc") or decode_code ("dec") per call, bf16x3."""
    lv = [cfg["c_hidden"] // 2**i for i in reversed(range(cfg["levels"]))]
    tc = simt = byt = 0.0
    P = 3  # bf16x3 passes

    def conv(px, k_macs, cin, cout, on_tc, in_bytes, out_bytes):
        nonlocal tc, simt, byt
        fl = 2.0 * px * k_macs * cout
        if on_tc:
            tc += P * fl
        else:
            simt += fl
        byt += px * (in_bytes + out_bytes)

    def resblock(px, c):
        nonlocal simt, byt
        simt += 2.0 * px * 9 * c           # depthwise (CUDA cores)
        byt += px * 4 * c * 2              # statistics pass reads x; spatial pass reads x again (neighbours from cache)
        byt += px * 4 * c                  # writes x1
        t = tc_ok(c)
        conv(px, c, c, 4 * c, t, 4 * c if t else 4 * c, 16 * c if t else 16 * c)  # LN2 planes in, GELU planes out
        conv(px, 4 * c, 4 * c, c, t, 16 * c + 4 * c, 4 * c)                       # + residual x1 in, y out

    h = res // 2
    if half == "enc":
        conv(h * h * batch, 12, 12, lv[0], True, 12 + 2 * 64 * 2, 4 * lv[0])
        for i, c in enumerate(lv):
            if i > 0:
                h //= 2
                conv(h * h * batch, 36 * lv[i - 1], 4 * lv[i - 1], c, tc_ok(4 * lv[i - 1]), 4 * 4 * lv[i - 1] * 3, 4 * c)
            resblock(h * h * batch, c)
        conv(h * h * batch, lv[-1], lv[-1], 4, tc_ok(lv[-1]), 4 * lv[-1] * 2, 16)
        simt += 2.0 * h * h * batch * 4 * cfg["codebook_size"]  # the arg-min (fp32 SIMT)
    else:
        h = res // 2 ** cfg["levels"]
        conv(h * h * batch, 4, 4, lv[-1], True, 16 + 64 * 2 * 2, 4 * lv[-1])
        for i, c in enumerate(reversed(lv)):
            for _ in range(cfg["bottleneck_blocks"] if i == 0 else 1):
                resblock(h * h * batch, c)
            if i < len(lv) - 1:
                h *= 2
                cout = lv[len(lv) - 2 - i]
                conv(h * h * batch, 4 * c, c, cout, tc_ok(c), 4 * c * 3 / 4, 4 * cout)
        conv(h * h * batch, lv[0], lv[0], 12, tc_ok(lv[0]), 4 * lv[0] * 2, 48)
    return tc, simt, byt


def roofline(cfg, res, batch, half, ms, passes):
    tc, simt, byt = cost(cfg, res, batch, half)
    tc = tc * passes / 3
    t_c = tc / PEAK_BF16 + simt / PEAK_FP32
    t_b = byt / PEAK_BW
    t_min = max(t_c, t_b)
    return dict(gflop_tc=tc / 1e9, gflop_simt=simt / 1e9, gbytes=byt / 1e9, bound="compute" if t_c >= t_b else "memory",
                roofline_fraction=t_min / (ms * 1e-3))


def make_model(cfg, seed=0):
    torch.manual_seed(seed)
    m = PaellaVQModel(**cfg)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():  # trained-like: non-zero gammas, BatchNorm statistics, a codebook with the spread of z
        for k, p in m.named_parameters():
            if k.endswith("gammas"):
                p.copy_(torch.randn(6, generator=g) * 0.5)
        bn = m.down_blocks[-1][1]
        bn.running_mean.copy_(torch.randn(bn.num_features, generator=g) * 0.2)
        bn.running_var.copy_(torch.rand(bn.num_features, generator=g) + 0.5)
        m.vquantizer.codebook.weight.copy_(torch.randn(m.codebook_size, m.c_latent, generator=g))
    return m.eval().cuda()


def ref_model(cfg, sd):
    if not ref_snapshot.available():
        return None
    ref_snapshot.import_reference()  # registers the snapshot as the package `muse`
    from muse.modeling_paella_vq import PaellaVQModel as RefPaella  # noqa: E402

    m = RefPaella(**cfg)
    m.load_state_dict(sd)
    return m.eval().cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--res", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_paella needs a GPU"
    dev_card = card()
    shapes = {"f4_default": dict(levels=2, c_hidden=384, bottleneck_blocks=12, c_latent=4, codebook_size=8192),
              "f8_assumed": dict(levels=3, c_hidden=384, bottleneck_blocks=12, c_latent=4, codebook_size=8192)}
    img = torch.rand(args.batch, 3, args.res, args.res, generator=torch.Generator().manual_seed(7)).cuda() * 2 - 1
    out = {"card": dev_card, "batch": args.batch, "res": args.res, "results": {}}
    for sname, cfg in shapes.items():
        m = make_model(cfg)
        ids = m.get_code(img)
        variants = {}
        for prec in ("bf16x3", "bf16"):
            variants[f"get_code/{prec}"] = (lambda p=prec: (m.set_conv_precision(p), m.get_code(img)))
            variants[f"decode_code/{prec}"] = (lambda p=prec: (m.set_conv_precision(p), m.decode_code(ids)))
        ref = ref_model(cfg, m.state_dict()) if sname == "f4_default" else None
        if ref is not None:
            with torch.no_grad():
                variants["get_code/reference"] = lambda: ref.get_code(img)
                variants["decode_code/reference"] = lambda: ref.decode_code(ids)
        times = {k: [] for k in variants}
        for _ in range(args.rounds):
            for k, fn in variants.items():
                with torch.no_grad():
                    times[k].append(timed(fn, args.steps, args.warmup))
        m.set_conv_precision("bf16x3")
        res = {}
        for k, ts in times.items():
            ms = statistics.median(ts)
            half = "enc" if k.startswith("get_code") else "dec"
            r = dict(ms=ms, images_per_s=args.batch / (ms * 1e-3), rounds_ms=ts)
            if not k.endswith("reference"):
                r.update(roofline(cfg, args.res, args.batch, half, ms, 3 if k.endswith("bf16x3") else 1))
            res[k] = r
        # share of the 4x4 strided convolutions in get_code (bf16x3): time them alone on their own inputs
        h = ops.conv2d_unshuffle(ops.to_nhwc(img), m.in_block[1].weight, m.in_block[1].bias)
        s_ms = 0.0
        for blk in m.down_blocks[:-1]:
            if isinstance(blk, torch.nn.Conv2d):
                s_ms += timed(lambda b=blk, x=h: ops.conv2d_s2p1(x, b.weight, b.bias), args.steps, args.warmup)
                h = ops.conv2d_s2p1(h, blk.weight, blk.bias)
            else:
                h = blk.run(h)
        res["strided_conv_share_of_get_code"] = s_ms / res["get_code/bf16x3"]["ms"]
        m.set_conv_precision("bf16")
        res["bf16_id_agreement"] = float((m.get_code(img) == ids).float().mean())
        m.set_conv_precision("bf16x3")
        if ref is not None:
            with torch.no_grad():
                res["reference_id_agreement"] = float((ref.get_code(img) == ids).float().mean())
            for half in ("get_code", "decode_code"):
                res[f"{half}/speedup_vs_reference"] = res[f"{half}/reference"]["ms"] / res[f"{half}/bf16x3"]["ms"]
        out["results"][sname] = res
        del m, ref
        torch.cuda.empty_cache()
    line = json.dumps(out)
    print(line)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
