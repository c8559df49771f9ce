#!/usr/bin/env python
"""MOVQ throughput: get_code (pixels -> ids) and decode_code (ids -> pixels) at the class defaults (hidden 128, channel_mult
(1, 2, 2, 4), f8, 16384 codes), 256 px, batch 64, in both tensor-core precisions, and the unmodified reference
(oracle/_ref, fp32 eager with torch's default TF32 settings) on the same GPU when the snapshot is present.

  * CUDA events around --steps calls after --warmup calls, per variant; variants alternate within each of --rounds rounds
    and the median is reported.
  * Roofline: FLOPs and bytes are counted here from the layer shapes, by running the fp64 restatement
    (oracle/movq_oracle.py) on one image with counting wrappers around its convolutions: every convolution as written in
    the reference (the upsample convolutions at the high resolution they are written at, although the kernels run them as
    2x2 parity convolutions with 4/9 of those MACs), three tensor-core passes in bf16x3, plus the attention products.  Bytes
    per convolution: its fp32 input read twice by the GroupNorm pass (statistics, apply), written and read once more as
    bf16 hi + lo planes, and its fp32 output written.  The least time is the larger of FLOPs over the data-sheet bf16 peak
    and bytes over 3.35 TB/s; the fraction is that over the measured time, and the bound that sets it is named.
  * Also: the share of decode_code time (bf16x3) in the SpatialNorm passes (statistics, finalize and modulated apply
    kernels, from torch.profiler: every GroupNorm of the decoder is a SpatialNorm), and the token-id agreement of "bf16"
    with "bf16x3".
  * The card's name and power limit are read in the same run.

    python tools/bench_movq.py [--batch 64] [--res 256] [--rounds 2] [--steps 3] [--warmup 1] [--json OUT.json]"""
import argparse
import json
import os
import statistics
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_gemm import card  # noqa: E402
from oracle import movq_oracle as O  # noqa: E402
from oracle import ref_snapshot  # noqa: E402
from open_muse_b200 import MOVQ  # noqa: E402

PEAK_BF16, PEAK_BW = 989e12, 3.35e12  # H100 SXM data sheet (dense), HBM3


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


def cost(m, res, batch):
    """{half: (tensor-core FLOPs of one bf16 pass, bytes)} per call, counted on one image of the fp64 restatement"""
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    cfg = dict(m.config)
    tally = {"fl": 0.0, "by": 0.0}
    conv = F.conv2d

    def counting(x, w, b=None, stride=1, padding=0, *a, **k):
        y = conv(x, w, b, stride, padding, *a, **k)
        tally["fl"] += 2.0 * y.numel() * w[0].numel()
        tally["by"] += 4.0 * x.numel() * 4 + 4.0 * y.numel()
        return y

    def attn_flops(n_blocks, t, c):
        return n_blocks * (4 * 2.0 * t * c * c + 4.0 * t * t * c)

    t = m.config.latent_size ** 2
    c = m.config.hidden_channels * m.config.channel_mult[-1]
    n_att_enc = sum(len(d.attn) for d in m.encoder.down if len(d.attn) > 1) + 1
    n_att_dec = sum(len(u.attn) for u in m.decoder.up if len(u.attn) > 1) + 1
    out = {}
    img = torch.zeros(1, 3, res, res, device="cuda", dtype=torch.float64)
    ids = torch.zeros(1, t, dtype=torch.long, device="cuda")
    F.conv2d = counting
    try:
        with torch.no_grad():
            O.encoder(sd, cfg, img)
            out["get_code"] = ((tally["fl"] + attn_flops(n_att_enc, t, c)) * batch, tally["by"] * batch)
            tally["fl"] = tally["by"] = 0.0
            O.decode_code(sd, cfg, ids)
            out["decode_code"] = ((tally["fl"] + attn_flops(n_att_dec, t, c)) * batch, tally["by"] * batch)
    finally:
        F.conv2d = conv
    return out


def roofline(fl_pass, byt, ms, passes):
    t_c, t_b = fl_pass * passes / PEAK_BF16, byt / PEAK_BW
    return dict(gflop_tc=fl_pass * passes / 1e9, gbytes=byt / 1e9, bound="compute" if t_c >= t_b else "memory",
                roofline_fraction=max(t_c, t_b) / (ms * 1e-3))


def spatial_norm_share(m, ids):
    from torch.profiler import ProfilerActivity, profile

    m.decode_code(ids)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m.decode_code(ids)
        torch.cuda.synchronize()
    tot = gn = 0.0
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if e.key.startswith(("cudaLaunch", "cudaDevice", "cudaStream", "cudaEvent", "cudaMemcpy", "cudaFunc")):
            continue
        tot += us
        if "gn_stats" in e.key or "gn_finalize" in e.key or "gn_apply" in e.key:
            gn += us
    return gn / tot if tot else float("nan")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--res", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_movq needs a GPU"
    dev_card = card()
    torch.manual_seed(0)
    m = MOVQ(resolution=args.res).eval().cuda()
    g = torch.Generator().manual_seed(1)
    img = torch.rand(args.batch, 3, args.res, args.res, generator=g).cuda() * 2 - 1
    with torch.no_grad():  # a codebook with the spread of z, so that the ids are not all near-ties
        z = m._encode_nhwc(img[:4])
        m.quantize.embedding.weight.copy_(torch.randn(16384, 4, generator=g).cuda() * z.std() + z.mean())
    ids = m.get_code(img)
    variants = {}
    for prec in ("bf16x3", "bf16"):
        variants[f"get_code/{prec}"] = (lambda p=prec: (m.set_conv_precision(p), m.get_code(img)))
        variants[f"decode_code/{prec}"] = (lambda p=prec: (m.set_conv_precision(p), m.decode_code(ids)))
    ref = None
    if ref_snapshot.available():
        ref_snapshot.import_reference()
        from muse.modeling_movq import MOVQ as RefMOVQ  # noqa: E402

        ref = RefMOVQ(resolution=args.res)
        ref.load_state_dict(m.state_dict())
        ref = ref.eval().cuda()
        variants["get_code/reference"] = lambda: ref.get_code(img)
        variants["decode_code/reference"] = lambda: ref.decode_code(ids)
    times = {k: [] for k in variants}
    for _ in range(args.rounds):
        for k, fn in variants.items():
            with torch.no_grad():
                times[k].append(timed(fn, args.steps, args.warmup))
    m.set_conv_precision("bf16x3")
    counted = cost(m, args.res, args.batch)
    res = {}
    for k, ts in times.items():
        ms = statistics.median(ts)
        r = dict(ms=ms, images_per_s=args.batch / (ms * 1e-3), rounds_ms=ts)
        if not k.endswith("reference"):
            half = k.split("/")[0]
            r.update(roofline(*counted[half], ms, 3 if k.endswith("bf16x3") else 1))
        res[k] = r
    res["spatial_norm_share_of_decode_code"] = spatial_norm_share(m, ids)
    m.set_conv_precision("bf16")
    res["bf16_id_agreement"] = float((m.get_code(img) == ids).float().mean())
    m.set_conv_precision("bf16x3")
    if ref is not None:
        with torch.no_grad():
            res["reference_id_agreement"] = float((ref.get_code(img) == ids).float().mean())
        for half in ("get_code", "decode_code"):
            res[f"{half}/speedup_vs_reference"] = res[f"{half}/reference"]["ms"] / res[f"{half}/bf16x3"]["ms"]
    out = {"card": dev_card, "batch": args.batch, "res": args.res, "config": "MOVQ class defaults", "results": res}
    line = json.dumps(out)
    print(line)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
