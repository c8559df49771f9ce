"""Local error checks for the bf16 training kernels: the error of every row, tile or head against an fp64 reference.

A whole-tensor ||out - ref|| / ||ref|| divides the error of one wrong row by the square root of the number of rows, so a
tiled kernel that gets one row, one tile or one head wrong (a ragged tail tile, an off-by-one mask, state carried from
one tile to the next) can stay under it.  check_local() splits both tensors into groups -- rows of the kernel's output,
output tiles, (batch, head, row) of attention -- and bounds the error of each group on its own:

    e_g    = ||out_g - ref_g|| / max(||ref_g||, median_g ||ref_g|| / 16)
    elem_g = max |out_g - ref_g| / (the same denominator / sqrt(n))     (n = elements per group)

The floor keeps near-zero groups (a key nobody attends to, an ignored row) from dividing by nothing.  A failure names
the worst group in the kernel's own coordinates and gives the next-worst one.

BOUNDS holds one (group bound, elementwise bound) pair per kernel output.  Each group bound is about twice the worst
per-group error measured on an H100 SXM over all cases of tests/test_kernel_local_gpu.py (value in the comment), rounded
up; bf16 outputs stay at or below 2e-2, where tests/test_local_error_cpu.py shows that the bounds reject subtly wrong
kernels."""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Callable

import torch


@dataclass
class Groups:
    """view: tensor -> [G, n] (one group per row); where: group index -> its coordinates in the kernel's terms;
    sizes: elements per group when the view pads groups with zeros (default: n each)."""
    view: Callable[[torch.Tensor], torch.Tensor]
    where: Callable[[int], str]
    sizes: torch.Tensor | None = None


@dataclass
class Local:
    worst: float          # largest e_g
    where: str            # its group
    second: float         # next-largest e_g
    second_where: str
    elem: float           # largest elem_g
    elem_where: str
    whole: float          # whole-tensor rel-L2, the old single-number check


def rows(n_rows: int, label: str = "row") -> Groups:
    return Groups(lambda t: t.reshape(n_rows, -1), lambda g: f"{label} {g}")


def balanced_rows(S: int) -> int:
    """Rows per owned tile of the attention kernels: ceil(S / 64) tiles of equal height (attention_tc.cu balanced_tiles)."""
    return -(-S // -(-S // 64))


def attn_rows(B: int, nh: int, S: int, hd: int) -> Groups:
    """[B * S, nh * hd] token-major attention operand -> one group per (b, h, row); the owned tile is the 64-row-box CTA
    whose kept rows include `row` (q rows for O / dQ, kv rows for dK / dV)."""
    R = balanced_rows(S)

    def view(t):
        return t.reshape(B, S, nh, hd).permute(0, 2, 1, 3).reshape(B * nh * S, hd)

    def where(g):
        b, h, r = g // (nh * S), (g // S) % nh, g % S
        return f"(b {b}, h {h}, row {r}, owned tile {r // R} of {R} rows)"

    return Groups(view, where)


def gemm_rows(M: int, N: int, BM: int = 128) -> Groups:
    return Groups(lambda t: t[:, :N].reshape(M, N), lambda g: f"(m tile {g // BM}, all n tiles, row {g})")


def gemm_tiles(M: int, N: int, BN: int, BM: int = 128) -> Groups:
    """One group per BM x BN output tile; the ragged M / N tails are zero-padded in both tensors (adding nothing)."""
    nm, nn = -(-M // BM), -(-N // BN)

    def view(t):
        p = t.new_zeros(nm * BM, nn * BN)
        p[:M, :N] = t[:, :N]
        return p.reshape(nm, BM, nn, BN).permute(0, 2, 1, 3).reshape(nm * nn, BM * BN)

    sizes = (torch.arange(nm)[:, None] * BM).neg().add(M).clamp(max=BM) * \
        (torch.arange(nn)[None] * BN).neg().add(N).clamp(max=BN)
    return Groups(view, lambda g: f"(m tile {g // nn}, n tile {g % nn}, rows {g // nn * BM}..{min(M, g // nn * BM + BM) - 1})",
                  sizes.reshape(-1).double())


def conv_bn(Cout: int) -> int:
    """N tile of the tensor-core convolution (conv_tc.cu): 256, 128 or 16 output channels."""
    return 256 if Cout >= 256 else (128 if Cout > 16 else 16)


def conv_tile_pixels(t: torch.Tensor, up: bool = False) -> torch.Tensor:
    """NHWC [B, H, W, C] -> [B, parities, tiles, 128, C]: the pixels of each 128-pixel tile of the tensor-core convolution,
    tile_w = min(W, 128) wide and 128 / tile_w high, in the kernel's tile order.  up: the tiles are taken per parity
    (py, px) on the H/2 x W/2 grid, parity = 2 py + px (the layout of the upsample statistics)."""
    B, H, W, C = t.shape
    if up:
        H, W = H // 2, W // 2
        t = t.reshape(B, H, 2, W, 2, C).permute(0, 2, 4, 1, 3, 5).reshape(B * 4, H, W, C)
    tw = min(W, 128)
    th = 128 // tw
    t = t.reshape(-1, H // th, th, W // tw, tw, C).permute(0, 1, 3, 2, 4, 5)
    return t.reshape(B, 4 if up else 1, (H // th) * (W // tw), 128, C)


def conv_tiles(B: int, H: int, W: int, Cout: int, up: bool = False) -> Groups:
    """NHWC output [B, H, W, Cout] of the tensor-core convolution -> one group per (image, parity, pixel tile, n tile).
    The ragged last n tile is zero-padded in both tensors."""
    BN = conv_bn(Cout)
    nn = -(-Cout // BN)
    h, w = (H // 2, W // 2) if up else (H, W)
    tw = min(w, 128)
    th = 128 // tw
    tiles = (h // th) * (w // tw)
    P = 4 if up else 1

    def view(t):
        p = conv_tile_pixels(t, up)
        if nn * BN != Cout:
            p = torch.cat([p, p.new_zeros(*p.shape[:-1], nn * BN - Cout)], -1)
        return p.reshape(B, P, tiles, 128, nn, BN).permute(0, 1, 2, 4, 3, 5).reshape(-1, 128 * BN)

    def where(g):
        n, rest = g % nn, g // nn
        tt, rest = rest % tiles, rest // tiles
        par, img = rest % P, rest // P
        y0, x0 = (tt // (w // tw)) * th, (tt % (w // tw)) * tw
        return f"(image {img}, parity {par}, tile y0 {y0} x0 {x0}, n tile {n})" if up else \
            f"(image {img}, tile y0 {y0} x0 {x0}, n tile {n})"

    sizes = torch.tensor([128.0 * min(BN, Cout - n * BN) for n in range(nn)], dtype=torch.float64).repeat(B * P * tiles)
    return Groups(view, where, sizes)


def gn_groups(B: int, HW: int, C: int, G: int) -> Groups:
    """NHWC [B, HW, C] -> one group per (image, GroupNorm group)."""
    cpg = C // G
    return Groups(lambda t: t.reshape(B, HW, G, cpg).permute(0, 2, 1, 3).reshape(B * G, HW * cpg),
                  lambda g: f"(image {g // G}, group {g % G})")


def check_local(out, ref, groups: Groups, bound: float, elem_bound: float, what: str) -> Local:
    d = groups.view(out.detach().double()) - groups.view(ref.detach().double())
    r = groups.view(ref.detach().double())
    n = torch.full((r.shape[0],), float(r.shape[1]), dtype=r.dtype) if groups.sizes is None else groups.sizes
    nrm = r.norm(dim=1)
    floor = max(float(nrm.median()) / 16, 1e-300)
    den = nrm.clamp_min(floor)
    e = torch.nan_to_num(d.norm(dim=1) / den, nan=math.inf)
    el = torch.nan_to_num(d.abs().amax(dim=1) / (den / n.to(den.device).sqrt()), nan=math.inf)
    top = torch.topk(e, min(2, e.numel()))
    gi = [int(i) for i in top.indices]
    ei = int(el.argmax())
    whole = float(d.norm() / r.norm().clamp_min(1e-300))
    res = Local(float(top.values[0]), groups.where(gi[0]), float(top.values[-1]) if len(gi) > 1 else 0.0,
                groups.where(gi[-1]) if len(gi) > 1 else "-", float(el[ei]), groups.where(ei), whole)
    msg = (f"{what}: worst group error {res.worst:.3e} at {res.where} (bound {bound:.1e}); next worst {res.second:.3e} "
           f"at {res.second_where}; worst elementwise {res.elem:.3e} at {res.elem_where} (bound {elem_bound:.1e}); "
           f"whole-tensor rel-L2 {res.whole:.3e}")
    assert res.worst <= bound and res.elem <= elem_bound, msg
    return res


def check_abs(out, ref, where: Callable[[int], str], bound: float, what: str) -> Local:
    """one value per row (a log-sum-exp, a row's loss): the largest absolute error and its row"""
    d = torch.nan_to_num((out.detach().double() - ref.detach().double()).abs().reshape(-1), nan=math.inf)
    top = torch.topk(d, min(2, d.numel()))
    gi = [int(i) for i in top.indices]
    whole = float(d.norm() / ref.detach().double().norm().clamp_min(1e-300))
    res = Local(float(top.values[0]), where(gi[0]), float(top.values[-1]), where(gi[-1]), float(top.values[0]),
                where(gi[0]), whole)
    assert res.worst <= bound, (f"{what}: worst absolute error {res.worst:.3e} at {res.where} (bound {bound:.1e}); "
                                f"next worst {res.second:.3e} at {res.second_where}; whole-tensor rel-L2 {whole:.3e}")
    return res


# ------------------------------------------------------------------------------------------------ element-wise fp32 kernels
ULP32 = 2.0 ** -24  # unit roundoff of fp32


def check_ulps(out, ref, terms, group, where: Callable[[int], str], bound: float, what: str) -> Local:
    """Element-wise kernels (no reduction): the error of each element in fp32 units of its own terms,
    |out - ref| / (2^-24 * terms), where `terms` is the sum of the magnitudes of what the kernel adds up for that element.
    A whole-tensor rel-L2 of an updated parameter is dominated by the unchanged part and hides a wrong update; this does
    not.  An element whose terms are all zero must be exact.  group: int64 id per element (a kernel block); the failure
    names the group with the largest error."""
    d = (out.detach().double() - ref.detach().double()).abs()
    den = terms.detach().double() * ULP32
    e = torch.where(d == 0, torch.zeros_like(d), d / den)  # d != 0 over zero terms: inf
    e = torch.nan_to_num(e, nan=math.inf)
    n = int(group.max()) + 1
    per = torch.zeros(n, dtype=e.dtype, device=e.device).scatter_reduce_(0, group, e, "amax", include_self=True)
    top = torch.topk(per, min(2, n))
    gi = [int(i) for i in top.indices]
    whole = float(d.norm() / ref.detach().double().norm().clamp_min(1e-300))
    res = Local(float(top.values[0]), where(gi[0]), float(top.values[-1]) if n > 1 else 0.0,
                where(gi[-1]) if n > 1 else "-", float(top.values[0]), where(gi[0]), whole)
    assert res.worst <= bound, (f"{what}: worst element {res.worst:.2f} ulps of its terms at {res.where} (bound {bound}); "
                                f"next worst group {res.second:.2f} at {res.second_where}; whole-tensor rel-L2 {whole:.3e}")
    return res


@dataclass
class AdamHyper:
    """what the kernel receives, as fp64 values of its fp32 arguments; inv_bc1 / inv_sqrt_bc2 / omd in fp64 from the
    formulas (omd = 1 - EMA decay, None: no EMA update this step)"""
    lr: float
    beta1: float
    beta2: float
    eps: float
    weight_decay: float
    step: int
    omd: float | None

    @property
    def inv_bc1(self):
        return 1.0 / (1.0 - self.beta1 ** self.step)

    @property
    def inv_sqrt_bc2(self):
        return 1.0 / math.sqrt(1.0 - self.beta2 ** self.step)


def f32(x: float) -> float:
    return float(torch.tensor(x, dtype=torch.float32))


def adamw_ref(p, g, m, v, h: AdamHyper):
    """fp64 AdamW of csrc/optim.cu from fp32 operands: {name: (reference, terms)} for p, m, v (terms for check_ulps)"""
    p, g, m, v = (t.double() for t in (p, g, m, v))
    c1, c2 = 1.0 - h.beta1, 1.0 - h.beta2
    wd = h.lr * h.weight_decay * p
    m1 = m + c1 * (g - m)
    m1_terms = m.abs() + c1 * (g - m).abs()
    v1 = h.beta2 * v + c2 * g * g
    den = v1.sqrt() * h.inv_sqrt_bc2 + h.eps
    step = h.lr * h.inv_bc1
    p1 = p - wd - step * m1 / den
    return {"p": (p1, p.abs() + wd.abs() + step * m1_terms / den), "m": (m1, m1_terms), "v": (v1, v1)}


def ema_ref(s, p_new, omd: float):
    """fp64 EMA step s - (1 - decay) (s - p') from the kernel's own updated p' (its error is measured on its own)"""
    s, p_new = s.double(), p_new.double()
    return s - omd * (s - p_new), s.abs() + omd * (s - p_new).abs()


# ------------------------------------------------------------------------------------------------ cross-entropy forward
def ce_inputs(rows: int, V: int, ld: int, seed: int):
    """fp32 logits [rows, ld] (bf16-exact, zero pad columns) and int64 labels: random rows plus the special ones -- a
    dominant +60 logit (labelled elsewhere / on the label), an all-equal row, labels at columns 0 and V - 1, a dominant
    logit in the scalar-tail column V - 1, ignored rows"""
    g = torch.Generator().manual_seed(seed)
    logits = torch.zeros(rows, ld)
    logits[:, :V] = torch.randn(rows, V, generator=g) * 2
    labels = torch.randint(0, V, (rows,), generator=g)
    labels[torch.rand(rows, generator=g) < 0.3] = -100
    labels[0], labels[1], labels[rows - 1] = 0, V - 1, V - 1
    logits[2, 5], labels[2] = 60.0, 7          # one +60 logit, labelled elsewhere
    logits[3, 9], labels[3] = 60.0, 9          # one +60 logit on the label
    logits[4, :V], labels[4] = 1.5, 11         # all-equal row
    logits[5, V - 1], labels[5] = 12.0, 3      # dominant logit in the last column
    labels[6] = labels[rows - 2] = -100
    return logits.to(torch.bfloat16).float(), labels


def ce_fwd_ref(logits, labels, V: int, ls: float):
    """fp64 (lse, row loss) of the label-smoothed cross-entropy per row; ignored rows have loss 0"""
    x = logits[:, :V].double()
    lse = torch.logsumexp(x, -1)
    valid = labels != -100
    zy = x.gather(1, labels.clamp_min(0)[:, None])[:, 0]
    loss = (1 - ls) * (lse - zy) + ls * (lse - x.mean(-1))
    return lse, torch.where(valid, loss, torch.zeros_like(loss))


# (group bound, elementwise bound) per kernel output; the comment gives the worst group / elementwise error measured on
# an H100 SXM (700 W) over all cases of tests/test_kernel_local_gpu.py.
BOUNDS = {
    # attention (ops.attn_fwd / attn_bwd), bf16 outputs
    "attn.o": (1e-2, 4e-2),        # 4.87e-3 / 1.84e-2
    "attn.dq": (1e-2, 4e-2),       # 4.86e-3 / 1.87e-2
    "attn.dk": (1.4e-2, 5e-2),     # 6.59e-3 / 2.19e-2
    "attn.dv": (1e-2, 4e-2),       # 4.85e-3 / 1.78e-2
    # GEMM epilogues
    "gemm.bf16": (5e-3, 7e-2),     # 2.16e-3 / 3.05e-2 (an element of the 2^3 column tile in a row of 2^-4 .. 2^3 tiles)
    "gemm.f32": (6e-7, 4e-6),      # 2.68e-7 / 1.89e-6
    "gemm.resadd": (4e-3, 2e-2),   # 1.69e-3 / 7.89e-3
    "gemm.splitk": (6e-7, 4e-6),   # 2.68e-7 / 1.89e-6
    "gemm.atomic": (4e-7, 4e-6),   # 1.90e-7 / 1.62e-6
    # row norms; a row with one element 1e3 x the others puts that element at 64 x the row's rms
    "norm.y_bf16": (5e-3, 3e-1),   # 2.27e-3 / 1.45e-1
    "norm.dx": (3e-5, 4e-5),       # 1.38e-5 / 1.52e-5
    "norm.dw": (2e-4, 2e-4),       # 8.46e-5 / 8.46e-5
    "norm2.dx2": (3e-7, 1.5e-6),   # 1.09e-7 / 6.36e-7
    "norm2.da": (4e-3, 3e-2),      # 1.94e-3 / 1.36e-2
    "norm2.dw": (1.5e-5, 1.5e-5),  # 7.18e-6 / 7.18e-6
    "glu_norm.y": (5e-3, 1.5e-1),  # 2.05e-3 / 6.23e-2
    "glu_norm.dab": (5e-3, 1.5e-1),  # 2.04e-3 / 5.83e-2
    "glu_norm.dw": (3e-5, 3e-5),   # 1.34e-5 / 1.34e-5
    # cross-entropy; a row dominated by one +60 logit has its gradient in two elements
    "ce.dlogits": (8e-3, 4e-1),    # 3.60e-3 / 1.62e-1
    # U-ViT
    "anm.y": (5e-3, 3e-2),         # 2.31e-3 / 1.34e-2
    "anm.da_bf16": (5e-3, 3e-2),   # 2.19e-3 / 1.24e-2
    "anm.da_f32": (3e-7, 1.5e-6),  # 1.17e-7 / 6.77e-7
    "anm.dw": (2e-5, 2e-5),        # 8.49e-6 / 8.49e-6
    "anm.dmod": (4e-7, 1.5e-6),    # 1.54e-7 / 5.65e-7
    "dwconv.y": (5e-3, 4e-2),      # 2.03e-3 / 1.55e-2
    "dwconv.dx": (3e-5, 6e-4),     # 1.37e-5 / 2.68e-4
    "dwconv.dwk": (4e-6, 8e-5),    # 1.89e-6 / 3.39e-5
    "dwconv.dnw": (6e-3, 6e-3),    # 2.55e-3 / 2.55e-3 (from the bf16 conv output the kernel saves)
    "grn.out": (6e-3, 4e-2),       # 2.51e-3 / 1.56e-2
    "grn.dx": (5e-3, 5e-2),        # 2.25e-3 / 2.13e-2
    "grn.dgamma": (1.2e-4, 1.2e-4),  # 5.20e-5 / 5.20e-5
    "grn.dbeta": (8e-7, 8e-7),     # 3.18e-7 / 3.18e-7
    # tokenizer kernels (tests/test_tokenizer_local_gpu.py, same H100 SXM at 700 W), fp32 outputs against fp64 of the
    # exact fp32 operands
    "conv.bf16x3": (3.2e-5, 8e-4),   # 1.55e-5 / 3.98e-4
    "conv.bf16": (5e-3, 7e-2),       # 2.38e-3 / 3.44e-2 (single-pass bf16 mode)
    "conv.stats_sum": (2e-7, 1e-6),  # 9.12e-8 / 4.83e-7 (epilogue statistics against fp64 sums of the y written)
    "conv.stats_m2": (3e-7, 2.5e-6),  # 1.51e-7 / 1.20e-6
    "conv.simt": (6e-7, 1.2e-5),     # 2.61e-7 / 5.91e-6
    "attn1.out": (3e-5, 3e-4),       # 1.50e-5 / 1.39e-4
    "softmax.split": (1e-5, 3e-4),   # 4.97e-6 / 1.48e-4 (hi + lo: representation error 2^-18)
    "softmax.f32": (3e-7, 4e-6),     # 1.46e-7 / 2.03e-6
    # fused AdamW + EMA step (tests/test_optim_local_gpu.py, same H100 SXM at 700 W): worst element error in fp32 ulps
    # of its own terms (check_ulps), the same number for the group and the element
    "adamw.p": (10.0, 10.0),       # 4.91
    "adamw.m": (4.0, 4.0),         # 1.80
    "adamw.v": (6.0, 6.0),         # 2.82
    "adamw.ema": (5.0, 5.0),       # 2.48
    # cross-entropy forward per row (tests/test_kernel_local_gpu.py): absolute error of the row's log-sum-exp and loss
    # (natural-log units); relative error of the mean and of the row_scale-weighted sum
    "ce.lse": (1.5e-6, 1.5e-6),    # 7.47e-7
    "ce.loss": (4e-6, 4e-6),       # 2.01e-6 (the +60 logit row)
    "ce.mean": (2.5e-7, 2.5e-7),   # 1.03e-7
}
ATTN_LSE_ABS = 4e-5  # max |lse - lse_ref| in natural-log units; measured 1.53e-5
