"""GPU: the 8-bit AdamW pass (csrc/optim.cu muse_adamw8bit_ema_step) per tensor and per block against fp64, past its first
launch chunk and with guard zones around every buffer; FusedAdamW8bit's 32-bit path against FusedAdamW bit for bit; CUDA
graph replays against eager steps bit for bit; and U-ViT training against FusedAdamW.  CPU twin:
tests/test_adamw8bit_cpu.py, whose fp64 verifier this file runs on the kernel's output."""
import numpy as np
import pytest
import torch

from open_muse_b200 import EMAModel, FusedAdamW, FusedAdamW8bit, MaskGitTransformer, MaskGiTUViT_v2, ops
from open_muse_b200.optim import MIN_8BIT_SIZE, QBLOCK, _maps_buffer
from tests.local_error import BOUNDS, AdamHyper, adamw_ref, check_ulps, ema_ref, f32
from tests import test_adamw8bit_cpu as cpu8
from tests.test_adamw8bit_cpu import verify

pytestmark = pytest.mark.gpu
DEV = "cuda"
KOPT = 48  # table entries per launch (kOptChunk, csrc/optim.cu)
NUMELS = [4, 4092, 4096, 4100, 4352, 2 ** 18 + 4, 2 ** 20]
GUARD = 1024
SENT32, SENT8 = 0x7FBADBAD, 0xA5


class Buf:
    """one guarded buffer per operand: [guard][entry 0][guard][entry 1]...[guard], sentinel bits in the guards"""

    def __init__(self, sizes, dtype):
        self.off, pos = [], GUARD
        for k in sizes:
            self.off.append(pos)
            pos += k + GUARD
        bits = {torch.float32: (torch.int32, SENT32), torch.bfloat16: (torch.int16, 0x7FAB), torch.uint8: (torch.uint8, SENT8)}
        self.view_dtype, sent = bits[dtype]
        self.t = torch.empty(pos, dtype=dtype, device=DEV)
        self.t.view(self.view_dtype).fill_(sent)
        self.sizes = sizes

    def __getitem__(self, i):
        return self.t[self.off[i]:self.off[i] + self.sizes[i]]

    def ptr(self, i):
        return self.t.data_ptr() + self.off[i] * self.t.element_size()

    def outside(self, mask_of):
        """bool mask over the buffer: True where nothing may change (guards, and entries mask_of(i) says are untouched)"""
        m = torch.ones(self.t.numel(), dtype=torch.bool, device=DEV)
        for i, (o, k) in enumerate(zip(self.off, self.sizes)):
            m[o:o + k] = not mask_of(i)
        return m


# (n_entries, step before the call, EMA on, lr on the host or the device)
CASES = [(1, 0, False, "host"), (7, 3, True, "dev"), (47, 1, True, "host"), (48, 9, False, "dev"), (49, 99, True, "host"),
         (97, 9, True, "dev"), (145, 0, True, "host")]


@pytest.mark.parametrize("n,step0,ema_on,lr_mode", CASES)
def test_adamw8bit_step_per_block(n, step0, ema_on, lr_mode):
    numel = [NUMELS[(i + n) % len(NUMELS)] for i in range(n)]
    q8 = [k >= MIN_8BIT_SIZE for k in numel]
    nblk = [-(-k // QBLOCK) if b else 1 for k, b in zip(numel, q8)]
    has_ema = [ema_on and i % 2 == 0 for i in range(n)]
    has_packed = [(i // 2) % 2 == 0 for i in range(n)]
    gen = torch.Generator(device=DEV).manual_seed(100 + n)
    P, G, S, K = (Buf(numel, d) for d in (torch.float32, torch.float32, torch.float32, torch.bfloat16))
    C1, C2 = Buf(numel, torch.uint8), Buf(numel, torch.uint8)
    A1, A2 = Buf(nblk, torch.float32), Buf(nblk, torch.float32)
    M32, V32 = Buf(numel, torch.float32), Buf(numel, torch.float32)
    for i, k in enumerate(numel):
        scale = 2.0 ** ((i * 7) % 13 - 6)  # a different magnitude per entry
        P[i].copy_(torch.randn(k, device=DEV, generator=gen) * scale)
        G[i].copy_(torch.randn(k, device=DEV, generator=gen) * 1e-3 * scale)
        S[i].copy_(torch.randn(k, device=DEV, generator=gen) * scale)
        if q8[i]:
            C1[i].copy_(torch.randint(0, 256, (k,), device=DEV, generator=gen, dtype=torch.uint8))
            C2[i].copy_(torch.randint(0, 256, (k,), device=DEV, generator=gen, dtype=torch.uint8))
            A1[i].copy_(torch.rand(nblk[i], device=DEV, generator=gen) * 1e-3 * scale)
            A2[i].copy_(torch.rand(nblk[i], device=DEV, generator=gen) * 1e-6 * scale * scale)
            C1[i][:QBLOCK], C2[i][:QBLOCK], A1[i][0], A2[i][0] = 0, 0, 0.0, 0.0  # a fresh first block
        else:
            M32[i].copy_(torch.randn(k, device=DEV, generator=gen) * 1e-3 * scale)
            V32[i].copy_((torch.randn(k, device=DEV, generator=gen) * 1e-3 * scale) ** 2)
    bufs = [P, G, C1, C2, A1, A2, S, K, M32, V32]
    before = [b.t.clone() for b in bufs]
    ins = [[b[i].clone() for b in (P, G, C1, C2, A1, A2)] for i in range(n)]
    ins32 = [[b[i].clone() for b in (P, G, M32, V32)] for i in range(n)]
    table = np.zeros((n, 10), dtype=np.int64)
    for i in range(n):
        m, v = (C1.ptr(i), C2.ptr(i)) if q8[i] else (M32.ptr(i), V32.ptr(i))
        table[i] = (P.ptr(i), G.ptr(i), m, v, S.ptr(i) if has_ema[i] else 0, K.ptr(i) if has_packed[i] else 0,
                    numel[i], 0, A1.ptr(i) if q8[i] else 0, A2.ptr(i) if q8[i] else 0)
    beta1, beta2, eps, wd = f32(0.9), f32(0.999) if n % 2 else f32(0.95), f32(1e-8), f32(0.1)
    lr = f32(2e-3)
    lr_dev = torch.tensor([lr], device=DEV) if lr_mode == "dev" else None
    ema_args = (1, f32(0.9999), 0.0, 0, 1, 1, 1.0, f32(2 / 3)) if ema_on else (0, 0.0, 0.0, 0, 1, 0, 1.0, 1.0)
    step_dev = torch.tensor([step0], dtype=torch.int64, device=DEV)
    scal = torch.zeros(8, device=DEV)
    maps = _maps_buffer(DEV)
    ops._call("muse_adamw8bit_ema_step", table.ctypes.data, n, maps.data_ptr(), scal.data_ptr(), step_dev.data_ptr(),
              None if lr_dev is None else lr_dev.data_ptr(), lr if lr_dev is None else 7.0, beta1, beta2, eps, wd,
              *ema_args, ops._prep(scal))
    torch.cuda.synchronize()
    case = f"(entries {n}, step {step0} -> {step0 + 1}, EMA {ema_on}, lr on the {lr_mode})"
    assert int(step_dev) == step0 + 1, case
    s = step0 + 1
    omd = float(scal[4]) if ema_on else None

    # guards, untouched entries' buffers and g: bit-unchanged
    rules = {0: lambda i: True, 1: lambda i: False, 2: lambda i: q8[i], 3: lambda i: q8[i], 4: lambda i: q8[i],
             5: lambda i: q8[i], 6: lambda i: has_ema[i], 7: lambda i: has_packed[i], 8: lambda i: not q8[i],
             9: lambda i: not q8[i]}
    for k, (b, b0) in enumerate(zip(bufs, before)):
        keep = b.outside(rules[k])
        changed = (b.t.view(b.view_dtype) != b0.view(b.view_dtype)) & keep
        assert not bool(changed.any()), f"{case}: buffer {k} changed outside what the table lets the kernel write, first " \
                                        f"at element {int(changed.nonzero()[0])}"

    ah = AdamHyper(lr, beta1, beta2, eps, wd, s, None)
    where = lambda e: f"launch {e // KOPT}, entry {e % KOPT}, numel {numel[e]}"  # noqa: E731
    idx8 = [i for i in range(n) if q8[i]]
    if idx8:
        outs = [[b[i] for b in (P, G, C1, C2, A1, A2)] for i in idx8]
        near, worst = verify([ins[i] for i in idx8], outs, ah, where=lambda j: where(idx8[j]))
        print(f"\n{case}: {len(idx8)} 8-bit entries, {near} codes within 4 ulps of a midpoint (either neighbour "
              f"accepted); worst absmax1 {worst[0]:.2f}, absmax2 {worst[1]:.2f} ulps of the terms")
    for i in range(n):
        blk = torch.arange(numel[i], device=DEV) // 1024
        at = lambda b, i=i: f"({where(i)}, block {b})"  # noqa: E731
        if not q8[i]:
            ref = adamw_ref(*ins32[i], ah)
            for key, out in (("p", P[i]), ("m", M32[i]), ("v", V32[i])):
                check_ulps(out, *ref[key], blk, at, BOUNDS[f"adamw.{key}"][0], f"32-bit {key} {case}")
        if has_ema[i] and omd is not None and omd >= 0:
            sref, terms = ema_ref(before[6][S.off[i]:S.off[i] + numel[i]], P[i], omd)
            check_ulps(S[i], sref, terms, blk, at, BOUNDS["adamw.ema"][0], f"shadow {case}")
        if has_packed[i]:
            assert torch.equal(K[i].view(torch.int16), P[i].to(torch.bfloat16).view(torch.int16)), f"bf16 operand {case}"


def test_kernel_sends_exact_ties_to_the_lower_code():
    """the CPU verifier's fixture through the kernel: one block per tensor has every x exactly on a midpoint of the signed
    map (1 - beta1 = 1/8 makes m = g / 8 exact, and the block's absmax is 1), one block starts fresh; the kernel's codes
    must take the lower code at every tie, and everything else must pass the same checks as the restatement"""
    ops_in = [[t.to(DEV) for t in e] for e in cpu8.make_operands()]
    out = [[t.clone() for t in e] for e in ops_in]
    n = len(out)
    table = np.zeros((n, 10), dtype=np.int64)
    for i, (p, g, c1, c2, a1, a2) in enumerate(out):
        table[i] = (p.data_ptr(), g.data_ptr(), c1.data_ptr(), c2.data_ptr(), 0, 0, p.numel(), 0, a1.data_ptr(),
                    a2.data_ptr())
    step_dev = torch.tensor([cpu8.STEP - 1], dtype=torch.int64, device=DEV)
    scal = torch.zeros(8, device=DEV)
    maps = _maps_buffer(DEV)
    ops._call("muse_adamw8bit_ema_step", table.ctypes.data, n, maps.data_ptr(), scal.data_ptr(), step_dev.data_ptr(),
              None, cpu8.LR, cpu8.B1, cpu8.B2, cpu8.EPS, cpu8.WD, 0, 0.0, 0.0, 0, 1, 0, 1.0, 1.0, ops._prep(scal))
    torch.cuda.synchronize()
    mid1 = maps[512:767]
    ties = sum(int(torch.isin(e[1] / 8, mid1).sum()) for e in ops_in)
    assert ties >= 4 * 255
    near, worst = verify(ops_in, out)
    print(f"\n{ties} exact ties, {near} codes within 4 ulps of a midpoint; worst absmax {worst[0]:.2f} / {worst[1]:.2f}")


# ------------------------------------------------------------------------------------------------ 32-bit path = FusedAdamW
TINY_V1 = dict(vocab_size=72, hidden_size=48, num_hidden_layers=1, num_attention_heads=1, intermediate_size=64,
               hidden_dropout=0.0, attention_dropout=0.0, max_position_embeddings=16)


@pytest.mark.parametrize("tensor_lr", [False, True])
def test_small_tensors_step_exactly_like_fused_adamw(tensor_lr):
    """a MaskGitTransformer whose tensors all lie below 4096 elements: FusedAdamW8bit and FusedAdamW give bit-identical
    parameters, moments, EMA shadows and bf16 operands over 12 steps"""
    torch.manual_seed(0)
    a = MaskGitTransformer(**TINY_V1).to(DEV)
    b = MaskGitTransformer(**TINY_V1).to(DEV)
    b.load_state_dict(a.state_dict())
    assert max(p.numel() for p in a.parameters()) < MIN_8BIT_SIZE
    lr = (lambda: torch.tensor([2e-3], device=DEV)) if tensor_lr else (lambda: 2e-3)
    ea, eb = EMAModel(list(a.parameters()), decay=0.999), EMAModel(list(b.parameters()), decay=0.999)
    oa = FusedAdamW(a.parameters(), lr=lr(), weight_decay=0.05, ema=ea, model=a)
    ob = FusedAdamW8bit(b.parameters(), lr=lr(), weight_decay=0.05, ema=eb, model=b)
    gen = torch.Generator(device=DEV).manual_seed(1)
    for step in range(12):
        for pa, pb in zip(a.parameters(), b.parameters()):
            pa.grad = torch.randn(pa.shape, device=DEV, generator=gen) * 1e-2
            pb.grad = pa.grad.clone()
        oa.step(), ob.step()
    torch.cuda.synchronize()
    for (n, pa), pb, sa, sb in zip(a.named_parameters(), b.parameters(), ea.shadow_params, eb.shadow_params):
        assert torch.equal(pa, pb), n
        assert torch.equal(oa.state[pa]["exp_avg"], ob.state[pb]["exp_avg"]), n
        assert torch.equal(oa.state[pa]["exp_avg_sq"], ob.state[pb]["exp_avg_sq"]), n
        assert torch.equal(sa, sb), n
    assert torch.equal(a._packed.refresh().flat, b._packed.refresh().flat)
    assert int(ob.state[next(b.parameters())]["step"]) == 12


# ------------------------------------------------------------------------------------------------ CUDA graph
V1 = dict(vocab_size=72, hidden_size=64, num_hidden_layers=1, num_attention_heads=1, intermediate_size=128,
          hidden_dropout=0.0, attention_dropout=0.0, max_position_embeddings=16)


def test_graph_replays_equal_eager_steps():
    """one eager step, then a captured step replayed 4 times, against 5 eager steps: codes, absmax, p, shadows, bf16
    operands and the step counter bit for bit"""
    torch.manual_seed(0)
    models = [MaskGitTransformer(**V1).to(DEV) for _ in range(2)]
    models[1].load_state_dict(models[0].state_dict())
    gen = torch.Generator(device=DEV).manual_seed(2)
    grads = [torch.randn(p.shape, device=DEV, generator=gen) * 1e-2 for p in models[0].parameters()]
    opts, emas = [], []
    for m in models:
        for p, g in zip(m.parameters(), grads):
            p.grad = g.clone()
        emas.append(EMAModel(list(m.parameters()), decay=0.99, use_ema_warmup=True))
        opts.append(FusedAdamW8bit(m.parameters(), lr=torch.tensor([1e-2], device=DEV), weight_decay=0.05, ema=emas[-1],
                                   model=m))
    assert {p.numel() >= MIN_8BIT_SIZE for p in models[0].parameters()} == {True, False}
    for _ in range(5):
        opts[0].step()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        opts[1].step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        opts[1].step()
    for _ in range(4):
        graph.replay()
    torch.cuda.synchronize()
    for (n, pa), pb in zip(models[0].named_parameters(), models[1].parameters()):
        assert torch.equal(pa, pb), n
        sa, sb = opts[0].state[pa], opts[1].state[pb]
        assert sa.keys() == sb.keys()
        for k in sa:
            assert torch.equal(sa[k], sb[k]), (n, k)
    assert int(opts[1].state[next(models[1].parameters())]["step"]) == 5
    for sa, sb in zip(emas[0].shadow_params, emas[1].shadow_params):
        assert torch.equal(sa, sb)
    assert torch.equal(models[0]._packed.refresh().flat, models[1]._packed.refresh().flat)


# ------------------------------------------------------------------------------------------------ training
UVIT_ARGS = ("input_ids", "encoder_hidden_states", "cond_embeds", "micro_conds")


def test_uvit_training_tracks_fused_adamw(golden):
    """200 steps of the micro U-ViT fixture on its fixed batch, with ema= and model=: the 8-bit run's final loss within 5 %
    of FusedAdamW's"""
    g = golden("micro_uvit_v2.pt")
    args = [g[k].to(DEV) for k in UVIT_ARGS]
    labels = g["labels"].to(DEV)
    curves = {}
    for cls in (FusedAdamW, FusedAdamW8bit):
        m = MaskGiTUViT_v2(**g["config"])
        m.load_state_dict(g["state_dict"])
        m.to(DEV).train()
        ema = EMAModel(list(m.parameters()), decay=0.999)
        opt = cls(m.parameters(), lr=1e-3, weight_decay=0.01, ema=ema, model=m)
        losses = []
        for _ in range(200):
            with torch.autocast("cuda", dtype=torch.bfloat16):
                _, loss = m(*args, labels=labels)
            loss.backward()
            opt.step()
            opt.zero_grad(set_to_none=True)
            losses.append(float(loss))
        curves[cls.__name__] = losses
    a, b = curves["FusedAdamW"][-1], curves["FusedAdamW8bit"][-1]
    print("\nloss every 20 steps:\n  FusedAdamW     " + " ".join(f"{x:.4f}" for x in curves["FusedAdamW"][::20])
          + f" final {a:.4f}\n  FusedAdamW8bit " + " ".join(f"{x:.4f}" for x in curves["FusedAdamW8bit"][::20])
          + f" final {b:.4f}")
    assert b < curves["FusedAdamW8bit"][0]
    assert abs(b - a) / a <= 0.05, (a, b)
