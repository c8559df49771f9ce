"""``FusedAdamW``: AdamW + EMA + bf16 operand packing as ONE pass over the parameters (SURVEY.md 8f-4).

Reference: the training scripts step ``torch.optim.AdamW`` / apex ``FusedAdam`` (training/train_maskgit_imagenet.py:
242-261,438; train_muse.py:427-452 with name-based no-decay groups) and then ``ema.step(model.parameters())``
(train_muse.py:761-762; muse/modeling_ema.py:108-126), and autocast re-casts every Linear weight to bf16 on the next
forward.  Here one kernel reads p, g, m, v (and the EMA shadow) once and writes p, m, v, the shadow and the packed bf16
GEMM operand.  A ``torch.optim.Optimizer`` subclass, so LR schedulers, ``state_dict`` / ``load_state_dict``,
``zero_grad`` and ``accelerate`` treat it like AdamW.  CUDA-graph capturable (step counter and per-step scalars live on
the device).

``FusedLion`` is the reference's ``training/optimizer.py::Lion`` (the scripts' ``optimizer.name: lion``; one moment instead
of two) on the same machinery, and ``FusedAdamW8bit`` is AdamW with block-wise 8-bit moments (train_muse.py's
``optimizer.name: 8bit_adamw``).  All three keep a model's bf16 operand cache current (see ``_FusedOptimizer``)."""
from __future__ import annotations

from typing import Optional

import torch

from . import _lib, ops


def _check_lr(lr, device=None, who="FusedAdamW"):
    """the kernel reads a tensor learning rate as ONE fp32 value at a device address: a host tensor would hand it a host
    address, another dtype the wrong bits"""
    if torch.is_tensor(lr) and (lr.numel() != 1 or lr.dtype != torch.float32 or (device is not None and lr.device != device)):
        raise ValueError(f"{who}: a tensor lr must be a one-element float32 tensor on the parameters' device"
                         f"{'' if device is None else ' ' + str(device)}; got {lr.numel()} element(s) of {lr.dtype} "
                         f"on {lr.device}")


class _FusedOptimizer(torch.optim.Optimizer):
    """The launch plan, EMA wiring and operand-cache protocol shared by ``FusedAdamW``, ``FusedLion`` and
    ``FusedAdamW8bit``.

    A subclass names its per-parameter moment buffers (``_moments``: the table's m and v slots; or overrides
    ``_state_columns`` for another layout) and launches its kernel in ``_launch``.  The kernels write parameters through
    raw pointers, which autograd does not see, so after every step the written parameters' version counters are bumped:
    a model's operand cache keyed on ``(data_ptr, _version)`` then rebuilds on its next forward.  With ``model=`` the
    step also writes the bf16 operands itself: ``model._packed`` provides ``refresh()`` (bring the cache up to date;
    returns an object whose ``dst_of`` maps a parameter's data_ptr to its bf16 copy) and ``sync()`` (after the step:
    refresh the few operands that are not a plain copy of one parameter and move the cache's key to the new versions),
    so no re-pack follows the step."""

    _moments = ()

    def __init__(self, params, defaults, ema, model):
        super().__init__(params, defaults)
        self.ema, self.model = ema, model
        self._plans = {}
        if ema is not None:
            flat = [p for g in self.param_groups for p in g["params"]]
            if len(flat) != len(ema.shadow_params) or any(p.shape != s.shape for p, s in zip(flat, ema.shadow_params)):
                raise ValueError(f"{type(self).__name__}(ema=...): the EMAModel must be built over the same parameter list")

    def _state_columns(self, p):
        """the table's m and v addresses for p and the columns that follow its fixed eight (none here), creating its moment
        buffers on first use"""
        st = self.state[p]
        for k in self._moments:
            if k not in st:
                st[k] = torch.zeros_like(p, memory_format=torch.preserve_format)
        m, v = (st[k].data_ptr() for k in self._moments) if len(self._moments) == 2 else (st[self._moments[0]].data_ptr(), 0)
        return m, v, ()

    # ---- per-group launch plan (device table), rebuilt when pointers change (new grads storage, .to(device), ...)
    def _packed_cache(self):
        m = self.model
        return None if m is None or not hasattr(m, "_packed") else m._packed

    def _packed_dst(self, cache):
        """parameter data_ptr -> address of its bf16 copy in the model's packed operand cache (host-side bookkeeping kept
        by the cache itself: no device read, so this is legal during graph capture)."""
        if cache is None:
            return {}
        pk = cache.refresh()
        return dict(getattr(pk, "dst_of", {}) or {})

    def _plan(self, gi, group, shadow_of, packed_dst):
        name = type(self).__name__
        params = [p for p in group["params"] if p.grad is not None]
        # every address the kernel writes through is part of the key: EMAModel.load_state_dict / .to replace the shadow
        # tensors while parameters and gradients stay where they are
        key = tuple((p.data_ptr(), p.grad.data_ptr(), 0 if shadow_of.get(id(p)) is None else shadow_of[id(p)].data_ptr(),
                     packed_dst.get(p.data_ptr(), 0)) for p in params)
        plan = self._plans.get(gi)
        if plan is not None and plan["key"] == key:
            return plan
        entries = []
        dev = params[0].device
        for p, (_, _, sh_ptr, packed_ptr) in zip(params, key):
            if p.dtype != torch.float32 or p.grad.dtype != torch.float32 or not p.is_contiguous() or not p.grad.is_contiguous() \
                    or p.numel() % 4 != 0 or p.grad.is_sparse:
                raise RuntimeError(f"{name} needs contiguous fp32 parameters / gradients with numel % 4 == 0")
            sh = shadow_of.get(id(p))
            if sh is not None and (sh.dtype != torch.float32 or sh.device != p.device or sh.shape != p.shape
                                   or not sh.is_contiguous()):
                raise RuntimeError(f"{name}(ema=...) needs contiguous fp32 EMA shadows shaped and placed like the parameters")
            m, v, extra = self._state_columns(p)
            entries.append((p.data_ptr(), p.grad.data_ptr(), m, v, sh_ptr, packed_ptr, p.numel(), 0, *extra))
        plan = self._plans.get(gi) or {}
        if "step" not in plan:
            # one device-resident step counter per group, shared by the group's parameters' state entries so that
            # state_dict() / load_state_dict() carry it (a freshly loaded state brings its own copy per parameter; a
            # state without one -- e.g. the reference Lion's -- starts at 0)
            loaded = self.state[params[0]].get("step")
            step = loaded.to(device=dev, dtype=torch.int64).reshape(1).clone() if torch.is_tensor(loaded) else \
                torch.zeros(1, dtype=torch.int64, device=dev)
            for p in params:
                self.state[p]["step"] = step
            plan["step"] = step
            plan["scal"] = torch.zeros(8, dtype=torch.float32, device=dev)
        # host-side table (passed to the kernels as launch arguments by the library): numpy keeps the buffer alive
        import numpy as np

        plan.update(key=key, table=np.ascontiguousarray(np.array(entries, dtype=np.int64)), n=len(entries), params=params)
        self._plans[gi] = plan
        return plan

    @staticmethod
    def _ema_args(ema):
        """(enabled, decay, min_decay, update_after_step, update_every, use_warmup, inv_gamma, power) of the kernels"""
        if ema is None:
            return 0, 0.0, 0.0, 0, 1, 0, 1.0, 1.0
        return (1, float(ema.decay), float(ema.min_decay), int(ema.update_after_step), int(ema.update_every),
                1 if ema.use_ema_warmup else 0, float(ema.inv_gamma), float(ema.power))

    def _launch(self, plan, group, lr_dev, ema_args, stream):
        raise NotImplementedError

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        ema = self.ema
        shadow_of = {}
        if ema is not None:
            flat = [p for g in self.param_groups for p in g["params"]]
            shadow_of = {id(p): s for p, s in zip(flat, ema.shadow_params)}
        cache = self._packed_cache()
        packed_dst = self._packed_dst(cache)
        live = [(gi, group) for gi, group in enumerate(self.param_groups) if any(p.grad is not None for p in group["params"])]
        for _, group in live:  # every group before the first launch (a scheduler may have assigned any tensor)
            _check_lr(group["lr"], next(p.device for p in group["params"] if p.grad is not None), type(self).__name__)
        ema_args = self._ema_args(ema)
        written = []
        for gi, group in live:
            plan = self._plan(gi, group, shadow_of, packed_dst)
            lr = group["lr"]
            self._launch(plan, group, lr if torch.is_tensor(lr) else None, ema_args, ops._prep(plan["scal"]))
            written += plan["params"]
        if written:
            torch.autograd.graph.increment_version(written)
            if cache is not None:
                cache.sync()
        if ema is not None:  # host mirror of the device-side schedule (state_dict / logging), same rule as EMAModel.step
            ema.optimization_step += 1
            if (ema.optimization_step - 1) % ema.update_every == 0:
                ema.cur_decay_value = ema.get_decay(ema.optimization_step)
        return loss


class FusedAdamW(_FusedOptimizer):
    _moments = ("exp_avg", "exp_avg_sq")

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, ema=None, model=None):
        """ema: an ``open_muse_b200.EMAModel`` built over the SAME parameter list (its shadow params are updated in the fused
        pass; do not also call ``ema.step``).  model: a ``MaskGitTransformer`` or ``MaskGiTUViT_v2`` whose bf16 operand
        cache receives the updated weights directly (saves the re-pack of the next forward).

        lr: a Python number, or (for a CUDA-graph-capturable schedule) a one-element float32 tensor on the parameters'
        device, read by the kernel at every step; ``step`` raises ValueError for any other tensor.

        Every parameter of the groups is expected to have a gradient at every step, as in the training scripts.  A parameter
        without one is left out of that step's pass: its EMA shadow does not move (``EMAModel.step`` would move it toward
        the parameter), and its bias correction follows its group's step counter, which a group without any gradient does
        not advance."""
        _check_lr(lr)
        if lr < 0 or eps < 0 or not 0 <= betas[0] < 1 or not 0 <= betas[1] < 1 or weight_decay < 0:
            raise ValueError("invalid AdamW hyper-parameters")
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay), ema, model)

    def _launch(self, plan, group, lr_dev, ema_args, stream):
        b1, b2 = group["betas"]
        ops._call("muse_adamw_ema_step", plan["table"].ctypes.data, plan["n"], plan["scal"].data_ptr(),
                  plan["step"].data_ptr(), None if lr_dev is None else lr_dev.data_ptr(),
                  0.0 if lr_dev is not None else float(group["lr"]), float(b1), float(b2), float(group["eps"]),
                  float(group["weight_decay"]), *ema_args, stream)


class FusedLion(_FusedOptimizer):
    _moments = ("exp_avg",)

    def __init__(self, params, lr=1e-4, betas=(0.9, 0.99), weight_decay=0.0, ema=None, model=None, **kwargs):
        """Lion (training/optimizer.py::Lion) + EMA + bf16 operand copy in one pass; ``ema`` / ``model`` / a tensor ``lr``
        as in ``FusedAdamW``.  Other keywords (the training script passes ``eps`` to every optimizer class) are accepted
        and ignored, as the reference does.

        With a Python-number lr, parameters and ``exp_avg`` equal the reference's on the same GPU bit for bit
        (``1 - lr * weight_decay``, ``1 - beta1`` and ``1 - beta2`` are formed in double as the reference's Python
        scalars are).  With a tensor lr, ``1 - lr * weight_decay`` is formed in fp32 on the device.  The state of each
        parameter is ``exp_avg`` (loads into the reference ``Lion`` and back) plus the group's device-resident ``step``
        (the EMA schedule's counter; 0 when a reference state without one is loaded)."""
        _check_lr(lr, who="FusedLion")
        if not 0.0 <= lr:
            raise ValueError(f"FusedLion: invalid learning rate {lr}")
        for i in (0, 1):
            if not 0.0 <= betas[i] < 1.0:
                raise ValueError(f"FusedLion: invalid beta parameter at index {i}: {betas[i]}")
        super().__init__(params, dict(lr=lr, betas=betas, weight_decay=weight_decay), ema, model)

    def _launch(self, plan, group, lr_dev, ema_args, stream):
        b1, b2 = group["betas"]
        lr, wd = group["lr"], float(group["weight_decay"])
        ops._call("muse_lion_ema_step", plan["table"].ctypes.data, plan["n"], plan["scal"].data_ptr(),
                  plan["step"].data_ptr(), None if lr_dev is None else lr_dev.data_ptr(),
                  0.0 if lr_dev is not None else float(lr), 1.0 if lr_dev is not None else 1.0 - float(lr) * wd,
                  float(b1), float(b2), 1.0 - float(b1), 1.0 - float(b2), wd, *ema_args, stream)


MIN_8BIT_SIZE = 4096  # parameters with fewer elements keep fp32 moments (bitsandbytes' min_8bit_size)
QBLOCK = 256          # elements per quantisation block (one fp32 absmax each)


def dynamic_map(signed: bool) -> torch.Tensor:
    """The 256-entry dynamic quantisation map of the 8-bit moments, built in fp32 on the CPU: for each decade 10^-6 ..
    10^0, the midpoints of an evenly spaced grid over [0.1, 1] scaled into it (and their negatives when signed), plus 0
    and 1, sorted.  Signed (m): zero at index 127, 1.0 last; unsigned (v): zero at index 0."""
    data = []
    for i in range(7):
        n = 2 ** i + 1 if signed else 2 ** (i + 1) + 1
        b = torch.linspace(0.1, 1, n)
        means = (b[:-1] + b[1:]) / 2.0
        data += ((10 ** (-6 + i)) * means).tolist()
        if signed:
            data += (-(10 ** (-6 + i)) * means).tolist()
    data += [0.0, 1.0]
    return torch.tensor(sorted(data), dtype=torch.float32)


def midpoints(q: torch.Tensor) -> torch.Tensor:
    """the 255 fp32 decision boundaries (q[k] + q[k + 1]) / 2 of a map: a value x encodes to #{k : M[k] < x}"""
    return (q[:-1] + q[1:]) / 2


BUCKETS, BUCKET_BASE, START_BYTES = 769, 103 << 5, 784  # the encoder's first guess (csrc/optim.cu kBuckets, ...)


def bucket_starts(mid: torch.Tensor, negative: bool) -> torch.Tensor:
    """per bucket of |x| (its fp32 bits >> 18, less the bits of 2^-24 >> 18, clamped to [0, 768]), a code no larger than
    that of any x of the bucket: #{k : mid[k] < lowest x}.  For x >= 0 the lowest x is the bucket's lower bound (0 for
    bucket 0); for x < 0 it lies above minus the bucket's upper bound (no bound for the last bucket)."""
    b = torch.arange(BUCKETS, dtype=torch.int32)
    lo = ((b + BUCKET_BASE) << 18).view(torch.float32).clone()
    lo[0] = 0.0
    if not negative:
        return torch.searchsorted(mid, lo, side="left")
    hi = torch.cat([lo[1:], torch.tensor([float("inf")])])
    return torch.searchsorted(mid, -hi, side="left")


def _maps_buffer(device) -> torch.Tensor:
    """what the kernel stages in shared memory: [Q1 | Q2 | M1 | M2] (both maps and their midpoints, each padded to 256
    entries), then the encoder's start-code tables as bytes (signed map for x >= 0 and for x < 0, unsigned map), each
    padded to START_BYTES"""
    q1, q2 = dynamic_map(True), dynamic_map(False)
    m1, m2 = midpoints(q1), midpoints(q2)
    pad = torch.tensor([float("inf")])  # never read
    tables = torch.zeros(3, START_BYTES, dtype=torch.uint8)
    for row, (mid, neg) in enumerate(((m1, False), (m1, True), (m2, False))):
        tables[row, :BUCKETS] = bucket_starts(mid, neg).to(torch.uint8)
    return torch.cat([q1, q2, m1, pad, m2, pad, tables.reshape(-1).view(torch.float32)]).to(device)


class FusedAdamW8bit(_FusedOptimizer):
    """AdamW with block-wise 8-bit moments (the scheme of bitsandbytes' ``AdamW8bit``; train_muse.py's ``optimizer.name:
    8bit_adamw``) + EMA + bf16 operand packing in one pass.

    A parameter with at least ``MIN_8BIT_SIZE`` elements keeps its moments as uint8 codes shaped like it (``state1``: m
    against the signed ``dynamic_map``, ``state2``: v against the unsigned one) plus one fp32 absmax per 256-element block
    (``absmax1`` / ``absmax2``; blocks start at the tensor's first element, the last may be partial).  A step decodes
    ``Q[code] * absmax``, applies ``FusedAdamW``'s element update (decay before the Adam step, as torch ``AdamW``; the
    parameter takes the un-requantised moments), sets each block's absmax to max |m| / max v and re-encodes to the
    nearest map entry (ties to the lower code).  Smaller parameters keep fp32 ``exp_avg`` / ``exp_avg_sq`` and are
    updated exactly as ``FusedAdamW`` updates them.  Every state also holds its group's device-resident ``step``.  The
    moments then take about 2 B per parameter instead of 8.  Bit-parity with bitsandbytes is not claimed; it applies
    decay after the step."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, ema=None, model=None):
        """``lr`` (a number or a one-element fp32 device tensor), ``ema`` and ``model`` as in ``FusedAdamW``."""
        _check_lr(lr, who="FusedAdamW8bit")
        if lr < 0 or eps < 0 or not 0 <= betas[0] < 1 or not 0 <= betas[1] < 1 or weight_decay < 0:
            raise ValueError("invalid AdamW hyper-parameters")
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay), ema, model)
        self._maps = {}

    @staticmethod
    def _layout(p):
        """state key -> (dtype, shape) of p's moments"""
        if p.numel() < MIN_8BIT_SIZE:
            return {"exp_avg": (torch.float32, p.shape), "exp_avg_sq": (torch.float32, p.shape)}
        nblk = -(-p.numel() // QBLOCK)
        return {"state1": (torch.uint8, p.shape), "state2": (torch.uint8, p.shape),
                "absmax1": (torch.float32, torch.Size([nblk])), "absmax2": (torch.float32, torch.Size([nblk]))}

    def _init_state(self, p):
        st = self.state[p]
        for k, (dtype, shape) in self._layout(p).items():
            if k not in st:
                st[k] = torch.zeros(shape, dtype=dtype, device=p.device)
        return st

    def _state_columns(self, p):
        st = self._init_state(p)
        if p.numel() < MIN_8BIT_SIZE:
            return st["exp_avg"].data_ptr(), st["exp_avg_sq"].data_ptr(), (0, 0)
        return st["state1"].data_ptr(), st["state2"].data_ptr(), (st["absmax1"].data_ptr(), st["absmax2"].data_ptr())

    def load_state_dict(self, state_dict):
        """checks every parameter's saved moments against the layout its size calls for before loading (the kernel reads
        the buffers through raw pointers of the layout's dtypes), and keeps the codes uint8 and every buffer dense"""
        saved = [i for g in state_dict["param_groups"] for i in g["params"]]
        params = [p for g in self.param_groups for p in g["params"]]
        if len(saved) != len(params):
            raise ValueError(f"FusedAdamW8bit.load_state_dict: the state has {len(saved)} parameters, the optimizer "
                             f"{len(params)}")
        for n, (i, p) in enumerate(zip(saved, params)):
            st = state_dict["state"].get(i)
            if st is None:
                continue
            want = self._layout(p)
            have = {k for k in st if k != "step"}
            if have and have != set(want):
                raise ValueError(f"FusedAdamW8bit.load_state_dict: parameter {n} ({p.numel()} elements) needs the state "
                                 f"{sorted(want)}, the loaded state has {sorted(have)}")
            for k in have:
                t, (dtype, shape) = st[k], want[k]
                if not torch.is_tensor(t) or t.dtype != dtype or t.shape != shape:
                    got = f"{t.dtype} {tuple(t.shape)}" if torch.is_tensor(t) else type(t).__name__
                    raise ValueError(f"FusedAdamW8bit.load_state_dict: parameter {n} state {k!r} must be {dtype} "
                                     f"{tuple(shape)}, got {got}")
        super().load_state_dict(state_dict)
        for p in params:
            # torch casts loaded state to the parameter's dtype (the codes go back to uint8, exactly) and keeps its strides;
            # the kernel walks every buffer as a dense array in logical order
            st = self.state.get(p, {})
            for k, (dtype, _) in self._layout(p).items():
                if k in st:
                    st[k] = st[k].to(dtype).contiguous()
        self._plans = {}  # the next step builds its tables over the loaded buffers and step counters

    def _launch(self, plan, group, lr_dev, ema_args, stream):
        dev = plan["params"][0].device
        if dev not in self._maps:
            self._maps[dev] = _maps_buffer(dev)
        b1, b2 = group["betas"]
        ops._call("muse_adamw8bit_ema_step", plan["table"].ctypes.data, plan["n"], self._maps[dev].data_ptr(),
                  plan["scal"].data_ptr(), plan["step"].data_ptr(), None if lr_dev is None else lr_dev.data_ptr(),
                  0.0 if lr_dev is not None else float(group["lr"]), float(b1), float(b2), float(group["eps"]),
                  float(group["weight_decay"]), *ema_args, stream)
