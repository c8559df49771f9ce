"""``FusedAdamW``: AdamW + EMA + bf16 operand packing as ONE pass over the parameters (SURVEY.md 8f-4).

Reference: the training scripts step ``torch.optim.AdamW`` / apex ``FusedAdam`` (training/train_maskgit_imagenet.py:
242-261,438; train_muse.py:427-452 with name-based no-decay groups) and then ``ema.step(model.parameters())``
(train_muse.py:761-762; muse/modeling_ema.py:108-126), and autocast re-casts every Linear weight to bf16 on the next
forward.  Here one kernel reads p, g, m, v (and the EMA shadow) once and writes p, m, v, the shadow and the packed bf16
GEMM operand.  A ``torch.optim.Optimizer`` subclass, so LR schedulers, ``state_dict`` / ``load_state_dict``,
``zero_grad`` and ``accelerate`` treat it like AdamW.  CUDA-graph capturable (step counter and per-step scalars live on
the device)."""
from __future__ import annotations

from typing import Optional

import torch

from . import _lib, ops


def _check_lr(lr, device=None):
    """the kernel reads a tensor learning rate as ONE fp32 value at a device address: a host tensor would hand it a host
    address, another dtype the wrong bits"""
    if torch.is_tensor(lr) and (lr.numel() != 1 or lr.dtype != torch.float32 or (device is not None and lr.device != device)):
        raise ValueError(f"FusedAdamW: a tensor lr must be a one-element float32 tensor on the parameters' device"
                         f"{'' if device is None else ' ' + str(device)}; got {lr.numel()} element(s) of {lr.dtype} "
                         f"on {lr.device}")


class FusedAdamW(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, ema=None, model=None):
        """ema: an ``open_muse_b200.EMAModel`` built over the SAME parameter list (its shadow params are updated in the fused
        pass; do not also call ``ema.step``).  model: a ``MaskGitTransformer`` whose packed bf16 operand cache receives
        the updated weights directly (saves the re-pack launch of the next forward).

        lr: a Python number, or (for a CUDA-graph-capturable schedule) a one-element float32 tensor on the parameters'
        device, read by the kernel at every step; ``step`` raises ValueError for any other tensor.

        Every parameter of the groups is expected to have a gradient at every step, as in the training scripts.  A parameter
        without one is left out of that step's pass: its EMA shadow does not move (``EMAModel.step`` would move it toward
        the parameter), and its bias correction follows its group's step counter, which a group without any gradient does
        not advance."""
        _check_lr(lr)
        if lr < 0 or eps < 0 or not 0 <= betas[0] < 1 or not 0 <= betas[1] < 1 or weight_decay < 0:
            raise ValueError("invalid AdamW hyper-parameters")
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        self.ema, self.model = ema, model
        self._plans = {}
        if ema is not None:
            flat = [p for g in self.param_groups for p in g["params"]]
            if len(flat) != len(ema.shadow_params) or any(p.shape != s.shape for p, s in zip(flat, ema.shadow_params)):
                raise ValueError("FusedAdamW(ema=...): the EMAModel must be built over the same parameter list")

    # ---- per-group launch plan (device table), rebuilt when pointers change (new grads storage, .to(device), ...)
    def _packed_dst(self):
        """parameter data_ptr -> address of its bf16 copy in the model's packed operand cache (host-side bookkeeping kept
        by the cache itself: no device read, so this is legal during graph capture)."""
        m = self.model
        if m is None or not hasattr(m, "_packed"):
            return {}
        pk = m._packed.refresh()
        return dict(getattr(pk, "dst_of", {}) or {})

    def _plan(self, gi, group, shadow_of, packed_dst):
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
                raise RuntimeError("FusedAdamW needs contiguous fp32 parameters / gradients with numel % 4 == 0")
            sh = shadow_of.get(id(p))
            if sh is not None and (sh.dtype != torch.float32 or sh.device != p.device or sh.shape != p.shape
                                   or not sh.is_contiguous()):
                raise RuntimeError("FusedAdamW(ema=...) needs contiguous fp32 EMA shadows shaped and placed like the parameters")
            st = self.state[p]
            if not st:
                st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
            entries.append((p.data_ptr(), p.grad.data_ptr(), st["exp_avg"].data_ptr(), st["exp_avg_sq"].data_ptr(),
                            sh_ptr, packed_ptr, p.numel(), 0))
        plan = self._plans.get(gi) or {}
        if "step" not in plan:
            # one device-resident step counter per group, shared by the group's parameters' state entries so that
            # state_dict() / load_state_dict() carry it (a freshly loaded state brings its own copy per parameter)
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
        packed_dst = self._packed_dst()
        live = [(gi, group) for gi, group in enumerate(self.param_groups) if any(p.grad is not None for p in group["params"])]
        for _, group in live:  # every group before the first launch (a scheduler may have assigned any tensor)
            _check_lr(group["lr"], next(p.device for p in group["params"] if p.grad is not None))
        for gi, group in live:
            plan = self._plan(gi, group, shadow_of, packed_dst)
            lr = group["lr"]
            lr_dev = lr if torch.is_tensor(lr) else None
            st = ops._prep(plan["scal"])
            b1, b2 = group["betas"]
            ops._call("muse_adamw_ema_step", plan["table"].ctypes.data, plan["n"], plan["scal"].data_ptr(),
                      plan["step"].data_ptr(), None if lr_dev is None else lr_dev.data_ptr(),
                      0.0 if lr_dev is not None else float(lr), float(b1), float(b2), float(group["eps"]),
                      float(group["weight_decay"]), 1 if ema is not None else 0,
                      float(ema.decay) if ema is not None else 0.0, float(ema.min_decay) if ema is not None else 0.0,
                      int(ema.update_after_step) if ema is not None else 0, int(ema.update_every) if ema is not None else 1,
                      1 if (ema is not None and ema.use_ema_warmup) else 0, float(ema.inv_gamma) if ema is not None else 1.0,
                      float(ema.power) if ema is not None else 1.0, st)
        if ema is not None:  # host mirror of the device-side schedule (state_dict / logging), same rule as EMAModel.step
            ema.optimization_step += 1
            if (ema.optimization_step - 1) % ema.update_every == 0:
                ema.cur_decay_value = ema.get_decay(ema.optimization_step)
        return loss
