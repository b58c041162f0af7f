"""Learning-rate schedulers: the mirror of neuronika-optim's lr_scheduler module (lr_scheduler/mod.rs,
{step_lr,multi_step_lr,exponential_lr,multiplicative_lr,lambda_lr}/mod.rs), used as there:

    optim.step(); optim.zero_grad(); scheduler.step()

Each step() advances the epoch to t = epoch + 1 and, when the scheduler's rule applies, sets the optimizer's lr in f32:

    StepLR            lr * gamma  when t % step_size == 0
    MultiStepLR       lr * gamma  when t is a milestone
    ExponentialLR     lr * gamma
    MultiplicativeLR  lr * lr_fn(t)
    LambdaLR          initial_lr * lr_fn(t)

`lr` is the optimizer's current lr, so chained schedulers compose (the reference's documented intent,
lr_scheduler/mod.rs:16-17; its code scales each scheduler's private copy instead, so with two schedulers the last one
wins -- SURVEY.md 8-c defect 10).  With one scheduler both give the same values.  get_last_lr() is the lr before the
last step and get_current_lr() the lr after it.

On an optim.Optimizer the scheduler's state lives on the device (nk_lr_sched) and step() launches a one-thread kernel
that rewrites the optimizer's device lr, so a captured step advances the schedule on every replay; the other methods
read and write the device state synchronously and raise NkError while capturing.  The device cannot call a Python
closure, so MultiplicativeLR and LambdaLR run there only when given `horizon`: lr_fn(1..horizon) is evaluated into a
device table at construction, and a step past the horizon leaves lr unchanged and makes the next read of the scheduler
raise NkError.  Without `horizon`, or on any other object with get_lr / set_lr, the scheduler runs on the host in
np.float32 and calls set_lr; inside a capture that call raises NkError."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib as L
from .device import F32, CuArray

__all__ = ["StepLR", "MultiStepLR", "ExponentialLR", "MultiplicativeLR", "LambdaLR"]

_f32 = np.float32


class _Scheduler:
    kind = None

    def __init__(self, optimizer, gamma=1.0, step_size=1, milestones=(), lr_fn=None, horizon=None):
        from .optim import Optimizer
        self.optimizer = optimizer
        self._lr_fn = lr_fn
        closure = self.kind in (L.NK_LR_MULTIPLICATIVE, L.NK_LR_LAMBDA)
        self._device = isinstance(optimizer, Optimizer) and (horizon is not None or not closure)
        lr = _f32(optimizer.get_lr())
        # host state (the device copy is the truth in device mode)
        self._epoch, self._gamma, self._step_size = 0, _f32(gamma), int(step_size)
        self._milestones = [int(m) for m in milestones]
        self._last, self._current, self._initial = _f32(0.0), lr, lr
        if not self._device:
            return
        if optimizer.hyper_ptr is None:
            raise L.NkError(-1, "a scheduler needs the optimizer's device block: register the parameters first")
        self._dev = optimizer._hyper.device
        self._block = CuArray(self._dev, (C.sizeof(L.LrSched) // 4,), F32)
        self._table = None
        if closure:
            if int(horizon) < 1:
                raise ValueError("a closure-based scheduler's horizon must be >= 1: lr_fn(1..horizon) is tabulated on "
                                 "the device")
            self._table = CuArray(self._dev, (int(horizon),), F32)
            self._table.copy_from(np.array([_f32(lr_fn(t)) for t in range(1, int(horizon) + 1)], dtype=np.float32))
        elif self.kind == L.NK_LR_MULTI_STEP:
            self._set_table_milestones()
        self._write(self._host_block())

    # ---- device state
    def _set_table_milestones(self):
        m = np.array(self._milestones or [0], dtype=np.int64)
        self._table = CuArray(self._dev, (2 * m.size,), F32)     # int64 entries, 8 bytes each
        L.check(L.lib.nk_h2d(self._dev.ctx, self._table.ptr, m.ctypes.data_as(C.c_void_p), m.nbytes), self._dev.ctx)
        self._dev.synchronize()

    def _table_len(self):
        if self.kind == L.NK_LR_MULTI_STEP:
            return len(self._milestones)
        return self._table.size if self._table is not None else 0

    def _host_block(self) -> L.LrSched:
        return L.LrSched(epoch=self._epoch, step_size=self._step_size,
                         table=self._table.ptr.value if self._table is not None else None, table_len=self._table_len(),
                         gamma=float(self._gamma), initial_lr=float(self._initial), last_lr=float(self._last),
                         current_lr=float(self._current), kind=self.kind, past_horizon=0)

    def _read(self, check=True) -> L.LrSched:
        s = L.LrSched()
        rc = L.lib.nk_lr_sched_get(self._dev.ctx, self._block.ptr, C.byref(s))
        if check or rc != -1:   # NK_ERR_INVALID_ARG: the block is copied even when it reports a step past the horizon
            L.check(rc, self._dev.ctx)
        return s

    def _write(self, s: L.LrSched) -> None:
        L.check(L.lib.nk_lr_sched_set(self._dev.ctx, self._block.ptr, C.byref(s)), self._dev.ctx)

    def _update(self, **fields) -> None:
        """read-modify-write of the device block; a rewrite clears the past-horizon flag"""
        s = self._read(check=False)
        for k, v in fields.items():
            setattr(s, k, v)
        s.past_horizon = 0
        self._write(s)

    # ---- the rule on the host
    def _factor(self, t):
        """the factor of epoch t, or None when the rule does not apply"""
        if self.kind == L.NK_LR_STEP:
            return self._gamma if t % self._step_size == 0 else None
        if self.kind == L.NK_LR_MULTI_STEP:
            return self._gamma if t in self._milestones else None
        if self.kind == L.NK_LR_EXPONENTIAL:
            return self._gamma
        return _f32(self._lr_fn(t))

    # ---- LRScheduler (lr_scheduler/mod.rs:34-63)
    def step(self) -> None:
        if self._device:
            L.check(L.lib.nk_lr_sched_step(self._dev.ctx, self._block.ptr, self.optimizer.hyper_ptr), self._dev.ctx)
            return
        t = self._epoch + 1
        lr = _f32(self.optimizer.get_lr())
        f = self._factor(t)
        nxt = lr if f is None else _f32((self._initial if self.kind == L.NK_LR_LAMBDA else lr) * f)
        self._epoch, self._last, self._current = t, lr, nxt
        if f is not None:
            self.optimizer.set_lr(float(nxt))

    def get_last_lr(self) -> float:
        return float(self._read().last_lr) if self._device else float(self._last)

    def get_current_lr(self) -> float:
        return float(self._read().current_lr) if self._device else float(self._current)

    def get_current_epoch(self) -> int:
        return int(self._read().epoch) if self._device else self._epoch

    def set_current_epoch(self, epoch: int) -> None:
        if int(epoch) < 0:
            raise ValueError(f"epoch must be >= 0, got {epoch}")
        if self._device:
            self._update(epoch=int(epoch))
        else:
            self._epoch = int(epoch)

    def print_lr(self) -> None:
        print(f"epoch {self.get_current_epoch()}: learning rate adjusted to [{self.get_current_lr()}]")


def _check_step_size(step_size):
    if int(step_size) < 1:   # the reference panics in rem_euclid (step_lr/mod.rs:117)
        raise ValueError(f"step_size must be >= 1, got {step_size}")
    return int(step_size)


class StepLR(_Scheduler):
    """`StepLR::new(optimizer, step_size, gamma)` (step_lr/mod.rs:37-48)"""
    kind = L.NK_LR_STEP

    def __init__(self, optimizer, step_size: int, gamma: float):
        super().__init__(optimizer, gamma=gamma, step_size=_check_step_size(step_size))

    def set_gamma(self, gamma: float) -> None:
        self._gamma = _f32(gamma)
        if self._device:
            self._update(gamma=float(self._gamma))

    def set_step_size(self, step_size: int) -> None:
        self._step_size = _check_step_size(step_size)
        if self._device:
            self._update(step_size=self._step_size)


class MultiStepLR(_Scheduler):
    """`MultiStepLR::new(optimizer, milestones, gamma)` (multi_step_lr/mod.rs:37-48)"""
    kind = L.NK_LR_MULTI_STEP

    def __init__(self, optimizer, milestones, gamma: float):
        super().__init__(optimizer, gamma=gamma, milestones=milestones)

    def set_milestones(self, milestones) -> None:
        self._milestones = [int(m) for m in milestones]
        if self._device:
            self._set_table_milestones()
            self._update(table=self._table.ptr.value, table_len=len(self._milestones))


class ExponentialLR(_Scheduler):
    """`ExponentialLR::new(optimizer, gamma)` (exponential_lr/mod.rs:33-43)"""
    kind = L.NK_LR_EXPONENTIAL

    def __init__(self, optimizer, gamma: float):
        super().__init__(optimizer, gamma=gamma)

    def set_gamma(self, gamma: float) -> None:
        self._gamma = _f32(gamma)
        if self._device:
            self._update(gamma=float(self._gamma))


class MultiplicativeLR(_Scheduler):
    """`MultiplicativeLR::new(optimizer, lr_fn)` (multiplicative_lr/mod.rs:35-44); `horizon` as in the module doc"""
    kind = L.NK_LR_MULTIPLICATIVE

    def __init__(self, optimizer, lr_fn, horizon=None):
        super().__init__(optimizer, lr_fn=lr_fn, horizon=horizon)


class LambdaLR(_Scheduler):
    """`LambdaLR::new(optimizer, lr_fn)` (lambda_lr/mod.rs:36-47); `horizon` as in the module doc"""
    kind = L.NK_LR_LAMBDA

    def __init__(self, optimizer, lr_fn, horizon=None):
        super().__init__(optimizer, lr_fn=lr_fn, horizon=horizon)
