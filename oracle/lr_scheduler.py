"""f32 numpy restatement of neuronika-optim's learning-rate schedulers (lr_scheduler/mod.rs:34-79 and
{step_lr,multi_step_lr,exponential_lr,multiplicative_lr,lambda_lr}/mod.rs), independent of the product.

`Lr` stands for the optimizer's lr (a np.float32).  Each scheduler's step() follows prepare_step (mod.rs:66-79) and then
its rule, applied to the optimizer's current lr so that chained schedulers compose (mod.rs:16-17; SURVEY.md 8-c defect
10 -- the reference's code scales a private copy instead, which gives the same values for a single scheduler)."""
from __future__ import annotations

import numpy as np

f32 = np.float32


class Lr:
    def __init__(self, lr):
        self.lr = f32(lr)


class Scheduler:
    def __init__(self, opt: Lr):
        self.opt = opt
        self.epoch = 0
        self.last_lr = f32(0.0)
        self.current_lr = f32(opt.lr)
        self.initial_lr = f32(opt.lr)

    def factor(self, t):
        raise NotImplementedError

    def step(self):
        t = self.epoch + 1
        lr = f32(self.opt.lr)
        f = self.factor(t)
        self.epoch, self.last_lr = t, lr
        if f is not None:
            base = self.initial_lr if isinstance(self, LambdaLR) else lr
            self.opt.lr = f32(base * f32(f))
        self.current_lr = f32(self.opt.lr)

    def get_last_lr(self):
        return self.last_lr

    def get_current_lr(self):
        return self.current_lr

    def get_current_epoch(self):
        return self.epoch

    def set_current_epoch(self, epoch):
        self.epoch = int(epoch)


class StepLR(Scheduler):
    def __init__(self, opt, step_size, gamma):
        if step_size < 1:
            raise ValueError("step_size must be >= 1")
        super().__init__(opt)
        self.step_size, self.gamma = int(step_size), f32(gamma)

    def factor(self, t):
        return self.gamma if t % self.step_size == 0 else None


class MultiStepLR(Scheduler):
    def __init__(self, opt, milestones, gamma):
        super().__init__(opt)
        self.milestones, self.gamma = [int(m) for m in milestones], f32(gamma)

    def factor(self, t):
        return self.gamma if t in self.milestones else None


class ExponentialLR(Scheduler):
    def __init__(self, opt, gamma):
        super().__init__(opt)
        self.gamma = f32(gamma)

    def factor(self, t):
        return self.gamma


class MultiplicativeLR(Scheduler):
    def __init__(self, opt, lr_fn):
        super().__init__(opt)
        self.lr_fn = lr_fn

    def factor(self, t):
        return f32(self.lr_fn(t))


class LambdaLR(MultiplicativeLR):
    pass
