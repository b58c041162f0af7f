"""Optimizer registry and optimizers: the mirror of neuronika-optim (optimizer.rs:4-104, sgd/mod.rs:11-236,
adam/mod.rs, amsgrad/mod.rs, rmsprop/mod.rs, adagrad/mod.rs, penalty.rs:2-79).  Optimizer state lives on the device
in f32, and so do lr and the step count (nk_optim_hyper).  step() updates every registered parameter with one fused
multi-tensor launch per 64 tensors of one (data, gradient) dtype pair (nkg_multi_*_step), so a captured step advances
the step count, and sees lr changes, on every replay."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib as L
from . import variable as V
from .device import F32, CuArray


class L2:
    """`L2::penalize(w) = 2*lambda*w` (penalty.rs:63-67)."""

    def __init__(self, lambda_: float = 0.0):
        self.lambda_ = float(lambda_)


class NoPenalty(L2):
    def __init__(self):
        super().__init__(0.0)


class L1:
    """`L1::penalize(w) = lambda*signum(w)` (penalty.rs:69-73)."""

    def __init__(self, lambda_: float):
        self.lambda_ = float(lambda_)


class ElasticNet:
    """`lambda_l1*signum(w) + 2*lambda_l2*w` (penalty.rs:75-79)."""

    def __init__(self, lambda_l1: float, lambda_l2: float):
        self.lambda_l1, self.lambda_l2 = float(lambda_l1), float(lambda_l2)


def _l1_l2(penalty):
    """(l1, l2) coefficients of a penalty object for the fused kernels."""
    if isinstance(penalty, ElasticNet):
        return penalty.lambda_l1, penalty.lambda_l2
    if isinstance(penalty, L1):
        return penalty.lambda_, 0.0
    return 0.0, penalty.lambda_


class Optimizer:
    """`Optimizer<T>`: register / step / zero_grad / get_lr / set_lr (optimizer.rs:33-95).  lr and the step count live
    in a device block that the first register() allocates; step() launches (Adam, AMSGrad, Adagrad) the one-thread
    prologue that advances the step count, then one update launch per 64 tensors per (data, gradient) dtype pair.  Every
    other hyperparameter is a kernel argument: a captured step keeps the values it was captured with.  get_lr / set_lr
    read and write the device block (synchronously; NkError while capturing).  All parameters must be registered before
    the first step, since the step count is shared."""

    def __init__(self, status):
        self.status = status
        self.params = []
        self._hyper = None
        self._stepped = False

    @property
    def hyper_ptr(self):
        """device address of the nk_optim_hyper block (None before the first register)"""
        return self._hyper.ptr if self._hyper is not None else None

    def _read(self) -> L.OptimHyper:
        h = L.OptimHyper()
        dev = self._hyper.device
        L.check(L.lib.nk_optim_hyper_get(dev.ctx, self._hyper.ptr, C.byref(h)), dev.ctx)
        return h

    def _write(self, h: L.OptimHyper) -> None:
        dev = self._hyper.device
        L.check(L.lib.nk_optim_hyper_set(dev.ctx, self._hyper.ptr, C.byref(h)), dev.ctx)

    def get_lr(self) -> float:
        return self.status.lr if self._hyper is None else float(self._read().lr)

    def set_lr(self, lr: float) -> None:
        if self._hyper is None:
            self.status.lr = float(lr)
            return
        h = self._read()
        h.lr = float(lr)
        self._write(h)

    def register(self, variable: V.VarDiff) -> None:
        if self._hyper is None:
            block = CuArray(variable.device, (C.sizeof(L.OptimHyper) // 4,), F32)
            self._hyper = block
            try:
                self._write(L.OptimHyper(lr=self.status.lr))
            except L.NkError:
                self._hyper = None
                raise
        else:
            if variable.device is not self._hyper.device:
                raise L.NkError(-1, "register: an optimizer's parameters share one device")
            self._read()                                  # refused while capturing, like every host access
            if self._stepped:
                raise L.NkError(-1, "register: an optimizer counts steps for all its parameters together; "
                                "register every parameter before the first step()")
        self.params.append(self.status.into_param(variable))

    def step(self) -> None:
        if self.params:
            self.status.multi_step(self.params, self._hyper.ptr)
            self._stepped = True

    def zero_grad(self) -> None:
        for p in self.params:
            p.zero_grad()


def _ptrs(arrays):
    """ctypes array of device pointers (NULL for None), or None when every entry is None"""
    if all(a is None for a in arrays):
        return None
    return (C.c_void_p * len(arrays))(*[a.ptr.value if a is not None else None for a in arrays])


def _handles(params):
    return (C.c_void_p * len(params))(*[p.variable._h.value for p in params])


class _SGDParam:
    """SGDParam (sgd/mod.rs:150-236): momentum buffer created on first use."""

    def __init__(self, variable: V.VarDiff, status: "StochasticGD"):
        self.variable, self.status, self.buffer, self.master = variable, status, None, None
        if status.master_weights and variable.dtype != F32:
            self.master = variable.data_array().astype(F32)

    def prepare(self) -> None:
        s = self.status
        use_mom = s.momentum is not None and s.momentum > np.finfo(np.float32).eps
        if use_mom and self.buffer is None:
            self.buffer = CuArray(self.variable.device, self.variable.shape, F32)
        if not use_mom:
            self.buffer = None

    def zero_grad(self) -> None:
        self.variable.zero_grad()


class StochasticGD:
    """`StochasticGD::new(lr, penalty, momentum, dampening, nesterov) -> Optimizer<Self>` (sgd/mod.rs:43-85),
    same argument validation.  `grad_scale` (1/world_size under data parallel) and `master_weights`
    (f32 master copy of bf16 parameters, kept as optimizer state) are additions."""

    def __init__(self, lr, penalty, momentum, dampening, nesterov, grad_scale=1.0, master_weights=False):
        if momentum is None:
            assert dampening is None and not nesterov, \
                "Dampening and Nesterov momentum flag should be enabled together with momentum."
        if dampening is not None:
            assert 0.0 <= dampening <= 1.0, f"Dampening value should be between 0.0 and 1.0, got: {dampening}"
        self.lr, self.penalty, self.momentum, self.dampening, self.nesterov = float(lr), penalty, momentum, dampening, nesterov
        self.grad_scale, self.master_weights = float(grad_scale), bool(master_weights)

    @staticmethod
    def new(lr, penalty=None, momentum=None, dampening=None, nesterov=False, **kw) -> Optimizer:
        return Optimizer(StochasticGD(lr, penalty or NoPenalty(), momentum, dampening, nesterov, **kw))

    def into_param(self, variable: V.VarDiff) -> _SGDParam:
        return _SGDParam(variable, self)

    def multi_step(self, params, hyper) -> None:
        for p in params:
            p.prepare()
        V._ck(V.lib.nkg_multi_sgd_step(_handles(params), len(params), _ptrs([p.buffer for p in params]),
                                       _ptrs([p.master for p in params]), hyper, float(self.penalty.lambda_),
                                       float(self.momentum or 0.0), float(self.dampening or 0.0),
                                       int(bool(self.nesterov)), float(self.grad_scale)))


# ------------------------------------------------------------------------------------------- Adam family (8-f rank 2)
def _state(variable: V.VarDiff) -> CuArray:
    return CuArray(variable.device, variable.shape, F32)          # zero-filled, like Array::zeros(raw_dim)


class _MasterMixin:
    def _init_master(self, variable, status):
        self.master = None
        if getattr(status, "master_weights", False) and variable.dtype != F32:
            self.master = variable.data_array().astype(F32)


class _AdamParam(_MasterMixin):
    """AdamParam / AMSGradParam (adam/mod.rs:113-175, amsgrad/mod.rs:136-210)."""

    def __init__(self, variable, status):
        self.variable = variable
        self.exp_avg, self.exp_avg_sq = _state(variable), _state(variable)
        self.max_exp_avg_sq = _state(variable) if status.amsgrad else None
        self._init_master(variable, status)

    def zero_grad(self) -> None:
        self.variable.zero_grad()


class Adam:
    """`Adam::new(lr, beta1, beta2, penalty, eps)` (adam/mod.rs:43-60)."""
    amsgrad = False

    def __init__(self, lr, beta1, beta2, penalty, eps, grad_scale=1.0, master_weights=False):
        self.lr, self.beta1, self.beta2, self.penalty, self.eps = float(lr), float(beta1), float(beta2), penalty, float(eps)
        self.grad_scale, self.master_weights = float(grad_scale), bool(master_weights)

    @classmethod
    def new(cls, lr, beta1=0.9, beta2=0.999, penalty=None, eps=1e-8, **kw) -> Optimizer:
        return Optimizer(cls(lr, beta1, beta2, penalty or NoPenalty(), eps, **kw))

    def into_param(self, variable):
        return _AdamParam(variable, self)

    def multi_step(self, params, hyper) -> None:
        l1, l2 = _l1_l2(self.penalty)
        V._ck(V.lib.nkg_multi_adam_step(_handles(params), len(params), _ptrs([p.exp_avg for p in params]),
                                        _ptrs([p.exp_avg_sq for p in params]),
                                        _ptrs([p.max_exp_avg_sq for p in params]), _ptrs([p.master for p in params]),
                                        hyper, float(self.beta1), float(self.beta2), float(self.eps), l1, l2,
                                        float(self.grad_scale)))


class AMSGrad(Adam):
    """`AMSGrad::new(lr, beta1, beta2, penalty, eps)` (amsgrad/mod.rs:45-62)."""
    amsgrad = True


class _RMSPropParam(_MasterMixin):
    """RMSPropParam (rmsprop/mod.rs:150-305): `buffer` / `grad_avg` exist only while momentum / centered are on."""

    def __init__(self, variable, status):
        self.variable, self.status = variable, status
        self.square_avg = _state(variable)
        self.buffer = _state(variable) if status.momentum is not None else None
        self.grad_avg = _state(variable) if status.centered else None
        self._init_master(variable, status)

    def prepare(self) -> None:
        s = self.status
        use_mom = s.momentum is not None and s.momentum > np.finfo(np.float32).eps
        if use_mom and self.buffer is None:
            self.buffer = _state(self.variable)
        if not use_mom:
            self.buffer = None
        if s.centered and self.grad_avg is None:
            self.grad_avg = _state(self.variable)
        if not s.centered:
            self.grad_avg = None

    def zero_grad(self) -> None:
        self.variable.zero_grad()


class RMSProp:
    """`RMSProp::new(lr, penalty, alpha, momentum, centered, eps)` (rmsprop/mod.rs:67-100), same validation."""

    def __init__(self, lr, penalty, alpha, momentum, centered, eps, grad_scale=1.0, master_weights=False):
        if alpha is not None:
            assert 0.0 <= alpha <= 1.0, f"Dampening value should be between 0.0 and 1.0, got: {alpha}"
        self.lr, self.penalty, self.alpha, self.momentum = float(lr), penalty, alpha, momentum
        self.centered, self.eps = bool(centered), float(eps)
        self.grad_scale, self.master_weights = float(grad_scale), bool(master_weights)

    @staticmethod
    def new(lr, penalty=None, alpha=0.99, momentum=None, centered=False, eps=1e-8, **kw) -> Optimizer:
        return Optimizer(RMSProp(lr, penalty or NoPenalty(), alpha, momentum, centered, eps, **kw))

    def into_param(self, variable):
        return _RMSPropParam(variable, self)

    def multi_step(self, params, hyper) -> None:
        for p in params:
            p.prepare()
        l1, l2 = _l1_l2(self.penalty)
        V._ck(V.lib.nkg_multi_rmsprop_step(_handles(params), len(params), _ptrs([p.square_avg for p in params]),
                                           _ptrs([p.grad_avg for p in params]), _ptrs([p.buffer for p in params]),
                                           _ptrs([p.master for p in params]), hyper,
                                           float(self.alpha if self.alpha is not None else 0.0), float(self.eps),
                                           float(self.momentum or 0.0), l1, l2, float(self.grad_scale)))


class _AdagradParam(_MasterMixin):
    """AdagradParam (adagrad/mod.rs:96-145)."""

    def __init__(self, variable, status):
        self.variable = variable
        self.grad_sq = _state(variable)
        self._init_master(variable, status)

    def zero_grad(self) -> None:
        self.variable.zero_grad()


class Adagrad:
    """`Adagrad::new(lr, lr_decay, penalty, eps)` (adagrad/mod.rs:50-63)."""

    def __init__(self, lr, lr_decay, penalty, eps, grad_scale=1.0, master_weights=False):
        self.lr, self.lr_decay, self.penalty, self.eps = float(lr), float(lr_decay), penalty, float(eps)
        self.grad_scale, self.master_weights = float(grad_scale), bool(master_weights)

    @staticmethod
    def new(lr, lr_decay=0.0, penalty=None, eps=1e-10, **kw) -> Optimizer:
        return Optimizer(Adagrad(lr, lr_decay, penalty or NoPenalty(), eps, **kw))

    def into_param(self, variable):
        return _AdagradParam(variable, self)

    def multi_step(self, params, hyper) -> None:
        l1, l2 = _l1_l2(self.penalty)
        V._ck(V.lib.nkg_multi_adagrad_step(_handles(params), len(params), _ptrs([p.grad_sq for p in params]),
                                           _ptrs([p.master for p in params]), hyper, float(self.lr_decay),
                                           float(self.eps), l1, l2, float(self.grad_scale)))


# ------------------------------------------------------------------------------------------- gradient clipping
# torch.nn.utils' clipping functions over the gradients of VarDiff parameters, on the device's stream: one multi-tensor
# launch per 64 gradients of one dtype (nkg_grad_norm / nkg_clip_grads_with_norm / nkg_clip_grad_value), nothing read
# back to the host unless error_if_nonfinite.  `grad_scale` is the optimizer's (1/world under data parallel): the norm
# is that of grad_scale * g, and the coefficient multiplies the raw buffers.
def _grad_params(params):
    return [params] if isinstance(params, V.VarDiff) else list(params)


def _var_handles(ps):
    return (C.c_void_p * len(ps))(*[p._h.value for p in ps])


def get_total_norm(params, norm_type=2.0, error_if_nonfinite=False, grad_scale=1.0) -> CuArray:
    """The norm of all the gradients together as one vector (a 0-d f32 CuArray on the device; reading it is the
    caller's sync).  norm_type > 0 or inf.  With error_if_nonfinite the total is read back, which a capture refuses."""
    ps = _grad_params(params)
    if not ps:
        raise ValueError("get_total_norm: no parameters, so no device to hold the total")
    dev = ps[0].device
    if error_if_nonfinite and dev.capturing:
        raise L.NkError(-5, "get_total_norm: error_if_nonfinite reads the total back, which a captured step could not "
                            "repeat on replay")
    total = CuArray(dev, (), F32)
    V._ck(V.lib.nkg_grad_norm(_var_handles(ps), len(ps), float(norm_type), float(grad_scale), total.ptr))
    if error_if_nonfinite and not np.isfinite(total.as_ndarray()):
        raise RuntimeError(
            f"The total norm of order {float(norm_type)} for gradients from `parameters` is non-finite, so it cannot be "
            "clipped. To disable this error and scale the gradients by the non-finite norm anyway, set "
            "`error_if_nonfinite=False`")
    return total


def clip_grads_with_norm_(params, max_norm, total_norm: CuArray) -> None:
    """grad *= min(max_norm / (total_norm + 1e-6), 1), with total_norm a 0-d f32 CuArray on the device."""
    ps = _grad_params(params)
    if total_norm.dtype != F32 or total_norm.size != 1:
        raise ValueError("clip_grads_with_norm_: total_norm must be one f32 element")
    V._ck(V.lib.nkg_clip_grads_with_norm(_var_handles(ps), len(ps), float(max_norm), total_norm.ptr))


def clip_grad_norm_(params, max_norm, norm_type=2.0, error_if_nonfinite=False, grad_scale=1.0) -> CuArray:
    """get_total_norm, then clip_grads_with_norm_; returns the total.  Inside a capture the total lives in the graph's
    arena and every replay rewrites it."""
    ps = _grad_params(params)
    total = get_total_norm(ps, norm_type, error_if_nonfinite, grad_scale)
    clip_grads_with_norm_(ps, max_norm, total)
    return total


def clip_grad_value_(params, clip_value, grad_scale=1.0) -> None:
    """grad = clamp(grad, -b, b) with b = clip_value / grad_scale (in f32)."""
    ps = _grad_params(params)
    V._ck(V.lib.nkg_clip_grad_value(_var_handles(ps), len(ps), float(clip_value), float(grad_scale)))


from . import lr_scheduler  # noqa: E402  (optim.lr_scheduler, as in the reference)
