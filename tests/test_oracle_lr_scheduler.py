"""The learning-rate scheduler oracle (oracle/lr_scheduler.py) against the reference's five scheduler tests
(tests/golden/lr_scheduler.json, transcribed from neuronika-optim/src/lr_scheduler/*/test.rs), chaining against the
composed product, and the package's host-side schedulers (the mode a closure scheduler without `horizon` runs in)
against the oracle on a stub optimizer.  No GPU needed."""
import json
import os
import re

import numpy as np
import pytest

from oracle import lr_scheduler as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lr_scheduler.json")
with open(GOLDEN) as fh:
    CASES = json.load(fh)


def oracle_from_golden(case, opt):
    """the scheduler of a reference test, built from the constructor arguments as the test wrote them"""
    args = case["args"]
    cls = getattr(O, case["scheduler"])
    if case["scheduler"] in ("MultiplicativeLR", "LambdaLR"):
        assert args.strip() == "|epoch| epoch as f32"
        return cls(opt, lambda epoch: float(epoch))
    if case["scheduler"] == "MultiStepLR":
        ms, gamma = re.fullmatch(r"vec!\[([\d,\s]*)\],\s*([\d.]+)", args.strip()).groups()
        return cls(opt, [int(m) for m in ms.split(",")], float(gamma))
    nums = [float(v) for v in args.split(",")]
    return cls(opt, int(nums[0]), nums[1]) if case["scheduler"] == "StepLR" else cls(opt, nums[0])


def loop_value(expr, epoch):
    m = re.fullmatch(r"(\d+)_f32\.powi\(epoch as i32\)", expr)
    if m:
        return float(int(m.group(1)) ** epoch)
    assert expr == "epoch as f32", expr
    return float(epoch)


def run_reference_test(case, make):
    """the reference test's loop over any scheduler implementation; make(lr) -> (scheduler, optimizer)"""
    sched, _ = make(case["optimizer_lr"])
    for e in case["set_current_epoch"]:
        sched.set_current_epoch(e)
        assert sched.get_current_epoch() == e
    eps = np.finfo(np.float32).eps
    in_loop = [a for a in case["asserts"] if a["in_loop"]]
    for epoch in range(case["epochs"]):
        for a in in_loop:
            if a["guard"] is None or eval(a["guard"], {"epoch": epoch}):
                assert abs(sched.get_current_lr() - loop_value(a["expr"], epoch)) <= eps, (a["line"], epoch)
        assert sched.get_current_epoch() == epoch
        sched.step()
    for a in case["asserts"]:
        if not a["in_loop"]:
            got = sched.get_last_lr() if a["which"] == "last" else sched.get_current_lr()
            assert abs(got - a["value"]) <= eps, a["line"]


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_reproduces_the_reference_test(name):
    case = CASES[name]

    def make(lr):
        opt = O.Lr(lr)
        return oracle_from_golden(case, opt), opt
    run_reference_test(case, make)


def test_chained_schedulers_compose():
    """each scheduler scales the optimizer's current lr: two chained schedulers give the product of both rules"""
    opt = O.Lr(0.5)
    a, b = O.StepLR(opt, 2, 0.5), O.ExponentialLR(opt, 0.9)
    want = np.float32(0.5)
    for t in range(1, 8):
        a.step()
        b.step()
        if t % 2 == 0:
            want = np.float32(want * np.float32(0.5))
        want = np.float32(want * np.float32(0.9))
        assert opt.lr == want and b.current_lr == want and a.epoch == b.epoch == t


def test_lambda_stays_absolute_when_chained():
    opt = O.Lr(2.0)
    lam, exp = O.LambdaLR(opt, lambda t: 1.0 / t), O.ExponentialLR(opt, 0.5)
    for t in range(1, 5):
        lam.step()
        assert opt.lr == np.float32(np.float32(2.0) * np.float32(1.0 / t))
        exp.step()
        assert opt.lr == np.float32(np.float32(2.0) * np.float32(1.0 / t) * np.float32(0.5))


def test_step_size_zero_is_rejected():
    with pytest.raises(ValueError):
        O.StepLR(O.Lr(1.0), 0, 0.5)


def test_set_current_epoch_moves_the_schedule():
    opt = O.Lr(1.0)
    s = O.StepLR(opt, 3, 0.5)
    s.epoch = 2
    s.step()          # epoch 3: a multiple of the step size
    assert s.epoch == 3 and opt.lr == np.float32(0.5) and s.last_lr == np.float32(1.0)


# ------------------------------------------------------------------------- the package's host-side schedulers
class StubOptimizer:
    """what a host-side scheduler needs of an optimizer: get_lr / set_lr of a Python float"""

    def __init__(self, lr):
        self.lr = float(lr)

    def get_lr(self):
        return self.lr

    def set_lr(self, lr):
        self.lr = float(lr)


def package_from_golden(case, opt):
    from neuronika_b200.optim import lr_scheduler as S
    o = oracle_from_golden(case, O.Lr(opt.get_lr()))
    name = case["scheduler"]
    if name == "StepLR":
        return S.StepLR(opt, o.step_size, float(o.gamma))
    if name == "MultiStepLR":
        return S.MultiStepLR(opt, o.milestones, float(o.gamma))
    if name == "ExponentialLR":
        return S.ExponentialLR(opt, float(o.gamma))
    return getattr(S, name)(opt, o.lr_fn)


@pytest.mark.parametrize("name", sorted(CASES))
def test_host_scheduler_passes_the_reference_test(name):
    case = CASES[name]

    def make(lr):
        opt = StubOptimizer(lr)
        return package_from_golden(case, opt), opt
    run_reference_test(case, make)


SPECS = [
    ("StepLR", dict(step_size=3, gamma=0.7)),
    ("MultiStepLR", dict(milestones=[2, 5, 6], gamma=0.3)),
    ("ExponentialLR", dict(gamma=0.93)),
    ("MultiplicativeLR", dict(lr_fn=lambda t: 1.0 - 0.05 * t)),
    ("LambdaLR", dict(lr_fn=lambda t: 0.9 ** t + 0.01)),
]


@pytest.mark.parametrize("name,kw", SPECS, ids=[s[0] for s in SPECS])
def test_host_scheduler_matches_the_oracle_bit_for_bit(name, kw):
    from neuronika_b200.optim import lr_scheduler as S
    opt, ref = StubOptimizer(0.1), O.Lr(0.1)
    s, o = getattr(S, name)(opt, **kw), getattr(O, name)(ref, *kw.values())
    for t in range(12):
        if t == 7:
            s.set_current_epoch(1)
            o.epoch = 1
        s.step()
        o.step()
        assert np.float32(opt.get_lr()) == ref.lr
        assert (s.get_last_lr(), s.get_current_lr(), s.get_current_epoch()) == (o.last_lr, o.current_lr, o.epoch)


def test_host_scheduler_rejects_step_size_zero():
    from neuronika_b200.optim import lr_scheduler as S
    with pytest.raises(ValueError):
        S.StepLR(StubOptimizer(1.0), 0, 0.5)
    s = S.StepLR(StubOptimizer(1.0), 1, 0.5)
    with pytest.raises(ValueError):
        s.set_step_size(0)
