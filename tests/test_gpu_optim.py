"""Optimizers and learning-rate schedulers on the GPU (csrc/nk_optim_multi.cu, optim.Optimizer, optim.lr_scheduler):
the weights, written-back gradients and optimizer state of every step of every optimizer variant, penalty, dtype pair,
master weights and grad_scale, across the 64-tensors-per-launch boundary, match one step of the numpy oracle from the
state the device held before it; a captured training step with a scheduler replays to the bits of the same step run
eagerly, lr and epoch included; device lr changes reach the next replay; host reads and writes are refused while
capturing; and the launch count is 1 + ceil(P/64) (+1 per scheduler)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SIZES = [1, 3, 4, 5, 4097, (1 << 20) + 3]
MISALIGNED = 4097                     # a view one element past an aligned base: element accesses only
N_TENSORS = 70                        # crosses the 64-per-launch boundary
PAIRS = [("f32", "f32"), ("bf16", "bf16"), ("bf16", "f32"), ("f32", "bf16")]


@pytest.fixture(scope="module")
def nk():
    import neuronika_b200 as nk
    return nk


@pytest.fixture(scope="module")
def dev(nk):
    return nk.Device(0)


def _variants(optim):
    O = optim
    return [
        ("sgd", O.StochasticGD, dict(lr=0.05)),
        ("sgd_l2_momentum", O.StochasticGD, dict(lr=0.05, penalty=O.L2(0.01), momentum=0.9, dampening=0.1)),
        ("sgd_nesterov", O.StochasticGD, dict(lr=0.05, momentum=0.8, dampening=0.0, nesterov=True)),
        ("adam", O.Adam, dict(lr=1e-3)),
        ("amsgrad", O.AMSGrad, dict(lr=1e-3, beta1=0.8, beta2=0.99)),
        ("rmsprop", O.RMSProp, dict(lr=1e-3)),
        ("rmsprop_centered", O.RMSProp, dict(lr=1e-3, centered=True)),
        ("rmsprop_momentum", O.RMSProp, dict(lr=1e-3, momentum=0.5)),
        ("rmsprop_centered_momentum", O.RMSProp, dict(lr=1e-3, momentum=0.5, centered=True)),
        ("adagrad", O.Adagrad, dict(lr=1e-2)),
        ("adagrad_decay", O.Adagrad, dict(lr=1e-2, lr_decay=0.05)),
    ]


VARIANT_NAMES = ["sgd", "sgd_l2_momentum", "sgd_nesterov", "adam", "amsgrad", "rmsprop", "rmsprop_centered",
                 "rmsprop_momentum", "rmsprop_centered_momentum", "adagrad", "adagrad_decay"]


def _penalty(optim, k):
    return [optim.L1(0.003), optim.L2(0.01), optim.ElasticNet(0.002, 0.005), None][k % 4]


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _make_params(nk, dev, data, wdt, gdt, keep):
    """the parameters; `keep` receives the storage under the misaligned view, which must outlive the parameter"""
    from neuronika_b200 import variable as V
    ps = []
    for i, x in enumerate(data):
        if i == len(SIZES):                             # the misaligned view
            base = dev.zeros((x.size + 1,), wdt)
            keep.append(base)
            view = base.slice_flat(1, x.shape)
            view.copy_from(x)
            ps.append(V.from_device_memory(dev, view).requires_grad(gdt))
        else:
            ps.append(nk.from_ndarray(dev, x, wdt).requires_grad(gdt))
    return ps


def _states(p):
    names = ("buffer", "exp_avg", "exp_avg_sq", "max_exp_avg_sq", "square_avg", "grad_avg", "grad_sq", "master")
    return [(n, getattr(p, n).as_ndarray()) for n in names if getattr(p, n, None) is not None]


def _oracle_step(O, optim, status, t, lr, w, g, st):
    """one step of the numpy oracle, in place: w the f32 weight (the master copy when there is one), g the gradient
    with grad_scale applied, st the state arrays by name; t the step count after the step"""
    l1, l2 = optim._l1_l2(status.penalty)
    if isinstance(status, optim.StochasticGD):
        buf = O.sgd_step(w, g, lr, l2, status.momentum, status.dampening, status.nesterov, st.get("buffer"))
        if buf is not None:
            st["buffer"] = buf                         # created by the first step
    elif isinstance(status, optim.Adam):
        O.adam_step(w, g, st["exp_avg"], st["exp_avg_sq"], t, lr, status.beta1, status.beta2, status.eps, l1, l2,
                    max_exp_avg_sq=st.get("max_exp_avg_sq"))
    elif isinstance(status, optim.RMSProp):
        O.rmsprop_step(w, g, st["square_avg"], lr, status.alpha, status.eps, momentum=status.momentum,
                       centered=status.centered, grad_avg=st.get("grad_avg"), buffer=st.get("buffer"), l1=l1, l2=l2)
    else:
        O.adagrad_step(w, g, st["grad_sq"], t, lr, status.lr_decay, status.eps, l1, l2)


def _close(got, want, bf16, where):
    """bf16 storage: one rounding of the oracle's f32 value; f32: test_gpu_next's optimizer tolerances"""
    if bf16:
        assert np.all(np.abs(got - want) <= 2.0 ** -8 * np.abs(want) + 1e-6), where
    else:
        assert np.allclose(got, want, rtol=2e-5, atol=2e-6), where


@pytest.mark.parametrize("pair", range(4), ids=["%s-%s" % p for p in PAIRS])
@pytest.mark.parametrize("variant", range(len(VARIANT_NAMES)), ids=VARIANT_NAMES)
def test_step_matches_the_oracle(nk, dev, variant, pair):
    import oracle as O
    from neuronika_b200 import optim
    name, cls, kw = _variants(optim)[variant]
    wdt, gdt = PAIRS[pair]
    kw = dict(kw)
    if cls is not optim.StochasticGD and "penalty" not in kw:
        pen = _penalty(optim, variant + pair)
        if pen is not None:
            kw["penalty"] = pen
    kw["grad_scale"] = 0.5 if pair in (0, 2) else 1.0
    kw["master_weights"] = (variant + pair) % 2 == 0
    rng = np.random.default_rng(1000 * variant + pair)
    sizes = SIZES + [MISALIGNED] + [17 + 29 * i for i in range(N_TENSORS - len(SIZES) - 1)]
    data = [rng.uniform(-1, 1, n).astype(np.float32) for n in sizes]
    data[0][:] = 0.0                                   # signum(+0) in the L1 penalty
    keep = []
    ps = _make_params(nk, dev, data, wdt, gdt, keep)
    opt = cls.new(**kw)
    for p in ps:
        opt.register(p)
    for step in range(5):
        for p, n in zip(ps, sizes):
            p.grad_array().copy_from(rng.normal(0, 1, n).astype(np.float32))
        if step in (2, 4):
            lr = opt.get_lr() * (0.5 if step == 2 else 3.0)
            opt.set_lr(lr)
            assert np.float32(opt.get_lr()) == np.float32(lr)
        lr = np.float32(opt.get_lr())
        before = [(p.data(), p.grad(), dict(_states(q))) for p, q in zip(ps, opt.params)]
        opt.step()
        for i, (p, q, (w, g, st)) in enumerate(zip(ps, opt.params, before)):
            where = "%s %s/%s step %d tensor %d (n=%d)" % (name, wdt, gdt, step, i, sizes[i])
            master = st.pop("master", None)
            w = master if master is not None else w
            g = (g * np.float32(kw["grad_scale"])).astype(np.float32)
            l1, l2 = optim._l1_l2(opt.status.penalty)
            sg = np.abs(g.astype(np.float64)) + l1 + 2 * l2 * np.abs(w.astype(np.float64))   # the terms of g'
            _oracle_step(O, optim, opt.status, step + 1, lr, w, g, st)
            if master is not None:
                got = dict(_states(q))["master"]
                _close(got, w, False, where + ": master")
                assert np.array_equal(_bits(p.data()), _bits(O.bf16_round(got))), where + ": weights != bf16(master)"
            else:
                _close(p.data(), w, wdt == "bf16", where + ": weights")
            _close(p.grad(), g, gdt == "bf16", where + ": written-back gradient")
            for sn, x in _states(q):
                if sn == "master":
                    continue
                want = st[sn].astype(np.float64)
                tol = 2e-5 * np.abs(want) + 2e-6
                if cls is optim.RMSProp and sn == "buffer":
                    # b = mu*b + g'/denom: when g' nearly cancels (g against its penalty) denom is about eps, and
                    # g''s few roundings, each at most 2^-24 of its terms, are divided by denom
                    var = st["square_avg"].astype(np.float64) - (st["grad_avg"].astype(np.float64) ** 2
                                                                if "grad_avg" in st else 0.0)
                    tol = tol + 16 * 2.0 ** -24 * sg / (np.sqrt(np.maximum(var, 0.0)) + opt.status.eps)
                assert np.all(np.abs(x - want) <= tol), where + ": " + sn
    if cls in (optim.Adam, optim.AMSGrad, optim.Adagrad):
        assert opt._read().step == 5                   # the prologue's count


# ------------------------------------------------------------------------------------- captured training step
def _mlp(nk, dev, seed):
    """Linear-ReLU-Linear, bf16 data, f32 gradients: (a function that builds the loss graph, the parameters)"""
    from neuronika_b200 import nn
    rng = np.random.default_rng(seed)
    l1 = nn.Linear(dev, 64, 128, dtype=nk.BF16, grad_dtype=nk.F32, rng=rng)
    l2 = nn.Linear(dev, 128, 32, dtype=nk.BF16, grad_dtype=nk.F32, rng=rng)
    x = nk.from_ndarray(dev, rng.uniform(-1, 1, (256, 64)).astype(np.float32), nk.BF16)
    t = nk.from_ndarray(dev, rng.uniform(-1, 1, (256, 32)).astype(np.float32), nk.BF16)
    return (lambda: l2.forward(l1.forward(x).relu()).mse_loss(t)), l1.parameters() + l2.parameters()


def _pairs(optim, S):
    return [
        ("adam_step", lambda **k: optim.Adam.new(1e-2, **k), lambda o: S.StepLR(o, 2, 0.5), None),
        ("amsgrad_multistep", lambda **k: optim.AMSGrad.new(1e-2, **k), lambda o: S.MultiStepLR(o, [2, 3, 5], 0.5),
         None),
        ("adagrad_exponential", lambda **k: optim.Adagrad.new(5e-2, lr_decay=0.05, **k),
         lambda o: S.ExponentialLR(o, 0.9), None),
        ("rmsprop_lambda", lambda **k: optim.RMSProp.new(1e-3, momentum=0.5, centered=True, **k),
         lambda o, h=None: S.LambdaLR(o, lambda t: 1.0 / (t + 1), horizon=h), 16),
        ("sgd_multiplicative", lambda **k: optim.StochasticGD.new(0.05, momentum=0.9, dampening=0.0, nesterov=True, **k),
         lambda o, h=None: S.MultiplicativeLR(o, lambda t: 0.95, horizon=h), 16),
    ]


PAIR_NAMES = ["adam_step", "amsgrad_multistep", "adagrad_exponential", "rmsprop_lambda", "sgd_multiplicative"]


@pytest.mark.parametrize("k", range(len(PAIR_NAMES)), ids=PAIR_NAMES)
def test_captured_step_with_scheduler_replays_the_eager_step(nk, dev, k):
    from neuronika_b200 import optim
    from neuronika_b200.optim import lr_scheduler as S
    from oracle import lr_scheduler as OS
    name, make_opt, make_sched, horizon = _pairs(optim, S)[k]

    def sched_for(o, device):   # a closure scheduler without horizon runs on the host: eager only
        return make_sched(o, horizon) if horizon is not None and device else make_sched(o)

    loss_d, params_d = _mlp(nk, dev, 7)
    loss_c, params_c = _mlp(nk, dev, 7)
    od, oc = make_opt(), make_opt()
    for p in params_d:
        od.register(p)
    for p in params_c:
        oc.register(p)
    sd, sc = sched_for(od, False), sched_for(oc, True)
    ref_opt = OS.Lr(od.get_lr())
    ref = {"adam_step": lambda o: OS.StepLR(o, 2, 0.5), "amsgrad_multistep": lambda o: OS.MultiStepLR(o, [2, 3, 5], 0.5),
           "adagrad_exponential": lambda o: OS.ExponentialLR(o, 0.9),
           "rmsprop_lambda": lambda o: OS.LambdaLR(o, lambda t: 1.0 / (t + 1)),
           "sgd_multiplicative": lambda o: OS.MultiplicativeLR(o, lambda t: 0.95)}[name](ref_opt)

    def step(build, opt, sched):             # a new graph every step, as a training loop written against the reference
        opt.zero_grad()
        loss = build()
        loss.forward()
        loss.backward(1.0)
        opt.step()
        sched.step()

    def same(where):
        for i, (a, b) in enumerate(zip(params_d, params_c)):
            assert np.array_equal(_bits(a.data()), _bits(b.data())), "%s %s: parameter %d" % (name, where, i)
        assert np.float32(od.get_lr()) == np.float32(oc.get_lr()) == ref_opt.lr, where
        assert sd.get_current_epoch() == sc.get_current_epoch() == ref.epoch, where
        assert sc.get_current_lr() == ref.current_lr and sc.get_last_lr() == ref.last_lr, where

    step(loss_d, od, sd)
    step(loss_c, oc, sc)
    ref.step()
    same("eager step")
    with dev.capture(256 << 20) as cap:
        step(loss_c, oc, sc)
    for r in range(6):
        step(loss_d, od, sd)
        ref.step()
        cap.graph.launch()
        dev.synchronize()
        same("replay %d" % r)
    if name in ("adam_step", "amsgrad_multistep", "adagrad_exponential"):
        assert oc._read().step == 7
    w = params_c[0].data()
    assert np.all(np.isfinite(w)) and not np.array_equal(w, _mlp(nk, dev, 7)[1][0].data())   # it trained
    cap.graph.close()


def test_set_lr_between_replays_reaches_the_next_replay(nk, dev):
    from neuronika_b200 import optim
    rng = np.random.default_rng(3)
    x = rng.uniform(-1, 1, 1000).astype(np.float32)
    g = rng.normal(0, 1, 1000).astype(np.float32)
    pd, pc = nk.from_ndarray(dev, x).requires_grad(), nk.from_ndarray(dev, x).requires_grad()
    od, oc = optim.StochasticGD.new(0.1), optim.StochasticGD.new(0.1)
    od.register(pd)
    oc.register(pc)
    pd.grad_array().copy_from(g)
    pc.grad_array().copy_from(g)
    od.step()
    oc.step()
    with dev.capture(1 << 20) as cap:
        oc.step()
    for lr in (0.1, 0.025, 0.3):
        od.set_lr(lr)
        oc.set_lr(lr)
        od.step()
        cap.graph.launch()
        assert np.array_equal(_bits(pd.data()), _bits(pc.data())), lr
        assert oc.get_lr() == np.float32(lr)
    cap.graph.close()


def test_host_access_is_refused_while_capturing(nk, dev):
    from neuronika_b200 import optim
    from neuronika_b200.optim import lr_scheduler as S
    ps = [nk.from_ndarray(dev, np.ones(8, np.float32)).requires_grad() for _ in range(2)]
    opt = optim.Adam.new(1e-3)
    opt.register(ps[0])
    sched = S.StepLR(opt, 2, 0.5)
    for what in (lambda: opt.set_lr(0.5), lambda: opt.get_lr(), lambda: sched.set_current_epoch(3),
                 lambda: sched.get_current_lr(), lambda: opt.register(ps[1])):
        with pytest.raises(nk.NkError):
            with dev.capture(1 << 20):
                what()
    assert len(opt.params) == 1 and opt.get_lr() == np.float32(1e-3) and sched.get_current_epoch() == 0
    opt.register(ps[1])                                # fine outside a capture, before the first step
    opt.step()
    with pytest.raises(nk.NkError, match="before the first step"):
        opt.register(nk.from_ndarray(dev, np.ones(8, np.float32)).requires_grad())


def test_lambda_past_its_horizon_raises_at_the_next_read(nk, dev):
    from neuronika_b200 import optim
    from neuronika_b200.optim import lr_scheduler as S
    p = nk.from_ndarray(dev, np.ones(8, np.float32)).requires_grad()
    opt = optim.StochasticGD.new(1.0)
    opt.register(p)
    sched = S.LambdaLR(opt, lambda t: 0.5 ** t, horizon=2)
    sched.step()
    sched.step()
    assert opt.get_lr() == 0.25 and sched.get_current_epoch() == 2
    sched.step()                                       # past the table: lr unchanged, the flag set
    assert opt.get_lr() == 0.25
    with pytest.raises(nk.NkError, match="past the end"):
        sched.get_current_lr()
    sched.set_current_epoch(0)                         # a rewrite of the state clears the flag
    sched.step()
    assert sched.get_current_epoch() == 1 and opt.get_lr() == 0.5
    host = S.LambdaLR(opt, lambda t: 1.0)              # no horizon: the rule runs on the host and calls set_lr
    with pytest.raises(nk.NkError):
        with dev.capture(1 << 20):
            host.step()
    assert opt.get_lr() == 0.5 and host.get_current_epoch() == 0


@pytest.mark.parametrize("count", [1, 64, 65, 130])
def test_launch_count(nk, dev, count):
    from neuronika_b200 import optim
    from neuronika_b200.optim import lr_scheduler as S
    ps = [nk.from_ndarray(dev, np.ones(100 + i, np.float32)).requires_grad() for i in range(count)]
    opt = optim.Adam.new(1e-3)
    for p in ps:
        opt.register(p)
    sched = S.ExponentialLR(opt, 0.9)
    opt.step()
    with dev.capture(1 << 20) as cap:
        opt.step()
    assert cap.graph.kernel_count == 1 + -(-count // 64)
    cap.graph.close()
    with dev.capture(1 << 20) as cap:
        opt.step()
        sched.step()
    assert cap.graph.kernel_count == 1 + -(-count // 64) + 1
    cap.graph.close()
