"""The oracle of the 1-d / 3-d convolution layers -- pad_mode_forward -> conv_forward -> + bias, backward through
conv_backward_input / conv_backward_kernel and pad_mode_backward -- against torch's CPU autograd in float64 (F.pad modes
constant, reflect and replicate, then F.conv1d / F.conv3d with the bias).  The forward, dW and db agree for every mode,
and so does dX for the zero and constant modes.  For reflective and replicative padding the reference's pad backward
keeps the interior slice of the padded input's gradient (pad/mod.rs:157-182) while torch folds the border gradient back
onto the input: there dX is the gradient torch computes for the PADDED input, sliced to its interior."""
import numpy as np
import pytest

import oracle as O

torch = pytest.importorskip("torch")
F = torch.nn.functional

TORCH_MODE = {"zero": "constant", "constant": "constant", "reflective": "reflect", "replicative": "replicate"}
VALUE = {"zero": 0.0, "constant": 0.75, "reflective": 0.0, "replicative": 0.0}

# nsp: (x shape, cout, kernel, padding, stride, dilation)
CASES = {
    1: ((3, 4, 17), 5, (3,), (2,), (2,), (3,)),
    3: ((2, 3, 6, 5, 7), 4, (2, 3, 2), (1, 2, 3), (2, 1, 1), (1, 1, 2)),
}


def oracle_layer(x, w, b, pad, mode, stride, dil, g):
    om = "constant" if mode == "zero" else mode
    xp = O.pad_mode_forward(x, pad, om, VALUE[mode])
    y = O.conv_forward(xp, w, stride, dil).astype(np.float64) + b.reshape((1, -1) + (1,) * len(pad))
    gp = O.conv_backward_input(np.zeros(xp.shape), g, w, stride, dil)
    dx = O.pad_mode_backward(gp, np.zeros(x.shape), pad)
    dw = O.conv_backward_kernel(np.zeros(w.shape), g, xp, stride, dil)
    db = g.sum(axis=tuple(i for i in range(g.ndim) if i != 1))
    return y, dx, dw, db


def torch_layer(x, w, b, pad, mode, stride, dil, g):
    """forward and gradients of torch's layer; also the gradient of the padded input"""
    xt, wt, bt = (torch.tensor(a, dtype=torch.float64, requires_grad=True) for a in (x, w, b.ravel()))
    widths = [p for p in reversed(pad) for _ in range(2)]
    if mode in ("zero", "constant"):
        xp = F.pad(xt, widths, mode="constant", value=VALUE[mode])
    else:
        xp = F.pad(xt, widths, mode=TORCH_MODE[mode])
    xp.retain_grad()
    conv = F.conv1d if len(pad) == 1 else F.conv3d
    y = conv(xp, wt, bt, stride=stride, dilation=dil)
    y.backward(torch.tensor(g))
    return y.detach().numpy(), xt.grad.numpy(), xp.grad.numpy(), wt.grad.numpy(), bt.grad.numpy()


def close(a, b, what):
    scale = np.abs(b).max() + 1e-30
    assert a.shape == b.shape, (what, a.shape, b.shape)
    assert np.abs(a - b).max() <= 1e-5 * scale, (what, float(np.abs(a - b).max()), scale)


@pytest.mark.parametrize("mode", list(TORCH_MODE))
@pytest.mark.parametrize("nsp", [1, 3])
def test_layer_matches_torch(nsp, mode):
    xs, cout, k, pad, stride, dil = CASES[nsp]
    rng = np.random.default_rng(nsp * 10 + len(mode))
    x = rng.uniform(-1, 1, xs)
    w = rng.uniform(-0.5, 0.5, (cout, xs[1]) + k)
    b = rng.uniform(-0.5, 0.5, (cout,) + (1,) * nsp)
    xp_shape = xs[:2] + tuple(s + 2 * p for s, p in zip(xs[2:], pad))
    g = rng.uniform(-1, 1, O.conv_out_shape(xp_shape, w.shape, stride, dil))
    y, dx, dw, db = oracle_layer(x, w, b, pad, mode, stride, dil, g)
    ty, tdx, tdxp, tdw, tdb = torch_layer(x, w, b, pad, mode, stride, dil, g)
    close(y, ty, "y")
    close(dw, tdw, "dw")
    close(db, tdb, "db")
    interior = tuple([slice(None)] * 2 + [slice(p, p + s) for p, s in zip(pad, xs[2:])])
    close(dx, tdxp[interior], "dx (interior of the padded input's gradient)")
    if mode in ("zero", "constant"):
        close(dx, tdx, "dx")
    else:
        # torch's dX adds the border gradient back onto the mirrored / repeated elements: not the reference's rule
        assert np.abs(dx - tdx).max() > 1e-3 * np.abs(tdx).max()
