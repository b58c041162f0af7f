"""The host convolution model of tests/tf32_conv_oracle.py against torch's float64 CPU autograd on an explicitly padded
input: forward, the padded input's gradient sliced to its interior (the reference's pad backward), and dW, in 1-D, 2-D
and 3-D, every padding mode, with stride and dilation."""
import numpy as np
import pytest

import tf32_conv_oracle as C

TORCH_PAD = {"zero": "constant", "constant": "constant", "reflective": "reflect", "replicative": "replicate"}
CASES = [   # (x shape, Cout, kernel, padding, stride, dilation)
    ((2, 3, 11), 4, (3,), (2,), (2,), (1,)),
    ((2, 3, 7, 9), 5, (3, 2), (1, 2), (1, 2), (2, 1)),
    ((2, 2, 4, 5, 6), 3, (2, 3, 2), (1, 1, 2), (2, 1, 1), (1, 2, 2)),
]


@pytest.mark.parametrize("mode", list(TORCH_PAD))
@pytest.mark.parametrize("case", CASES, ids=["1d", "2d", "3d"])
def test_model_matches_torch_autograd(case, mode):
    import torch
    import torch.nn.functional as F
    xs, cout, k, pad, s, d = case
    rng = np.random.default_rng(len(xs) * 10 + len(mode))
    x = rng.standard_normal(xs)
    w = rng.standard_normal((cout, xs[1]) + k)
    b = rng.standard_normal(cout)
    fill = 0.7 if mode == "constant" else 0.0
    widths = [p for q in reversed(pad) for p in (q, q)]
    xt = torch.tensor(x)
    xp = (F.pad(xt, widths, mode="constant", value=fill) if TORCH_PAD[mode] == "constant"
          else F.pad(xt, widths, mode=TORCH_PAD[mode])).requires_grad_(True)
    wt, bt = torch.tensor(w, requires_grad=True), torch.tensor(b, requires_grad=True)
    conv = {1: F.conv1d, 2: F.conv2d, 3: F.conv3d}[len(k)]
    y = conv(xp, wt, bt, stride=s, dilation=d)
    g = rng.standard_normal(tuple(y.shape))
    (y * torch.tensor(g)).sum().backward()
    np.testing.assert_allclose(C.forward(x, w, b, pad, mode, fill, s, d), y.detach().numpy(), rtol=1e-12, atol=1e-12)
    interior = (slice(None), slice(None)) + tuple(slice(p, p + n) for p, n in zip(pad, xs[2:]))
    np.testing.assert_allclose(C.backward_input(xs, g, w, pad, s, d), xp.grad.numpy()[interior], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(C.backward_kernel(g, x, w.shape, pad, mode, fill, s, d), wt.grad.numpy(), rtol=1e-12,
                               atol=1e-12)
