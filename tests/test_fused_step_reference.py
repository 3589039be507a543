"""The float64 reference of the fused optimizer step (tests/fused_step_reference.py) against torch.optim, and against
the repository's TorchFtrl / TorchRMSprop, all in float64 on the CPU, plus a few cases worked out by hand.  The GPU
test of the kernel (test_gpu_fused_step.py) trusts this reference, so it is pinned here first."""
import numpy as np
import pytest
import torch

import fused_step_reference as ref
from tf_yarn_b200.keras.optimizers import TorchFtrl, TorchRMSprop


def _torch_optimizer(name, params):
    kind, hp, init = ref.VARIANTS[name]
    h = ref.Hyper(**hp)
    if kind == "sgd":
        return torch.optim.SGD(params, lr=h.lr, momentum=h.p1, dampening=h.p2, nesterov=bool(h.flags & 1),
                               weight_decay=h.wd)
    if kind == "adadelta":
        return torch.optim.Adadelta(params, lr=h.lr, rho=h.p1, eps=h.eps, weight_decay=h.wd)
    if kind == "adam":
        cls = torch.optim.AdamW if h.flags & 1 else torch.optim.Adam
        return cls(params, lr=h.lr, betas=(h.p1, h.p2), eps=h.eps, weight_decay=h.wd)
    if kind == "adagrad":
        return torch.optim.Adagrad(params, lr=h.lr, eps=h.eps, weight_decay=h.wd, initial_accumulator_value=init)
    if kind == "ftrl":
        assert h.wd == 0.0
        return TorchFtrl(params, lr=h.lr, l1=h.p1, l2=h.p2, beta=h.eps, initial_accumulator_value=init)
    return TorchRMSprop(params, lr=h.lr, rho=h.p1, momentum=h.p2, eps=h.eps, centered=bool(h.flags & 1),
                        weight_decay=h.wd)


def _torch_states(name, opt, p):
    """The torch optimizer's state in the kernel's (s1, s2, s3) order, None where it has none."""
    kind, hp, _ = ref.VARIANTS[name]
    st = opt.state[p]
    get = {"sgd": ("momentum_buffer", None, None), "adadelta": ("square_avg", "acc_delta", None),
           "adam": ("exp_avg", "exp_avg_sq", None), "adagrad": ("sum", None, None), "ftrl": ("n", "z", None),
           "rmsprop": ("v", "m", "mg")}[kind]
    return [st[k].numpy() if k is not None and k in st else None for k in get]


@pytest.mark.parametrize("name", sorted(ref.VARIANTS))
def test_reference_matches_torch_optim_in_float64(name):
    kind, hp, init = ref.VARIANTS[name]
    h = ref.Hyper(**hp)
    rs = np.random.RandomState(7)
    n = 301
    p0 = rs.randn(n) * 0.3
    if kind == "ftrl":
        p0[::5] = 0.0
    param = torch.nn.Parameter(torch.from_numpy(p0.copy()))
    opt = _torch_optimizer(name, [param])
    p, s1, s2, s3 = p0.copy(), np.full(n, init), np.zeros(n), np.zeros(n)
    for step in range(10):
        g = rs.randn(n) * 0.5
        g[::7] = 0.0
        param.grad = torch.from_numpy(g.copy())
        opt.step()
        p, s1, s2, s3 = ref.step(kind, p, g, s1, s2, s3, h, step)
        want = param.detach().numpy()
        assert np.allclose(p, want, rtol=1e-12, atol=1e-14), (step, np.abs(p - want).max())
        for got, st in zip((s1, s2, s3), _torch_states(name, opt, param)):
            if st is not None:
                assert np.allclose(got, st, rtol=1e-12, atol=1e-14), (step, np.abs(got - st).max())
    if kind == "ftrl":
        assert np.array_equal(p == 0.0, param.detach().numpy() == 0.0)
        assert 0 < int((p == 0.0).sum()) < n                 # l1 zeroes some weights and keeps others


def test_reference_scales_the_summed_gradient():
    """The kernel reads the gradient summed over the ranks: the update uses summed * grad_scale / world."""
    h1 = ref.Hyper(lr=0.1)
    h4 = ref.Hyper(lr=0.1, grad_scale=0.5, world=4)
    p, g, z = np.array([1.0, -2.0]), np.array([0.3, -0.7]), np.zeros(2)
    assert np.array_equal(ref.sgd(p, g, z, z, z, h1, 0)[0], ref.sgd(p, g * 8, z, z, z, h4, 0)[0])


def test_hyper_holds_the_float32_values():
    h = ref.Hyper(lr=0.1, p2=0.999)
    assert h.lr == float(np.float32(0.1)) != 0.1
    assert h.p2 == float(np.float32(0.999))


def test_ftrl_zeroes_the_weight_when_z_is_within_l1():
    """One FTRL step by hand: lr 1, l1 0.5, l2 0, beta 0, n0 = 1, z0 = 0, p0 = 0.
    g = 0.4: n = 1.16, z = 0.4 (p0 = 0, so sigma * p vanishes): |z| <= l1, w = 0.
    g = 0.6: n = 1.36, z = 0.6: w = -(0.6 - 0.5) / sqrt(1.36)."""
    h = ref.Hyper(lr=1.0, p1=0.5)
    one, zero = np.ones(1), np.zeros(1)
    p, n, z, _ = ref.ftrl(zero, np.array([0.4]), one, zero, zero, h, 0)
    assert p[0] == 0.0 and z[0] == pytest.approx(0.4) and n[0] == pytest.approx(1.16)
    p, n, z, _ = ref.ftrl(zero, np.array([0.6]), one, zero, zero, h, 0)
    assert p[0] == pytest.approx(-0.1 / np.sqrt(1.36), rel=1e-12)
    p, _, z, _ = ref.ftrl(zero, np.array([-0.5]), one, zero, zero, h, 0)    # |z| == l1 exactly: still zero
    assert z[0] == -0.5 and p[0] == 0.0


def test_sgd_first_step_takes_the_gradient_as_momentum_buffer():
    """torch.optim.SGD: the first step sets buf = g (no dampening); later ones buf = m * buf + (1 - d) * g."""
    h = ref.Hyper(lr=0.5, p1=0.75, p2=0.5)
    p, z = np.array([1.0]), np.zeros(1)
    p1, buf, _, _ = ref.sgd(p, np.array([2.0]), z, z, z, h, 0)
    assert buf[0] == 2.0 and p1[0] == 0.0                    # 1 - 0.5 * 2
    p2, buf, _, _ = ref.sgd(p1, np.array([4.0]), buf, z, z, h, 1)
    assert buf[0] == 0.75 * 2.0 + 0.5 * 4.0 and p2[0] == -0.5 * 3.5
    h_nesterov = ref.Hyper(lr=0.5, p1=0.75, flags=1)
    p3, buf, _, _ = ref.sgd(p, np.array([2.0]), z, z, z, h_nesterov, 0)
    assert buf[0] == 2.0 and p3[0] == 1.0 - 0.5 * (2.0 + 0.75 * 2.0)


def test_adam_bias_correction_counts_the_step_being_taken():
    """From zero moments, step ``k`` (k completed updates) is update t = k + 1:
    m = (1 - b1) g, v = (1 - b2) g^2, p -= lr / (1 - b1^t) * m / (sqrt(v) / sqrt(1 - b2^t) + eps)."""
    h = ref.Hyper(lr=0.01, p1=0.9, p2=0.999, eps=1e-8)
    b1, b2 = h.p1, h.p2
    p, g, z = np.array([0.5]), np.array([0.2]), np.zeros(1)
    for k in (0, 3):
        t = k + 1
        m, v = (1 - b1) * 0.2, (1 - b2) * 0.04
        want = 0.5 - h.lr / (1 - b1 ** t) * m / (np.sqrt(v) / np.sqrt(1 - b2 ** t) + h.eps)
        got, s1, s2, _ = ref.adam(p, g, z, z, z, h, k)
        assert got[0] == pytest.approx(want, rel=1e-14) and s1[0] == pytest.approx(m) and s2[0] == pytest.approx(v)
    # at t = 1 the corrected step is lr * g / (|g| + eps): one learning rate, whatever |g|
    assert ref.adam(p, g, z, z, z, h, 0)[0][0] == pytest.approx(0.5 - h.lr * 0.2 / (0.2 + h.eps), rel=1e-12)
    # an off-by-one in t would show: step 3 with t = 3 differs from the right answer by far more than rounding
    t3 = 0.5 - h.lr / (1 - b1 ** 3) * (1 - b1) * 0.2 / (np.sqrt((1 - b2) * 0.04) / np.sqrt(1 - b2 ** 3) + h.eps)
    assert abs(ref.adam(p, g, z, z, z, h, 3)[0][0] - t3) > 1e-4
