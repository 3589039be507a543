"""Running error analysis of the fused optimizer step's fp32 arithmetic (ops/csrc/tfy_fused_step.cuh), shared by the
single-GPU test (test_gpu_fused_step.py) and the multi-GPU one (test_gpu_comm_reference.py).  Plain NumPy.

Each intermediate x of the kernel carries its exact value and a bound e(x) on the distance of the kernel's value from
it (class ``B``):

* an fp32 add, sub or mul of x and y has e = e(x) + e(y) (add, sub) or |x| e(y) + |y| e(x) + e(x) e(y) (mul),
  plus u (|r| + e) for the rounding of the result r, u = 2^-24, plus 2^-149 for a result in the subnormal range.
  A fused multiply-add rounds once where this counts two roundings, so contraction stays inside the bound.  This
  covers the fp32 rounding of each state update and the final rounding of the stored p (a half ulp).
* sqrt.approx / rsqrt.approx / div.approx (and rsqrtf) err by at most 2 ulp, i.e. 2^-22 of the result, on top of
  the propagated error of their inputs (evaluated exactly: sqrt(x) - sqrt(x - e), 1/sqrt(x - e) - 1/sqrt(x) and
  the quotient rule).  Being .ftz, they also flush subnormal inputs and results: an absolute 2^-126 on each.
  That is the absolute floor of the states: g * g underflows in fp32 where the reference keeps 1e-50.
* Adam's bias correction: powf(beta, t) errs by at most 8 ulp (twice CUDA's documented bound), which the
  cancellation in 1 - beta^t magnifies by beta^t / (1 - beta^t): about 1000 for beta2 = 0.999 at t = 1.
* The gradient's scale ``grad_scale / world`` is one IEEE fp32 division on the device: exact at 1, 2, 4 and 8 ranks,
  rounded at 3 or 5.  Its distance from the exact quotient is part of the bound.
"""
import numpy as np

U = 2.0 ** -24
SUB = 2.0 ** -149
APPROX = 2.0 ** -22
FLUSH = 2.0 ** -126
POW = 8 * 2.0 ** -23


class B:
    """Exact value ``v`` of an intermediate of the kernel and a bound ``e`` on the kernel's distance from it."""
    __slots__ = ("v", "e")

    def __init__(self, v, e=0.0):
        self.v = np.asarray(v, np.float64)
        self.e = np.asarray(e, np.float64)

    @staticmethod
    def of(x):
        return x if isinstance(x, B) else B(x)

    @staticmethod
    def rounded(v, e):
        return B(v, e + U * (np.abs(v) + e) + SUB)

    def __add__(self, o):
        o = B.of(o)
        return B.rounded(self.v + o.v, self.e + o.e)

    __radd__ = __add__

    def __sub__(self, o):
        o = B.of(o)
        return B.rounded(self.v - o.v, self.e + o.e)

    def __rsub__(self, o):
        return B.of(o) - self

    def __mul__(self, o):
        o = B.of(o)
        return B.rounded(self.v * o.v, np.abs(self.v) * o.e + np.abs(o.v) * self.e + self.e * o.e)

    __rmul__ = __mul__

    def __neg__(self):
        return B(-self.v, self.e)


def sqrt_a(x):
    z = np.sqrt(np.maximum(x.v, 0.0))
    e = z - np.sqrt(np.maximum(x.v - x.e - FLUSH, 0.0))
    return B(z, e + APPROX * (z + e))


def rsqrt_a(x):
    z = 1.0 / np.sqrt(x.v)
    lo = x.v - x.e - FLUSH
    e = np.where(lo > 0, 1.0 / np.sqrt(np.where(lo > 0, lo, 1.0)) - z, np.inf)
    return B(z, e + APPROX * (z + e))


def div_a(a, b, rel=APPROX, flush=FLUSH):
    a, b = B.of(a), B.of(b)
    z = a.v / b.v
    bb = np.abs(b.v) - b.e
    ea = a.e + flush
    e = np.where(bb > 0, (np.abs(a.v) * b.e + np.abs(b.v) * ea) / (np.abs(b.v) * np.where(bb > 0, bb, 1.0)), np.inf)
    return B(z, e + rel * (np.abs(z) + e) + flush)


def one_minus(x):
    return B(1.0) - B(x)


def grad_scale(h):
    """``tfy_step_consts``' ``gscale = grad_scale / (float)world`` as a bounded value: the exact quotient, off by the
    rounding of the fp32 division (zero when ``world`` is a power of two)."""
    exact = h.grad_scale / h.world
    device = float(np.float32(h.grad_scale) / np.float32(h.world))
    return B(exact, abs(device - exact))


def _kernel_update(kind, h, step, p, g, s1, s2, s3):
    """tfy_step_consts + tfy_opt_update_rt on bounded values, operation by operation.  Returns the new
    (p, s1, s2, s3) and, for FTRL, the elements whose |z| is too close to l1 to tell which side the kernel lands on."""
    g = g * grad_scale(h)
    if h.wd != 0.0 and not (kind == "adam" and h.flags & 1):
        g = g + B(h.wd) * p
    undecided = None
    if kind == "sgd":
        if h.p1 != 0.0:
            s1 = g if step == 0 else B(h.p1) * s1 + one_minus(h.p2) * g
            g = g + B(h.p1) * s1 if h.flags & 1 else s1
        p = p - B(h.lr) * g
    elif kind == "adadelta":
        s1 = B(h.p1) * s1 + one_minus(h.p1) * g * g
        upd = g * sqrt_a(s2 + B(h.eps)) * rsqrt_a(s1 + B(h.eps))
        s2 = B(h.p1) * s2 + one_minus(h.p1) * upd * upd
        p = p - B(h.lr) * upd
    elif kind == "adam":
        t = step + 1
        pw1, pw2 = h.p1 ** t, h.p2 ** t
        lr_bc1 = div_a(B(h.lr), B(1.0) - B(pw1, POW * pw1), rel=U, flush=0.0)
        bc2_rsqrt = rsqrt_a(B(1.0) - B(pw2, POW * pw2))
        if h.flags & 1:
            p = p * (B(1.0) - B(h.lr) * B(h.wd))
        s1 = B(h.p1) * s1 + one_minus(h.p1) * g
        s2 = B(h.p2) * s2 + one_minus(h.p2) * g * g
        denom = sqrt_a(s2) * bc2_rsqrt + B(h.eps)
        p = p - lr_bc1 * div_a(s1, denom)
    elif kind == "ftrl":
        n_new = s1 + g * g
        sq_new = sqrt_a(n_new)
        s2 = s2 + (g - (sq_new - sqrt_a(s1)) * div_a(p, B(h.lr)))
        s1 = n_new
        w = -div_a(s2 - B(np.copysign(h.p1, s2.v)), div_a(B(h.eps) + sq_new, B(h.lr)) + B(2.0 * h.p2))
        zero = np.abs(s2.v) <= h.p1
        undecided = np.abs(np.abs(s2.v) - h.p1) <= s2.e
        p = B(np.where(zero, 0.0, w.v), np.where(zero & ~undecided, 0.0, w.e))
    elif kind == "adagrad":
        s1 = s1 + g * g
        p = p - B(h.lr) * div_a(g, sqrt_a(s1) + B(h.eps))
    else:
        s1 = B(h.p1) * s1 + one_minus(h.p1) * g * g
        denom = s1
        if h.flags & 1:
            s3 = B(h.p1) * s3 + one_minus(h.p1) * g
            denom = denom - s3 * s3
        inc = B(h.lr) * g * rsqrt_a(denom + B(h.eps))
        if h.p2 > 0.0:
            s2 = B(h.p2) * s2 + inc
            p = p - s2
        else:
            p = p - inc
    return (p, s1, s2, s3), undecided
