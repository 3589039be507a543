"""The fast path's general-shape layer kernels (ops/csrc/tfy_nn.cu and the C_in = 1 tensor-core kernels of
ops/csrc/tfy_conv.cu) against the float64 reference (tests/nn_reference.py), called directly through the ctypes
declarations of keras/fastpath.py, at the shapes where their branches change.

Exact.  Dropout masks, pool code bytes, hit counts and the pooled maxima are pure functions of bf16 inputs and the
counter-based generator: they must match bit for bit.  A mask / code bit that depends on the sign of an fp32 SUM of
more than two terms (the C_in = 1 convolutions, the split-K slabs) is exact wherever that sum is farther from 0 than its
rounding bound below.  The dropout step is read from a device TfyOptHyper whose step is not 0.

Tolerances.  EPS32 = 2^-24 is the fp32 unit roundoff, U_BF16 = 2^-8 the bf16 one.  A sum whose terms each pass
through at most d fp32 additions (d = the depth of the longest path from a term to the result: the chain a thread
accumulates, then the thread / warp / CTA combination steps) is within d * EPS32 * sum|terms| of the exact sum.  A bf16
output of an fp32 value that is within e of the exact value v is within U_BF16 * |v| + 2 e of v.  So every bf16 output is
checked against U_BF16 * |ref| + 2 * d * EPS32 * sum|terms|, with d per kernel:

* C_in = 1 conv forward: 10 (bias + 9 FMAs); tensor core 16 (the K = 16 accumulation, products of bf16 are exact).
* C_in = 1 weight gradient, CUDA cores: rows per warp * (W - 2) (a lane's chain) + 8 warps + 296 CTAs + 2.  Tensor
  core: 128 * chunks per CTA + 160 CTAs + 4.
* bias + act + dropout: 3 (bias add, 1/(1-rate), the scaling); _f32: + the number of slabs.
* gated backward and pool backward, dz: 2; dbias: rows (a thread's chain) + 256 threads + 592 CTAs + 2.
* softmax: __expf(x) is within (2 + 1.2 |x|) ulp and x = v - max rounds once, so each exponential is within
  K = 4 + 2.2 max|x| ulp; the C-term sum se adds C; dlogits within ((K + C + 3) p + 2 |p - onehot|) EPS32 / B; the loss
  row l = max + __logf(se) - v within (K + C + 8) EPS32 (1 + |max| + |log se| + |v|) + 2^-21.41 (__logf's absolute
  error), summed over B rows (depth B), divided by B; dbias sums B dlogits (depth B) plus their own errors.

Every output sits between guard bytes that must stay untouched.  The reducing kernels (C_in = 1 weight gradients,
gated backward, pool backward, softmax head) run five times on the same inputs: their bf16 dbias / dW and the fp32
loss must be the same bits every time, and the scratch counters must be back at zero.
"""
import math

import numpy as np
import pytest
import torch

import nn_reference as ref

pytestmark = pytest.mark.gpu

EPS32, U_BF16 = ref.EPS32, ref.U_BF16
GUARD = 64                    # guard bytes before and after every output
SEED, STEP = 20261016, 5      # the step comes from a device TfyOptHyper
RUNS = 5


@pytest.fixture(scope="module")
def lib():
    from tf_yarn_b200.keras import fastpath  # noqa: F401  (declares the kernels)
    from tf_yarn_b200.ops import native
    return native.load()


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    lib = ref.host_lib(str(tmp_path_factory.mktemp("nnref")))
    assert lib is not None, "the host build of the dropout generator needs g++ and the CUDA headers"
    return lib


@pytest.fixture(scope="module")
def hp():
    from tf_yarn_b200.ops import native
    h = native.OptHyper(1.0, 0.0, 0.0, 0.0, 0.0, 1.0, STEP, 0, 0, 0)
    return torch.frombuffer(bytearray(bytes(h)), dtype=torch.uint8).cuda()


@pytest.fixture(scope="module")
def scratch():
    from tf_yarn_b200.keras import fastpath
    partial = torch.full((fastpath.PARTIAL_BLOCKS * 9 * 128,), float("nan"), device="cuda")   # any content on entry
    counter = torch.zeros(1, dtype=torch.int32, device="cuda")
    return partial, counter


def _s():
    return torch.cuda.current_stream().cuda_stream


class Out:
    """Device output between guard bytes (and pre-filled with the same byte, so an element the kernel skips shows)."""

    def __init__(self, shape, dtype):
        n = int(np.prod(shape)) * torch.empty((), dtype=dtype).element_size()
        self.full = torch.full((2 * GUARD + n,), 0xA5, dtype=torch.uint8, device="cuda")
        self.t = self.full[GUARD:GUARD + n].view(dtype).view(shape)

    def ptr(self):
        return self.t.data_ptr()

    def get(self):
        torch.cuda.synchronize()
        assert bool((self.full[:GUARD] == 0xA5).all()) and bool((self.full[-GUARD:] == 0xA5).all()), "guard written"
        return self.t.clone()


def _bf16(shape, gen, scale=1.0):
    return (torch.randn(shape, device="cuda", generator=gen) * scale).bfloat16()


def _np(t):
    return t.double().cpu().numpy()


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32).cpu()


def _assert_close(got, want, e, what):
    """bf16 output: |got - want| <= U_BF16 |want| + 2 e (module docstring)."""
    got = _np(got) if isinstance(got, torch.Tensor) else got
    tol = U_BF16 * np.abs(want) + 2.0 * e + 1e-30
    bad = ~(np.abs(got - want) <= tol)
    assert not bad.any(), (what, int(bad.sum()), float(np.abs(got - want)[bad].max()), float(tol[bad].min()))


def _assert_mask(got, want, v, e, what):
    """Mask / flow bits: exact, except where the fp32 value they test lies within its rounding bound e of 0."""
    diff = got != want
    assert not (diff & (np.abs(v) > e)).any(), (what, int(diff.sum()))


# ---------------------------------------------------------------------------------------------- C_in = 1, CUDA cores
@pytest.mark.parametrize("xdt", ["f32", "bf16"])
@pytest.mark.parametrize("B,H,W", [(64, 7, 5), (3, 29, 28), (1, 5, 32), (64, 31, 33), (3, 65, 64)])
@pytest.mark.parametrize("O", [8, 16, 40, 72])
def test_conv_c1_cuda_core_matches_reference(lib, scratch, O, B, H, W, xdt):
    g = torch.Generator(device="cuda").manual_seed(O * 1000 + W)
    partial, counter = scratch
    x = torch.rand(B, H, W, device="cuda", generator=g)
    if xdt == "bf16":
        x = x.bfloat16()
    w = _bf16((O, 9), g, 0.3)
    b = _bf16((O,), g, 0.1)
    y = Out((B, H - 2, W - 2, O), torch.bfloat16)
    assert lib.tfy_conv3x3_c1_fwd(x.data_ptr(), int(xdt == "f32"), w.data_ptr(), b.data_ptr(), y.ptr(), B, H, W, O,
                                  _s()) == 0
    want, mag = ref.conv_c1_fwd(_np(x), _np(w), _np(b))
    _assert_close(y.get(), want, 10 * EPS32 * mag, "c1_fwd")

    dz = _bf16((B, H - 2, W - 2, O), g)
    dw_ref, _, dw_mag, _ = ref.conv_c1_wgrad(_np(x), _np(dz))
    rows_per_warp = math.ceil(B * (H - 2) / (296 * 8))
    d = rows_per_warp * (W - 2) + 8 + 296 + 2
    first = None
    for run in range(RUNS):
        dw = Out((O, 9), torch.bfloat16)
        assert lib.tfy_conv3x3_c1_wgrad(x.data_ptr(), int(xdt == "f32"), dz.data_ptr(), partial.data_ptr(), dw.ptr(),
                                        counter.data_ptr(), B, H, W, O, _s()) == 0
        got = dw.get()
        assert int(counter.item()) == 0
        if first is None:
            first = got
            _assert_close(got, dw_ref, d * EPS32 * dw_mag, "c1_wgrad")
        else:
            assert torch.equal(_bits(got), _bits(first)), f"dW differs on run {run}"


# ---------------------------------------------------------------------------------------------- C_in = 1, tensor cores
@pytest.mark.parametrize("xdt", ["f32", "bf16"])
@pytest.mark.parametrize("B,H,W", [(1, 3, 3), (3, 19, 25), (128, 28, 28), (256, 30, 30)])
def test_conv_c1_tensor_core_matches_reference(lib, B, H, W, xdt):
    O = 32
    g = torch.Generator(device="cuda").manual_seed(B * 100 + H)
    x = torch.rand(B, H, W, device="cuda", generator=g)            # fp32 values that are not bf16 numbers
    if xdt == "bf16":
        x = x.bfloat16()
    w = _bf16((O, 9), g, 0.3)
    b = _bf16((O,), g, 0.1)
    y = Out((B, H - 2, W - 2, O), torch.bfloat16)
    assert lib.tfy_conv3x3_c1_fwd_tc(x.data_ptr(), int(xdt == "f32"), w.data_ptr(), b.data_ptr(), y.ptr(), B, H, W,
                                     _s()) == 0
    want, mag = ref.conv_c1_fwd(_np(x), _np(w), _np(b), round_x=True)
    _assert_close(y.get(), want, 16 * EPS32 * mag, "c1_fwd_tc")

    dz = _bf16((B, H - 2, W - 2, O), g)
    acc = torch.full((160 * 320,), float("nan"), device="cuda")      # every CTA overwrites its own partial
    counter = torch.zeros(1, dtype=torch.int32, device="cuda")
    dw_ref, db_ref, dw_mag, db_mag = ref.conv_c1_wgrad(_np(x), _np(dz), round_x=True)
    n_pix = B * (H - 2) * (W - 2)
    chunks = (n_pix + 127) // 128
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    grid = chunks if chunks <= sms else math.ceil(chunks / math.ceil(chunks / sms))
    d = 128 * math.ceil(chunks / grid) + 160 + 4
    first = None
    for run in range(RUNS):
        dw = Out((O, 9), torch.bfloat16)
        db = Out((O,), torch.bfloat16)
        assert lib.tfy_conv3x3_c1_wgrad_tc(x.data_ptr(), int(xdt == "f32"), dz.data_ptr(), acc.data_ptr(),
                                           counter.data_ptr(), dw.ptr(), db.ptr(), B, H, W, _s()) == 0
        got_w, got_b = dw.get(), db.get()
        assert int(counter.item()) == 0, "the scratch counter must be re-armed"
        if first is None:
            first = (got_w, got_b)
            _assert_close(got_w, dw_ref, d * EPS32 * dw_mag, "c1_wgrad_tc dW")
            _assert_close(got_b, db_ref, d * EPS32 * db_mag, "c1_wgrad_tc db")
        else:
            assert torch.equal(_bits(got_w), _bits(first[0])) and torch.equal(_bits(got_b), _bits(first[1])), run


# ---------------------------------------------------------------------------------------------- bias + act + dropout
# (relu, rate, bias present, y aliasing z, split-K slabs of the _f32 variant)
CONFIGS = [(True, 0.5, True, False, 3), (False, 0.25, False, True, 9), (True, 0.0, True, True, 1),
           (False, 0.0, True, False, 3)]


@pytest.mark.parametrize("rows", [1, 7, 128, 4099])
@pytest.mark.parametrize("C", [8, 24, 64, 128, 256, 520, 1024])
def test_bias_act_drop_forward_and_gated_backward(lib, host, hp, scratch, C, rows):
    g = torch.Generator(device="cuda").manual_seed(C * 7 + rows)
    partial, counter = scratch
    n = rows * C
    for ci, (relu, rate, has_bias, alias, splits) in enumerate(CONFIGS):
        seed = SEED + ci
        u = ref.uniform(host, seed, STEP, n) if rate > 0 else None
        z = _bf16((rows, C), g)
        b = _bf16((C,), g, 0.5) if has_bias else None
        bptr = b.data_ptr() if b is not None else None
        want, want_mask, v = ref.bias_act_drop_fwd(_np(z), _np(b) if b is not None else None, relu, rate, u)
        mask = Out((rows, C), torch.uint8)
        if alias:
            yb = Out((rows, C), torch.bfloat16)
            yb.t.copy_(z)
            zptr = yptr = yb.ptr()
        else:
            yb = Out((rows, C), torch.bfloat16)
            zptr, yptr = z.data_ptr(), yb.ptr()
        assert lib.tfy_bias_act_drop_fwd(zptr, bptr, yptr, mask.ptr(), rows, C, int(relu), rate, seed, hp.data_ptr(),
                                         _s()) == 0
        y = yb.get()
        _assert_close(y, want, 3 * EPS32 * np.abs(want), f"bias_act_drop_fwd cfg {ci}")
        # z + b of two bf16 numbers rounds at most once in fp32 and keeps its sign: the mask is exact
        assert np.array_equal(mask.get().cpu().numpy(), want_mask), f"mask cfg {ci}"

        # _f32: the split-K slabs summed in slab order, then the bias
        slabs = torch.randn(splits, rows, C, device="cuda", generator=g) * (1.0 / splits)
        s, smag = ref.sum_slabs(_np(slabs))
        want32, want_mask32, v32 = ref.bias_act_drop_fwd(s, _np(b) if b is not None else None, relu, rate, u)
        y32, mask32 = Out((rows, C), torch.bfloat16), Out((rows, C), torch.uint8)
        assert lib.tfy_bias_act_drop_fwd_f32(slabs.data_ptr(), bptr, y32.ptr(), mask32.ptr(), rows, C, int(relu),
                                             rate, seed, hp.data_ptr(), splits, _s()) == 0
        e32 = (splits + 3) * EPS32 * (smag + (np.abs(_np(b)) if b is not None else 0.0))
        scale = 1.0 / (1.0 - rate) if rate > 0 else 1.0
        _assert_close(y32.get(), want32, e32 * scale, f"bias_act_drop_fwd_f32 cfg {ci}")
        _assert_mask(mask32.get().cpu().numpy(), want_mask32, v32, e32, f"mask_f32 cfg {ci}")
        if rate > 0:
            kept = u[:n].reshape(rows, C) >= rate
            assert np.array_equal(mask32.get().cpu().numpy() & ~kept, np.zeros((rows, C), np.uint8))

        # gated backward: mask gate, y > 0 gate, no gate, and dbias only (dz = null)
        if ci >= 2:
            continue
        ymask = mask.get()
        dy = _bf16((rows, C), g)
        d = rows + 256 + 592 + 2
        gates = [("mask", ymask, None, _np(ymask).astype(bool)), ("y>0", None, y, _np(y) > 0),
                 ("none", None, None, None), ("dbias only", ymask, None, _np(ymask).astype(bool))]
        for name, m, yg, gate in gates:
            dz_ref, db_ref, db_mag = ref.act_drop_bwd_bias(_np(dy), gate, scale)
            dz = Out((rows, C), torch.bfloat16) if name != "dbias only" else None
            first = None
            for run in range(RUNS):
                db = Out((C,), torch.bfloat16)
                assert lib.tfy_act_drop_bwd_bias(dy.data_ptr(), m.data_ptr() if m is not None else None,
                                                 yg.data_ptr() if yg is not None else None,
                                                 dz.ptr() if dz is not None else None, scale, rows, C,
                                                 partial.data_ptr(), db.ptr(), counter.data_ptr(), _s()) == 0
                got = db.get()
                assert int(counter.item()) == 0
                if first is None:
                    first = got
                    _assert_close(got, db_ref, d * EPS32 * db_mag, f"dbias ({name}, cfg {ci})")
                    if dz is not None:
                        _assert_close(dz.get(), dz_ref, 2 * EPS32 * np.abs(dz_ref), f"dz ({name}, cfg {ci})")
                else:
                    assert torch.equal(_bits(got), _bits(first)), f"dbias ({name}) differs on run {run}"


# ---------------------------------------------------------------------------------------------- 2x2 max-pool
@pytest.mark.parametrize("rate", [0.0, 0.5])
@pytest.mark.parametrize("B,H,W", [(3, 6, 10), (64, 24, 24)])
@pytest.mark.parametrize("C", [8, 24, 64, 136])
def test_pool_forward_and_backward(lib, host, hp, scratch, C, B, H, W, rate):
    g = torch.Generator(device="cuda").manual_seed(C + H + int(rate * 10))
    partial, counter = scratch
    # values on a coarse grid: most 2x2 windows hold exact ties, and max + bias is exact in fp32
    z = (torch.randint(-4, 5, (B, H, W, C), device="cuda", generator=g).float() * 0.5).bfloat16()
    b = (torch.randint(-2, 3, (C,), device="cuda", generator=g).float() * 0.25).bfloat16()
    npool = B * (H // 2) * (W // 2) * C
    u = ref.uniform(host, SEED, STEP, npool) if rate > 0 else None
    want_p, want_code, best = ref.pool_fwd(_np(z), _np(b), rate, u)
    p = Out((B, H // 2, W // 2, C), torch.bfloat16)
    code = Out((B, H // 2, W // 2, C), torch.uint8)
    assert lib.tfy_bias_relu_pool_drop_fwd(z.data_ptr(), b.data_ptr(), p.ptr(), code.ptr(), B, H, W, C, rate, SEED,
                                           hp.data_ptr(), _s()) == 0
    got_code = code.get()
    assert np.array_equal(got_code.cpu().numpy(), want_code), "code bytes"
    ties = (np.stack([_np(z)[:, dy::2, dx::2] for dy in (0, 1) for dx in (0, 1)]) == best[None]).sum(0) > 1
    assert ties.mean() > 0.1, "the input must contain ties inside the windows"
    got_p = p.get()
    if rate == 0:
        assert np.array_equal(_np(got_p), want_p), "pooled maxima"          # max + b is exact: no rounding at all
    else:
        _assert_close(got_p, want_p, 2 * EPS32 * np.abs(want_p), "pool_fwd")
    assert (_np(got_p)[(want_code & 4) == 0] == 0).all()

    scale = 1.0 / (1.0 - rate) if rate > 0 else 1.0
    dp = _bf16((B, H // 2, W // 2, C), g)
    dz_ref, db_ref, db_mag = ref.pool_bwd(_np(dp), want_code, scale)
    d = B * (H // 2) * (W // 2) + 256 + 592 + 2
    first = None
    for run in range(RUNS):
        dz = Out((B, H, W, C), torch.bfloat16)
        db = Out((C,), torch.bfloat16)
        assert lib.tfy_pool_drop_relu_bwd(dp.data_ptr(), got_code.data_ptr(), dz.ptr(), scale, B, H, W, C,
                                          partial.data_ptr(), db.ptr(), counter.data_ptr(), _s()) == 0
        got_db = db.get()
        assert int(counter.item()) == 0
        if first is None:
            first = got_db
            _assert_close(dz.get(), dz_ref, 2 * EPS32 * np.abs(dz_ref), "pool_bwd dz")
            _assert_close(got_db, db_ref, d * EPS32 * db_mag, "pool_bwd dbias")
        else:
            assert torch.equal(_bits(got_db), _bits(first)), f"dbias differs on run {run}"


# ---------------------------------------------------------------------------------------------- softmax head
@pytest.mark.parametrize("C", [2, 17, 100, 1024])
@pytest.mark.parametrize("B", [1, 31, 1000, 1025, 3000])
def test_softmax_xent_matches_reference(lib, B, C):
    g = torch.Generator(device="cuda").manual_seed(B * 3 + C)
    lg = _bf16((B, C), g, 2.0)
    has_bias = (B + C) % 2 == 1
    b = _bf16((C,), g, 0.5) if has_bias else None
    bptr = b.data_ptr() if b is not None else None
    lab = torch.randint(0, C, (B,), device="cuda", generator=g)
    labn = lab.cpu().numpy()
    # the kernel adds the bias in fp32; a sum of two bf16 numbers rounds at most once, so the reference takes that fp32
    # sum as its logits: the argmax (and the hit count) then rests on exact comparisons only
    v32 = lg.float() + (b.float() if b is not None else 0.0)
    loss_ref, d_ref, db_ref, hits, rows, v = ref.softmax_xent(_np(v32), None, labn)
    mx = v.max(1, keepdims=True)
    p = np.exp(v - mx)
    se = p.sum(1, keepdims=True)
    p /= se
    K = 4 + 2.2 * np.abs(v - mx).max()
    onehot = np.zeros_like(p)
    onehot[np.arange(B), labn] = 1.0
    e_d = ((K + C + 3) * p + 2 * np.abs(p - onehot)) * EPS32 / B
    e_db = e_d.sum(0) + B * EPS32 * np.abs(d_ref).sum(0)
    e_row = (K + C + 8) * EPS32 * (1 + np.abs(mx[:, 0]) + np.abs(np.log(se[:, 0])) + np.abs(v[np.arange(B), labn])) \
        + 2 ** -21.41
    e_loss = (e_row.sum() + B * EPS32 * np.abs(rows).sum()) / B + EPS32 * abs(loss_ref)

    first = None
    for run in range(RUNS):
        loss = Out((1,), torch.float32)
        dl = Out((B, C), torch.bfloat16)
        db = Out((C,), torch.bfloat16)
        stats = torch.tensor([5.0, 7.0], device="cuda")                  # accumulates: += [hits, B]
        assert lib.tfy_softmax_xent(lg.data_ptr(), bptr, lab.data_ptr(), loss.ptr(), dl.ptr(), db.ptr(),
                                    stats.data_ptr(), B, C, _s()) == 0
        got = (loss.get(), dl.get(), db.get())
        assert stats.cpu().tolist() == [5.0 + hits, 7.0 + B], (stats.cpu().tolist(), hits, B)
        if first is None:
            first = got
            assert abs(float(got[0]) - loss_ref) <= e_loss, (float(got[0]), loss_ref, e_loss)
            _assert_close(got[1], d_ref, e_d, "dlogits")
            _assert_close(got[2], db_ref, e_db, "dbias")
        else:
            for a, c in zip(got, first):
                assert torch.equal(_bits(a), _bits(c)), f"softmax head differs on run {run}"

    # the weighted kernel with null weights is the same head: the same bits, and stats [hits, B, hits, B]
    loss = Out((1,), torch.float32)
    dl = Out((B, C), torch.bfloat16)
    db = Out((C,), torch.bfloat16)
    stats4 = torch.zeros(4, device="cuda")
    assert lib.tfy_softmax_xent_weighted(lg.data_ptr(), bptr, lab.data_ptr(), None, None, loss.ptr(), dl.ptr(), db.ptr(),
                                         stats4.data_ptr(), B, C, _s()) == 0
    for a, c in zip((loss.get(), dl.get(), db.get()), first):
        assert torch.equal(_bits(a), _bits(c)), "weighted head with null weights"
    assert stats4.cpu().tolist() == [float(hits), float(B), float(hits), float(B)]


# ---------------------------------------------------------------------------------------------- model level
def _generic_model(drop1, drop2):
    from tf_yarn_b200 import keras
    from tf_yarn_b200.keras import layers
    m = keras.Sequential(name="generic_kernels_test")
    m.add(layers.Conv2D(16, (3, 3), activation="relu", input_shape=(30, 30, 1)))
    m.add(layers.MaxPooling2D(pool_size=(2, 2)))
    m.add(layers.Dropout(drop1))
    m.add(layers.Flatten())
    m.add(layers.Dense(96, activation="relu"))
    m.add(layers.Dropout(drop2))
    m.add(layers.Dense(40))
    return m


def _train_generic(fast, drop1, drop2, steps, epochs=1, optimizer=None):
    """Trains the model above from torch seed 7; returns (model, per-batch losses, initial weights)."""
    from tf_yarn_b200 import keras
    torch.manual_seed(7)
    m = _generic_model(drop1, drop2)
    m.compile(loss=keras.losses.SparseCategoricalCrossentropy(from_logits=True),
              optimizer=optimizer or keras.optimizers.Adadelta(1.0), metrics=["accuracy"], use_fast_path=fast)
    w0 = m.get_weights()
    g = torch.Generator().manual_seed(11)
    x = torch.rand(128 * steps, 30, 30, 1, generator=g)
    y = torch.randint(0, 40, (128 * steps,), generator=g)
    losses = []

    class Rec(keras.callbacks.Callback):
        needs_batch_logs = True

        def on_train_batch_end(self, batch, logs=None):
            losses.append(logs["loss"])
    m.fit(x, y, batch_size=128, epochs=epochs, shuffle=False, verbose=0, callbacks=[Rec()])
    torch.cuda.synchronize()
    return m, losses, w0


def test_generic_model_training_is_bitwise_reproducible(monkeypatch):
    """Conv(C_in 1 -> 16) + pool + dropout, split-K Dense + dropout, a 40-class unfused head: the step runs cuDNN +
    tfy_bias_relu_pool_drop_fwd, the split-K GEMM + tfy_bias_act_drop_fwd_f32, tfy_softmax_xent, tfy_act_drop_bwd_bias,
    tfy_pool_drop_relu_bwd and tfy_conv3x3_c1_wgrad.  Two trainings must end with bit-identical losses and
    parameters."""
    from tf_yarn_b200.keras.fastpath import FastSequentialEngine
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)

    def train():
        m, losses, _ = _train_generic(True, 0.25, 0.5, steps=6, epochs=2)
        assert isinstance(m._engine, FastSequentialEngine)
        kinds = [(st.kind, getattr(st, "pool", None)) for st in m._engine.plan]
        assert kinds == [("conv", True), ("flatten", None), ("dense", None), ("head", None)], kinds
        return losses, m._engine.fused.flat_params.clone(), [torch.as_tensor(w) for w in m.get_weights()]

    l1, p1, w1 = train()
    l2, p2, w2 = train()
    assert all(math.isfinite(v) for v in l1)
    assert l1 == l2, (l1, l2)
    assert torch.equal(_bits(p1), _bits(p2))
    for a, b in zip(w1, w2):
        assert torch.equal(_bits(a), _bits(b))


def test_generic_model_matches_autograd_engine(monkeypatch):
    """Same init, same batches, dropout off: the generic-kernel plan must track the autograd engine.  Plain SGD, so
    that each parameter's update is proportional to its summed gradients (Adadelta's early steps are sign-like: a
    near-zero bias gradient that bf16 rounding flips moves the weight by a full step either way)."""
    from tf_yarn_b200 import keras
    from tf_yarn_b200.keras.fastpath import FastSequentialEngine
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    m_fast, l_fast, w0 = _train_generic(True, 0.0, 0.0, steps=4, optimizer=keras.optimizers.SGD(0.05))
    m_ref, l_ref, w0_ref = _train_generic(False, 0.0, 0.0, steps=4, optimizer=keras.optimizers.SGD(0.05))
    assert isinstance(m_fast._engine, FastSequentialEngine)
    assert not isinstance(m_ref._engine, FastSequentialEngine)
    assert len(l_fast) == len(l_ref) == 4
    for a, b in zip(l_fast, l_ref):
        assert math.isfinite(a) and abs(a - b) < 0.03 * max(1.0, abs(b)), (l_fast, l_ref)
    for a, b, a0, b0 in zip(m_fast.get_weights(), m_ref.get_weights(), w0, w0_ref):
        assert np.array_equal(a0, b0)
        da, db = a - a0, b - b0
        # bf16 activations and gradients: about 1 % per step, compounded over 4 steps
        assert np.abs(da - db).max() <= 0.1 * np.abs(db).max(), (a.shape, np.abs(da - db).max(), np.abs(db).max())
