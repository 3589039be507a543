"""Reference of the collective kernels (ops/csrc/tfy_comm.cu) and the case table their multi-GPU test runs.  Plain
NumPy: nothing here imports tf_yarn_b200 or touches a GPU.

* Inputs: every rank's input of a case is a pure function of ``(case, rank, seed)``, so the process that judges a
  run rebuilds all ranks' inputs without receiving them.
* P2P all-reduce (one-shot K1, two-shot K2, and the gradient of the fused step K4 in P2P mode): the kernel starts from
  +0.0f, adds the ranks in the order 0 ... world-1 in fp32, multiplies by the fp32 scale and rounds to nearest even
  when it packs bf16.  :func:`p2p_allreduce` does exactly that in float32 NumPy; the kernel must match it bit for bit.
* NVLS (K3, and K4 in NVLS mode): the switch's summation order, and its rounding of a bf16 result, are not
  specified.  :func:`nvls_bound` bounds the distance of any such result from the exact sum.
"""
from __future__ import annotations

import math
import zlib
from dataclasses import dataclass
from typing import Dict, List, Tuple

import numpy as np

PACK = {"bf16": 8, "f32": 4}         # elements per 16-byte pack
ESIZE = {"bf16": 2, "f32": 4}
ALGOS = ("oneshot", "twoshot", "nvls")
NUM_SMS = 132                        # TFY_NUM_SMS
DEFAULT_BLOCK = 512
U = 4                                # packs in flight per thread in K2 / K3
GRID_PASS = 2 * NUM_SMS * DEFAULT_BLOCK * U   # packs of one pass of the default two-shot grid: 264 x 512 x 4
MNIST_PARAMS = 1_199_882
WORLDS = (1, 2, 3, 5, 8)
GUARD = 4096                          # bytes of sentinel on each side of every buffer
ALIGN = 256
SEED = 20261018

U32 = 2.0 ** -24
SUB32 = 2.0 ** -149


# ---------------------------------------------------------------------------------------------------------------
# host-side launch geometry (tfy_pick_grid)
# ---------------------------------------------------------------------------------------------------------------
def pick_grid(work: int, block: int, max_grid: int) -> int:
    return max(1, min(max_grid, -(-work // block)))


def allreduce_default_grid(algo: str, n_packs: int, world: int, block: int = DEFAULT_BLOCK) -> int:
    work = n_packs if algo == "oneshot" else n_packs // world
    return pick_grid(work, block, 2 * NUM_SMS)


# ---------------------------------------------------------------------------------------------------------------
# the case table
# ---------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Size:
    """A buffer size: ``shard`` packs per rank (two-shot / NVLS), the buffer is ``world * shard`` packs; ``packs``
    overrides that for one-shot's one-pack case.  ``grid`` / ``block`` 0 are the host's choice."""
    name: str
    shard: int
    grid: int = 0
    block: int = 0
    oneshot_packs: int = 0


def sizes(world: int, dtype: str) -> List[Size]:
    mnist_shard = -(-MNIST_PARAMS // (PACK[dtype] * world))
    return [
        Size("min", 1, oneshot_packs=1),                       # 1 pack (one-shot), 1 pack per rank
        Size("sub_thread", 37),                                # fewer packs per rank than threads in the grid
        Size("u_tail", 2 * 2 * NUM_SMS * DEFAULT_BLOCK + 777),  # past one thread per pack, inside a U = 4 batch
        Size("multi_pass", GRID_PASS + 1234),                  # past one pass of the default grid
        Size("mnist", mnist_shard),                            # the MNIST-CNN's gradient, padded to world packs
        Size("grid1_block32", 32 * U * 3 + 32 * 2 + 5, grid=1, block=32),  # wraps 3 times, ends inside a batch
        Size("grid3_block64", 2 * 3 * 64 * U + 3 * 64 + 11, grid=3, block=64),
    ]


VALUES = ("gauss", "special", "int")


@dataclass(frozen=True)
class Case:
    dtype: str
    algo: str
    scale: str       # "one" or "mean": fl32(1/world); at one rank, where that is 1, fl32(1/3) stands in (not a power
                     # of two, so bf16 results round)
    size: str
    values: str

    @property
    def id(self) -> str:
        return f"{self.dtype}-{self.algo}-{self.scale}-{self.size}-{self.values}"

    @property
    def input_key(self) -> str:
        """What the inputs depend on: not the algorithm nor the scale, so every algorithm reduces the same data."""
        return f"{self.dtype}-{self.size}-{self.values}"


def scale_value(scale: str, world: int) -> float:
    if scale == "one":
        return 1.0
    return float(np.float32(1.0 / (world if world > 1 else 3)))


def cases() -> List[Case]:
    """Every all-reduce case; the sizes they name depend on the world (``size_of``).  Gaussian values at every size,
    the special and integer values at the small sizes."""
    out = []
    for dtype in ("bf16", "f32"):
        for algo in ALGOS:
            for scale in ("one", "mean"):
                for s in sizes(2, dtype):
                    out.append(Case(dtype, algo, scale, s.name, "gauss"))
                for s in ("sub_thread", "grid1_block32"):
                    for v in ("special", "int"):
                        out.append(Case(dtype, algo, scale, s, v))
    return out


CASES = cases()


def size_of(case: Case, world: int) -> Size:
    return {s.name: s for s in sizes(world, case.dtype)}[case.size]


def n_packs(case: Case, world: int) -> int:
    s = size_of(case, world)
    if case.algo == "oneshot" and s.oneshot_packs:
        return s.oneshot_packs
    return s.shard * world


def n_elems(case: Case, world: int) -> int:
    return n_packs(case, world) * PACK[case.dtype]


# ---------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------
def _rng(key: str, rank: int, seed: int = SEED) -> np.random.Generator:
    return np.random.default_rng([seed, zlib.crc32(key.encode()), rank])


def bf16_bits(x: np.ndarray) -> np.ndarray:
    """float32 -> bf16 bit patterns, round to nearest even (``__floats2bfloat162_rn``); NaN -> canonical 0x7fff."""
    b = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    r = ((b + 0x7FFF + ((b >> 16) & 1)) >> 16).astype(np.uint16)
    return np.where(np.isnan(x), np.uint16(0x7FFF), r)


def bf16_to_f32(bits: np.ndarray) -> np.ndarray:
    return (np.asarray(bits, np.uint16).astype(np.uint32) << 16).view(np.float32)


def values(kind: str, dtype: str, n: int, key: str, rank: int, seed: int = SEED) -> np.ndarray:
    """Rank ``rank``'s input: float32 values, each exactly representable in ``dtype``.

    * gauss: Gaussian values times 2^k, k uniform in [-20, 20]; 3 % exact +0 or -0.
    * special: by element index mod 8 (the same on every rank, so the ranks combine): +-0 with a rank-dependent sign,
      dtype subnormals, 1.5 * 2^127 of one sign on every rank (any two of them overflow), +inf on rank 0 and -inf on
      rank 1 (NaN at two ranks or more), +-inf on every rank, and Gaussian values between them.
    * int: integers small enough that every sum is exact in ``dtype`` (|x| <= 16 in bf16, 2^20 in fp32).
    """
    rs = _rng(key, rank, seed)
    if kind == "int":
        lim = 16 if dtype == "bf16" else 1 << 20
        x = rs.integers(-lim, lim + 1, n).astype(np.float32)
    else:
        x = (rs.standard_normal(n) * np.exp2(rs.integers(-20, 21, n))).astype(np.float32)
        u = rs.random(n)
        x[u < 0.015] = 0.0
        x[(u >= 0.015) & (u < 0.03)] = -0.0
        if kind == "special":
            i = np.arange(n) % 8
            sign = np.where(rs.random(n) < 0.5, -1.0, 1.0).astype(np.float32)
            x[i == 0] = np.float32(0.0) * (1.0 if rank % 2 else -1.0)
            tiny = 2.0 ** -133 if dtype == "bf16" else 2.0 ** -149
            k = rs.integers(1, 128 if dtype == "bf16" else 1 << 20, n)
            x[i == 1] = (sign * k * tiny).astype(np.float32)[i == 1]
            fixed_sign = np.where((np.arange(n) // 8) % 2 == 0, 1.0, -1.0).astype(np.float32)
            x[i == 2] = (fixed_sign * np.float32(1.5 * 2.0 ** 127))[i == 2]
            x[i == 3] = np.float32(np.inf) if rank == 0 else (np.float32(-np.inf) if rank == 1 else np.float32(1.0))
            x[i == 4] = (fixed_sign * np.float32(np.inf))[i == 4]
    if dtype == "bf16":
        x = bf16_to_f32(bf16_bits(x))
    return x


def case_input(case: Case, world: int, rank: int, seed: int = SEED) -> np.ndarray:
    return values(case.values, case.dtype, n_elems(case, world), f"{world}-{case.input_key}-{case.algo == 'oneshot'}",
                  rank, seed)


def to_bits(x: np.ndarray, dtype: str) -> np.ndarray:
    """The buffer's bytes as integers: uint16 bf16 patterns or uint32 fp32 patterns."""
    return bf16_bits(x) if dtype == "bf16" else np.ascontiguousarray(x, np.float32).view(np.uint32)


# ---------------------------------------------------------------------------------------------------------------
# emulation and bounds
# ---------------------------------------------------------------------------------------------------------------
def p2p_sum(xs) -> np.ndarray:
    """fp32 sum in rank order from +0.0f, as tfy_reduce_pack_rt computes it (P2P mode)."""
    acc = None
    for x in xs:
        x = np.asarray(x, np.float32)
        acc = np.float32(0.0) + x if acc is None else acc + x
    return acc


def p2p_allreduce(xs, scale: float, dtype: str) -> np.ndarray:
    """The bits a P2P all-reduce (K1 / K2) leaves: rank-order fp32 sum, times fp32(scale), packed to ``dtype``."""
    with np.errstate(over="ignore", invalid="ignore"):
        r = p2p_sum(xs) * np.float32(scale)
    return to_bits(r, dtype)


def exact_sums(xs) -> Tuple[np.ndarray, np.ndarray]:
    """The float64 sum of the ranks and the sum of their magnitudes (exact for up to 8 fp32 addends of the ranges used
    here, whose magnitudes span less than 2^52)."""
    s = a = None
    with np.errstate(invalid="ignore"):
        for x in xs:
            x = np.asarray(x, np.float64)
            s = x.copy() if s is None else s + x
            a = np.abs(x) if a is None else a + np.abs(x)
    return s, a


def bf16_ulp(mag) -> np.ndarray:
    """The spacing of bf16 values at magnitude ``mag`` (the subnormal spacing 2^-133 below 2^-126)."""
    mag = np.asarray(mag, np.float64)
    e = np.floor(np.log2(np.where(mag > 0, mag, 1.0)))
    return np.exp2(np.maximum(np.where(mag > 0, e, -126.0), -126.0) - 7.0)


def nvls_bound(s: np.ndarray, a: np.ndarray, world: int, scale: float, dtype: str) -> Tuple[np.ndarray, np.ndarray]:
    """Centre and radius of the results an NVLS all-reduce may return for exact sum ``s`` with magnitude sum ``a``.

    The switch adds ``world`` fp32 values in some order: ``world - 1`` roundings, at most gamma_{world-1} * a, plus
    2^-149 each in the subnormal range.  A bf16 result is rounded by the switch in an unspecified direction: one bf16
    ulp.  A scale other than 1 is applied by the kernel: one fp32 multiply, and for bf16 a second, round-to-nearest
    packing (half an ulp)."""
    k = world - 1
    gamma = k * U32 / (1.0 - k * U32)
    e = gamma * a + k * SUB32
    if dtype == "bf16":
        e = e + bf16_ulp(np.abs(s) + e)
    if scale != 1.0:
        sc = float(np.float32(scale))
        e = sc * e + U32 * sc * (np.abs(s) + e) + SUB32
        s = s * sc
        if dtype == "bf16":
            e = e + 0.5 * bf16_ulp(np.abs(s) + e)
    return s, e


def float_of(bits: np.ndarray, dtype: str) -> np.ndarray:
    return bf16_to_f32(bits) if dtype == "bf16" else np.asarray(bits, np.uint32).view(np.float32)


# ---------------------------------------------------------------------------------------------------------------
# the worker's arena: one region per buffer kind, each between two guard bands
# ---------------------------------------------------------------------------------------------------------------
def _up(x: int, a: int = ALIGN) -> int:
    return (x + a - 1) // a * a


def guarded(nbytes: int) -> Tuple[int, int]:
    """(offset of the buffer inside its guarded region, region bytes): GUARD | buffer | GUARD."""
    return GUARD, _up(GUARD + nbytes + GUARD)


BCAST_PACKS = (1, 37, 2 * NUM_SMS * DEFAULT_BLOCK + 11)   # 1 pack, odd, past one pass of the 132 x 512 grid
GATHER_PACKS = (1, 37, 2 * NUM_SMS * DEFAULT_BLOCK + 11)


def region_bytes(world: int) -> Dict[str, int]:
    """Bytes of the guarded regions the worker allocates: the all-reduce buffer and one-shot's output (sized for the
    largest case), the broadcast buffer and the all-gather buffer."""
    ar = max(n_packs(c, world) * 16 for c in CASES)
    return {"ar": guarded(ar)[1], "out": guarded(ar)[1], "bcast": guarded(max(BCAST_PACKS) * 16)[1],
            "gather": guarded(max(GATHER_PACKS) * 16 * world)[1]}


ARENA_BYTES = 1 << 30                 # the worker's arena (besides the communicator's fusion buffer)
FUSION_BYTES = 1 << 20                # the list API's fusion buffer in the worker: small, so big tensors go in pieces


def sentinel(nbytes: int, rank: int) -> np.ndarray:
    """The guard-band pattern of ``rank``: distinct per rank, so a peer's stray store cannot hide."""
    return ((np.arange(nbytes, dtype=np.uint32) * 37 + 0xA5 + 16 * rank) & 0xFF).astype(np.uint8)


def junk(nbytes: int, rank: int, tag: str) -> np.ndarray:
    """What a receive buffer holds before a broadcast or all-gather: bytes distinct per rank and buffer."""
    return _rng("junk-" + tag, rank).integers(0, 256, nbytes, dtype=np.uint8)


def payload(nbytes: int, key: str, rank: int) -> np.ndarray:
    return _rng("payload-" + key, rank).integers(0, 256, nbytes, dtype=np.uint8)


def sha(a) -> str:
    import hashlib
    return hashlib.sha256(np.ascontiguousarray(a).view(np.uint8).tobytes()).hexdigest()


# ---------------------------------------------------------------------------------------------------------------
# the fused step at several ranks
# ---------------------------------------------------------------------------------------------------------------
SMALL_SHAPES = [(33, 17), (129,), (7, 5, 3), (1,), (5,)]
MNIST_SHAPES = [(32, 3, 3, 1), (32,), (64, 3, 3, 32), (64,), (9216, 128), (128,), (128, 10), (10,)]
PAIRS = [("f32", "f32"), ("bf16", "bf16"), ("bf16", "f32"), ("f32", "bf16")]
STEP_SCALES = (1.0, 0.25, 1.0)


def flat_size(shapes, world: int) -> int:
    """FusedShardedOptimizer's flat buffer length: every tensor padded to 8 elements, the total to 8 * world."""
    n = sum(-(-math.prod(s) // 8) * 8 for s in shapes)
    per = 8 * world
    return -(-n // per) * per


def elem3_cuts(shard_n: int, world: int) -> Tuple[int, int]:
    """Cuts of the three-launch ranged step: [0, c1) ends 1/3 of the way into rank 1's shard (it straddles the
    boundary of shard 0), [c1, c2) lies inside rank 1's shard (every other rank has nothing to do)."""
    g = shard_n // 8
    base = shard_n if world > 1 else 0
    c1 = base + 8 * (g // 3)
    c2 = c1 + 8 * (g // 5 + 1)
    return c1, c2


def step_grads(n: int, key: str, rank: int, step: int) -> np.ndarray:
    """Rank ``rank``'s float32 gradient at ``step``: Gaussian with exact +-0, values whose square underflows in fp32
    and large ones, as the single-GPU test draws them."""
    rs = _rng(f"grad-{key}-{step}", rank)
    g = (rs.standard_normal(n) * 0.5).astype(np.float32)
    u = rs.random(n)
    sign = np.where(rs.random(n) < 0.5, -1.0, 1.0).astype(np.float32)
    g[u < 0.04] = 0.0
    g[(u >= 0.04) & (u < 0.08)] = -0.0
    tiny = (u >= 0.08) & (u < 0.12)
    g[tiny] = sign[tiny] * np.float32(1e-25) * (1 + rs.random(int(tiny.sum()))).astype(np.float32)
    big = (u >= 0.12) & (u < 0.14)
    g[big] = sign[big] * np.float32(1e3) * (1 + rs.random(int(big.sum()))).astype(np.float32)
    return g


def initial_master(n: int, key: str, ftrl: bool) -> np.ndarray:
    """The full fp32 master of a fused-step case (the same on every rank); FTRL: one in ten exactly 0."""
    rs = _rng(f"master-{key}", 0)
    p = (rs.standard_normal(n) * 0.3).astype(np.float32)
    if ftrl:
        p[rs.random(n) < 0.1] = 0.0
    return p


def as_dtype(x: np.ndarray, dtype: str) -> np.ndarray:
    """float32 values as ``dtype`` holds them, widened back to float32."""
    return bf16_to_f32(bf16_bits(x)) if dtype == "bf16" else np.asarray(x, np.float32)


@dataclass(frozen=True)
class StepCase:
    """One multi-GPU fused-step run: ``variant`` of fused_step_reference.VARIANTS, ``pair`` = (gradient, parameter)
    dtypes, ``split`` = how a step is launched, ``mode`` = p2p or nvls, ``layout`` = small, mnist or flat (one flat
    tensor, for the cross-check against LOCAL), ``sched`` = the learning rate follows SCHEDULES[variant],
    ``solo_grad`` = only rank 0 has a gradient (no -0) and grad_scale = world."""
    variant: str
    pair: Tuple[str, str]
    split: str
    mode: str
    layout: str
    sched: bool = False
    solo_grad: bool = False

    @property
    def id(self) -> str:
        tags = ["sched"] * self.sched + ["solo"] * self.solo_grad
        return "-".join([self.variant, *self.pair, self.split, self.mode, self.layout, *tags])


SPLITS = ("full", "elem3", "groups2")
SCHEDULES = {"adam": ("ExponentialDecay", dict(initial_learning_rate=1e-3, decay_steps=1, decay_rate=0.5)),
             "sgd_momentum_dampening": ("PiecewiseConstantDecay", dict(boundaries=[1], values=[0.05, 0.01]))}


def step_cases(world: int, multicast: bool) -> List[StepCase]:
    """Every variant at every dtype pair and split in P2P mode; in NVLS mode (with multicast) at the (bf16, bf16) and
    (fp32, fp32) pairs; two scheduled optimizers; the MNIST layout; the cross-check against LOCAL."""
    from fused_step_reference import VARIANTS
    same = [("bf16", "bf16"), ("f32", "f32")]
    out = []
    for v in sorted(VARIANTS):
        for pair in PAIRS:
            for split in SPLITS:
                out.append(StepCase(v, pair, split, "p2p", "small"))
        if multicast:
            for pair in same:
                for split in SPLITS:
                    out.append(StepCase(v, pair, split, "nvls", "small"))
    for v in sorted(SCHEDULES):
        for pair in same:
            out.append(StepCase(v, pair, "full", "p2p", "small", sched=True))
    for v in sorted(VARIANTS):
        for pair in same:
            out.append(StepCase(v, pair, "full", "p2p", "mnist"))
            out.append(StepCase(v, pair, "full", "p2p", "flat", solo_grad=True))
    return out


def layout_shapes(layout: str, world: int):
    if layout == "small":
        return SMALL_SHAPES
    if layout == "mnist":
        return MNIST_SHAPES
    return [(flat_size(SMALL_SHAPES, world),)]


def case_grads(n: int, case: StepCase, rank: int, step: int) -> np.ndarray:
    """Rank ``rank``'s gradient buffer at ``step``, as float32 values (the worker casts it to the gradient dtype)."""
    if case.solo_grad:
        if rank:
            return np.zeros(n, np.float32)
        g = step_grads(n, case.layout, 0, step)
        g[g == 0] = 0.0                      # no -0: 0 + (-0) is +0 at two ranks or more
        return g
    return step_grads(n, case.layout, rank, step)


def step_pieces(split: str, shard_n: int, world: int):
    """The launches of one step: (how, a, b, advance); ``range`` takes flat element bounds, ``groups`` shard-relative
    groups of 8."""
    if split == "full":
        return [("full", 0, 0, True)]
    if split == "elem3":
        c1, c2 = elem3_cuts(shard_n, world)
        n = shard_n * world
        return [("range", 0, c1, False), ("range", c1, c2, False), ("range", c2, n, True)]
    G = shard_n // 8
    return [("groups", 0, G // 3, False), ("groups", G // 3, G, True)]


def piece_span(piece, shard_n: int, rank: int) -> Tuple[int, int]:
    """The shard-relative element range [lo, hi) of rank ``rank``'s shard that a launch updates."""
    how, a, b, _ = piece
    if how == "full":
        return 0, shard_n
    if how == "groups":
        return 8 * a, 8 * b
    s0 = rank * shard_n
    lo, hi = min(max(a - s0, 0), shard_n), min(max(b - s0, 0), shard_n)
    return lo, max(lo, hi)


# ---------------------------------------------------------------------------------------------------------------
# the Communicator's list API
# ---------------------------------------------------------------------------------------------------------------
# (name, dtype, shape, non-contiguous): every dtype the list API takes, a strided view, an empty tensor and one larger
# than the worker's fusion buffer (FUSION_BYTES / 4 = 262,144 fp32 elements), which goes through it in pieces
LIST_TENSORS = [("bf16", "bf16", (37, 5), False), ("f32", "f32", (1000,), False), ("f16", "f16", (300,), False),
                ("strided", "f32", (64, 16), True), ("empty", "f32", (0,), False),
                ("big", "f32", (300_000,), False)]


def list_values(name: str, dtype: str, shape, rank: int, tag: str) -> np.ndarray:
    """Rank ``rank``'s values of list tensor ``name``: float32 (bf16-representable for bf16) or float16."""
    n = math.prod(shape)
    rs = _rng(f"list-{tag}-{name}", rank)
    if dtype == "f16":
        return (rs.standard_normal(n) * 4).astype(np.float16).reshape(shape)
    x = values("gauss", dtype, n, f"list-{tag}-{name}", rank)
    return x.reshape(shape)


def wide_values(dtype, rank: int) -> np.ndarray:
    """Integer values around 2^40 + rank, as float64 or int64: every sum of up to 8 ranks is exact in any order."""
    return (np.int64(1) << 40) + rank + np.arange(-32, 32, dtype=np.int64) * 1024 if dtype == np.int64 else \
        (2.0 ** 40 + rank + np.arange(-32, 32) * 1024.0).astype(np.float64)
