"""Bit-level GPU tests of the split-K Dense GEMM's fp32 slabs (tfy_gemm_bf16 with an fp32 workspace).

When the grid of 128 x 128 tiles times K-slices leaves most of the SMs idle, the kernel splits every tile over a 2- or
4-CTA cluster (64-row halves, and 64-column halves when the grid still fits one wave), with each operand box
multicast to the CTAs that share it.  Each output element still sees the same k16 steps, in the same order, in one
fp32 accumulator, so the slabs must not change by a single bit.  tests/golden/gemm_splitk_b128_sha256.json holds the
SHA-256 of the slabs written by the one-tile-per-CTA kernel: at the MNIST Dense layer's 128 x 128 x 9216 for 24 and 36
K-slices, and at ragged shapes, each at the split the fast path picks for it.
"""
import hashlib
import json
import os

import pytest
import torch

from tf_yarn_b200.keras import fastpath

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gemm_splitk_b128_sha256.json")
BF16 = torch.bfloat16
RAGGED = [(m, n, k) for m in (2, 3, 100, 128) for n in (10, 96, 128, 136) for k in (9216, 9224)]


@pytest.fixture(scope="module")
def lib():
    from tf_yarn_b200.ops import native
    return native.load()


def _inputs(M, N, K, seed):
    """x ~ N(0, 1), W ~ N(0, 0.02), seeded on the CPU: not integer-valued, so the digests pin wgmma's rounding."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, K, generator=g).to(BF16).cuda()
    w = (torch.randn(N, K, generator=g) * 0.02).to(BF16).cuda()
    return x, w


def _slabs(lib, x, w, split, launch=None):
    M, K = x.shape
    N = w.shape[0]
    n = int(lib.tfy_gemm_bf16_splitk_slabs(K, split))
    acc = torch.full((n, M, N), float("nan"), dtype=torch.float32, device="cuda")

    def run():
        return lib.tfy_gemm_bf16(x.data_ptr(), w.data_ptr(), None, acc.data_ptr(), None, M, N, K, K, K, N, 0, split,
                                 torch.cuda.current_stream().cuda_stream)
    assert (launch or (lambda f, _: f()))(run, acc) == 0
    torch.cuda.synchronize()
    return acc


def _sha(t):
    return hashlib.sha256(t.contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest()


def _name(M, N, K):
    return f"m{M}_n{N}_k{K}"


def splitk_digests(lib):
    """SHA-256 of the slabs: 128 x 128 x 9216 at 24 and 36 K-slices (seed 41), and every RAGGED shape at the fast
    path's split (seed 43)."""
    out = {}
    x, w = _inputs(128, 128, 9216, 41)
    for split in (24, 36):
        out[f"b128_split{split}"] = _sha(_slabs(lib, x, w, split))
    for M, N, K in RAGGED:
        x, w = _inputs(M, N, K, 43)
        out[_name(M, N, K)] = _sha(_slabs(lib, x, w, fastpath.FastSequentialEngine._split_k(M, N, K)))
    return out


def test_engine_splits_of_the_mnist_dense_layer():
    assert fastpath.FastSequentialEngine._split_k(128, 128, 9216) == 24
    assert fastpath.FastSequentialEngine._split_k(128, 128, 9216, 4) == 36


def test_slabs_bit_identical_to_recorded_digests(lib):
    with open(GOLDEN) as f:
        want = json.load(f)
    got = splitk_digests(lib)
    assert sorted(got) == sorted(k for k in want if k != "note")
    bad = {k: (got[k], want[k]) for k in got if got[k] != want[k]}
    assert not bad, bad


@pytest.mark.parametrize("split", [24, 36])
def test_slabs_repeat_eagerly_and_under_graph_replay(lib, split):
    """Two eager launches and a CUDA-graph replay (the cluster launch is captured like any other) write the same
    bytes."""
    x, w = _inputs(128, 128, 9216, 47)
    a = _slabs(lib, x, w, split)
    b = _slabs(lib, x, w, split)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))

    def in_graph(run, acc):
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s):
            assert run() == 0                                   # warm-up on the capture stream
            torch.cuda.synchronize()
            with torch.cuda.graph(graph, stream=s):
                rc = run()
        torch.cuda.current_stream().wait_stream(s)
        acc.fill_(float("nan"))                                 # only the replays write the slabs checked below
        for _ in range(2):
            graph.replay()
        torch.cuda.synchronize()
        return rc
    c = _slabs(lib, x, w, split, launch=in_graph)
    assert torch.equal(a.view(torch.int32), c.view(torch.int32))
    assert not torch.isnan(a).any()
