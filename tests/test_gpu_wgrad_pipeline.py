"""GPU (-m gpu): the weight-gradient mainloop (csrc/wgrad_tc.cu) at the places its stage rings can go wrong.

The loaders copy fp32 rows into a ring of shared-memory stages with cp.async (rows at or beyond K are zero-filled, not
read), split them into a ring of bf16 hi/lo plane stages, and the consumers keep one wgmma group in flight.  The batch
kernel carries both rings' positions from slab to slab and from problem to problem.  Every result is checked against
fp64 at 2e-5 of the output scale, and a second call must give the same bits."""
import pytest
import torch

from alignn_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _check(out, ref):
    scale = max(ref.abs().max().item(), 1e-30)
    err = (out.double() - ref).abs().max().item()
    assert err <= 2e-5 * scale, (err, scale)


def _batch(d, Ks, seed, wide_a=False, ldb=None):
    g = torch.Generator(device="cpu").manual_seed(seed)
    problems, refs = [], []
    for i, K in enumerate(Ks):
        if wide_a:                                             # A: column block i % 4 of a [K, 4d] matrix (GP)
            A = torch.randn(K, 4 * d, generator=g).to(DEV)[:, (i % 4) * d:(i % 4 + 1) * d]
        else:
            A = torch.randn(K, d, generator=g).to(DEV)
        B = torch.randn(K, ldb or d, generator=g).to(DEV)[:, :d]
        problems.append((A, B, torch.full((d, d), float("nan"), device=DEV)))
        refs.append(A.double().t() @ B.double())
    return problems, refs


def _run_twice(problems):
    ops.wgrad_batch(problems)
    first = [out.clone() for _, _, out in problems]
    ops.wgrad_batch(problems)
    for a, (_, _, out) in zip(first, problems):
        assert torch.equal(a, out)
    return first


@pytest.mark.parametrize("d", [256, 128, 64, 32])
def test_batch_ring_phase_carries_across_slabs_and_problems(d):
    """A small batch: every CTA column runs several slabs of different problems.  Chunk counts are multiples of neither
    ring's stage count nor of the promotion interval (8 chunks)."""
    Ks = [32 * c + r for c, r in ((1, 0), (3, 5), (5, 31), (7, 1), (9, 0), (11, 17), (13, 3), (17, 30), (19, 0),
                                  (25, 9), (29, 0), (37, 2), (41, 11), (53, 0), (61, 7), (67, 0))] * 2
    problems, refs = _batch(d, Ks, seed=d)
    for out, ref in zip(_run_twice(problems), refs):
        _check(out, ref)


@pytest.mark.parametrize("d", [256, 64])
def test_batch_short_and_zero_problems_at_exact_size(d):
    """K % 32 != 0 with A and B allocated at exactly K rows: the rows past K must be zero-filled, never read."""
    Ks = [1, 31, 0, 33, 0, 65, 1, 95, 31, 0, 33]
    problems, refs = _batch(d, Ks, seed=7 + d)
    for out, ref, K in zip(_run_twice(problems), refs, Ks):
        if K == 0:
            assert torch.equal(out, torch.zeros(d, d, device=DEV))
        else:
            _check(out, ref)


@pytest.mark.parametrize("K", [1, 31, 33])
@pytest.mark.parametrize("d", [256, 128, 64, 32])
def test_single_problem_short_k(K, d):
    g = torch.Generator(device="cpu").manual_seed(K * d)
    A, B = torch.randn(K, d, generator=g).to(DEV), torch.randn(K, d, generator=g).to(DEV)
    out = ops.wgrad(A, B, 1)
    _check(out, A.double().t() @ B.double())
    assert torch.equal(out, ops.wgrad(A, B, 1))


@pytest.mark.parametrize("d", [256, 64, 32])
def test_batch_strided_views(d):
    """A is a column block of a [K, 4d] matrix and B a column slice with row stride 3d."""
    Ks = [23040, 1920, 777, 4099, 33, 1920]
    problems, refs = _batch(d, Ks, seed=11 + d, wide_a=True, ldb=3 * d)
    for out, ref in zip(_run_twice(problems), refs):
        _check(out, ref)


@pytest.mark.parametrize("K", [23040, 276480])
def test_single_problem_four_groups(K):
    """The double backward's form: four weight gradients stacked along A's columns, one launch."""
    g = torch.Generator(device="cpu").manual_seed(K)
    d = 256
    A = torch.randn(K, 4 * d, generator=g).to(DEV)
    B = torch.randn(K, d, generator=g).to(DEV)
    out = ops.wgrad(A, B, 4)
    _check(out, A.double().t() @ B.double())
    assert torch.equal(out, ops.wgrad(A, B, 4))
