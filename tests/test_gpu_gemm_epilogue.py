"""GPU (-m gpu): the row-oriented epilogue of the Linear-layer GEMM (csrc/gemm_tc.cu) against fp64.

Each consumer warp stages its 16 accumulator rows through shared memory and writes them row by row, BN / 4 lanes per
row, with the addend rows of several rows loaded before the first store.  These cases cover what that layout depends
on: ragged and multi-wave M, every column tile width, gathered addends with repeated and shared indices, strided
addend and output views, and the column statistics.  Tolerances as in test_gpu_gemm.py."""
import pytest
import torch

from alignn_b200 import _lib, ops

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# 132 SMs, 128-row tiles: 265 N=32 tiles is more than two waves of CTAs, and the last tile holds 77 rows
MANY = 2 * 132 * 128 + 77


def _operands(M, N, K, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    A = torch.randn(M, K, generator=g).to(DEV)
    W = (torch.randn(N, K, generator=g) / K ** 0.5).to(DEV)
    bias = torch.randn(N, generator=g).to(DEV)
    return g, A, W, bias


@pytest.mark.parametrize("M", [1, 63, 64, 127, 129, MANY])
@pytest.mark.parametrize("N,K", [(32, 32), (64, 256), (96, 32), (128, 1024), (256, 256), (1024, 32)])
def test_ragged_rows_every_tile_width(M, N, K):
    g, A, W, bias = _operands(M, N, K, M + N + K)
    R = torch.randn(M, N, generator=g).to(DEV)
    img = ops.WeightImage(W)
    out = ops.gemm_gather(A, img, bias, add0=R)
    ref = A.double() @ W.double().t() + bias.double() + R.double()
    assert (out.double() - ref).abs().max().item() <= 2e-5 * ref.abs().max().item()
    assert torch.equal(out, ops.gemm_nt(A, img, bias, R))
    assert torch.equal(out, ops.gemm_gather(A, img, bias, add0=R))


@pytest.mark.parametrize("N", [32, 64, 128, 256])
def test_gather_repeats_shared_index_and_strided_views(N):
    """add0 / add1 are column slices of one wide table, the indices repeat, idx0 is idx1, and C has ldc > N."""
    M, K, Nn = 5003, 256, 37
    g, A, W, bias = _operands(M, N, K, N)
    P = torch.randn(Nn, 4 * N, generator=g).to(DEV)
    idx = torch.randint(0, Nn, (M,), generator=g).to(torch.int32).to(DEV)
    idx[:64] = 5                                                     # a whole warp's rows read the same row
    wide = torch.full((M, N + 32), float("nan"), device=DEV)
    out = wide[:, 16:16 + N]
    img = ops.WeightImage(W)
    res, part = ops.gemm_gather(A, img, bias, add0=P[:, 0:N], idx0=idx, add1=P[:, 2 * N:3 * N], idx1=idx, stats=True,
                                out=out)
    assert res.data_ptr() == out.data_ptr()
    il = idx.long()
    ref = A.double() @ W.double().t() + bias.double() + P[:, 0:N].double()[il] + P[:, 2 * N:3 * N].double()[il]
    assert (out.double() - ref).abs().max().item() <= 2e-5 * ref.abs().max().item()
    assert torch.isnan(wide[:, :16]).all() and torch.isnan(wide[:, 16 + N:]).all()   # nothing outside C's columns
    s = part.double().sum(0)
    assert (s[0] - ref.sum(0)).abs().max().item() <= 1e-5 * ref.abs().sum(0).max().item()
    assert (s[1] - (ref * ref).sum(0)).abs().max().item() <= 1e-5 * (ref * ref).sum(0).max().item()
    again = torch.empty(M, N, device=DEV)
    res2, part2 = ops.gemm_gather(A, img, bias, add0=P[:, 0:N], idx0=idx, add1=P[:, 2 * N:3 * N], idx1=idx, stats=True,
                                  out=again)
    assert torch.equal(out, again) and torch.equal(part, part2)


@pytest.mark.parametrize("M,N,K", [(1, 32, 32), (129, 64, 64), (MANY, 32, 96), (3001, 96, 256), (20000, 256, 256),
                                   (777, 128, 1024)])
def test_stats_match_fp64(M, N, K):
    g, A, W, bias = _operands(M, N, K, 3 * M + N + K)
    img = ops.WeightImage(W)
    out, part = ops.gemm_gather(A, img, bias, stats=True)
    assert part.shape[0] == _lib.load().alignn_b200_gemm_gather_stat_rows(M, N)
    ref = A.double() @ W.double().t() + bias.double()
    assert (out.double() - ref).abs().max().item() <= 2e-5 * ref.abs().max().item()
    s = part.double().sum(0)
    assert (s[0] - ref.sum(0)).abs().max().item() <= 1e-5 * ref.abs().sum(0).max().item()
    assert (s[1] - (ref * ref).sum(0)).abs().max().item() <= 1e-5 * (ref * ref).sum(0).max().item()
    out2, part2 = ops.gemm_gather(A, img, bias, stats=True)
    assert torch.equal(out, out2) and torch.equal(part, part2)
