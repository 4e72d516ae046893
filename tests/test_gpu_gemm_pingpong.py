"""GPU (-m gpu): the ping-pong schedule of the Linear-layer GEMM (csrc/gemm_tc.cu) against fp64.

A persistent CTA's local tile i belongs to consumer warpgroup i % 2, the producer warpgroup streams the chunks of all
its tiles through one stage ring, and the two warpgroups take turns adding their rows' column statistics into shared
partial rows.  These cases cover what only that schedule can get wrong: CTAs whose two warpgroups own unequal tile
counts (one tile, two tiles, one tile more than the grid, an odd number of tiles per CTA), ring phases carried across
tiles and warpgroups at one chunk per tile (K = 32) and at 32 chunks per tile (K = 1024), ragged M, every column tile
width with statistics on and off, and gathered addends with repeated indices.  Every case is run twice and must repeat
bit for bit.  Tolerances as in test_gpu_gemm_epilogue.py."""
import pytest
import torch

from alignn_b200 import _lib, ops

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SMS = 132


def _check(M, N, K, seed, stats, gather):
    g = torch.Generator(device="cpu").manual_seed(seed)
    A = torch.randn(M, K, generator=g).to(DEV)
    W = (torch.randn(N, K, generator=g) / K ** 0.5).to(DEV)
    bias = torch.randn(N, generator=g).to(DEV)
    img = ops.WeightImage(W)
    ref = A.double() @ W.double().t() + bias.double()
    kw = {}
    if gather:
        rows = 29
        P = torch.randn(rows, 3 * N, generator=g).to(DEV)
        idx0 = torch.randint(0, rows, (M,), generator=g).to(torch.int32).to(DEV)
        idx1 = torch.randint(0, rows, (M,), generator=g).to(torch.int32).to(DEV)
        idx0[: min(M, 200)] = 3                              # whole tiles' worth of rows read one addend row
        kw = dict(add0=P[:, 0:N], idx0=idx0, add1=P[:, 2 * N:3 * N], idx1=idx1)
        ref = ref + P[:, 0:N].double()[idx0.long()] + P[:, 2 * N:3 * N].double()[idx1.long()]
    else:
        R = torch.randn(M, N, generator=g).to(DEV)
        kw = dict(add0=R)
        ref = ref + R.double()
    runs = [ops.gemm_gather(A, img, bias, stats=stats, **kw) for _ in range(2)]
    out = runs[0][0] if stats else runs[0]
    assert (out.double() - ref).abs().max().item() <= 2e-5 * ref.abs().max().item()
    if stats:
        part = runs[0][1]
        assert part.shape[0] == _lib.load().alignn_b200_gemm_gather_stat_rows(M, N)
        s = part.double().sum(0)
        assert (s[0] - ref.sum(0)).abs().max().item() <= 1e-5 * ref.abs().sum(0).max().item()
        assert (s[1] - (ref * ref).sum(0)).abs().max().item() <= 1e-5 * (ref * ref).sum(0).max().item()
        assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    else:
        assert torch.equal(runs[0], runs[1])


# tiles of a 128 x BN grid: 1, 2, SMS - 1, SMS + 1, and 3 per CTA (warpgroup 0 gets two, warpgroup 1 one)
TILE_COUNTS = [1, 2, SMS - 1, SMS + 1, 3 * SMS]


@pytest.mark.parametrize("tiles", TILE_COUNTS)
@pytest.mark.parametrize("N", [32, 64, 128])
@pytest.mark.parametrize("stats", [False, True])
def test_unequal_tile_counts_per_warpgroup(tiles, N, stats):
    _check(tiles * 128, N, 256, tiles * 7 + N, stats, gather=False)


@pytest.mark.parametrize("K", [32, 1024])
@pytest.mark.parametrize("M", [128, 2 * SMS * 128 + 77, 3 * SMS * 128 - 5])
@pytest.mark.parametrize("N", [64, 256])
def test_ring_phases_across_tiles(K, M, N):
    _check(M, N, K, M + K + N, stats=True, gather=False)


@pytest.mark.parametrize("M", [1, 65, 127, 129, 255, SMS * 128 + 1, 5 * SMS * 128 - 63])
@pytest.mark.parametrize("N", [32, 128, 256])
def test_ragged_rows_with_gathered_addends(M, N):
    _check(M, N, 256, 3 * M + N, stats=True, gather=True)
