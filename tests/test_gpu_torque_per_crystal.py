"""GPU (-m gpu): per-crystal net-torque removal (`ops.remove_net_torque_per_crystal`, csrc/ff_device.cu) against
one-crystal calls of the batch-wide kernel (`ops.remove_net_torque`) bit for bit, and against the fp64 oracle."""
import numpy as np
import pytest
import torch

from alignn_b200 import _lib, ops
from oracle import ealignn_oracle as EO

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
# 70 000 atoms > 256 x 256: that crystal's partials are capped at 256 blocks
SIZES = [1, 2, 3, 4, 255, 257, 70000, 3]


def _batch(sizes, seed=0):
    rng = np.random.default_rng(seed)
    pos = [rng.uniform(-10.0, 10.0, (n, 3)) + rng.uniform(-50.0, 50.0, 3) for n in sizes]
    forces = [rng.normal(size=(n, 3)) for n in sizes]
    pos = torch.from_numpy(np.concatenate(pos)).float()
    forces = torch.from_numpy(np.concatenate(forces)).float()
    off = torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int64)
    return pos, forces, off


def _lone(pos, forces, off):
    """The batch-wide kernel on every crystal as a one-crystal batch."""
    out = []
    for b in range(off.numel() - 1):
        sl = slice(int(off[b]), int(off[b + 1]))
        one = torch.tensor([0, sl.stop - sl.start], dtype=torch.int64, device=DEV)
        out.append(ops.remove_net_torque(pos[sl].contiguous(), forces[sl].contiguous(), one))
    return torch.cat(out)


def test_per_crystal_equals_lone_calls_bitwise_and_is_repeatable():
    pos, forces, off = _batch(SIZES)
    pos, forces, off = pos.to(DEV), forces.to(DEV), off.to(DEV)
    got = ops.remove_net_torque_per_crystal(pos, forces, off)
    want = _lone(pos, forces, off)
    assert torch.equal(got, want)
    assert torch.equal(ops.remove_net_torque_per_crystal(pos, forces, off), got)
    assert not torch.equal(got, ops.remove_net_torque(pos, forces, off))      # the batch-wide quirks differ


def _row_wise(p, f):
    """remove_net_torque of one crystal with the row-wise cross product throughout (no dim-0 quirk), fp64."""
    r = p - p.mean(0)
    M = r.T @ r - (r * r).sum() * torch.eye(3, dtype=torch.float64)
    mu = torch.linalg.solve(M, -torch.cross(r, f, dim=1).sum(0))
    return f + torch.cross(r, mu.expand_as(r), dim=1)


def test_three_atom_crystal_takes_the_column_wise_cross():
    sizes = [3, 4, 3]
    pos, forces, off = _batch(sizes)
    got = ops.remove_net_torque_per_crystal(pos.to(DEV), forces.to(DEV), off.to(DEV)).cpu().double()
    for b, n in enumerate(sizes):
        sl = slice(int(off[b]), int(off[b + 1]))
        p, f = pos[sl].double(), forces[sl].double()
        want = EO.remove_net_torque(p, f, [n])                 # torch.cross without dim: dim 0 exactly for n == 3
        assert (got[sl] - want).abs().max() <= 1e-5 * max(want.abs().max().item(), 1.0), b
        rw = _row_wise(p, f)
        if n == 3:
            assert (got[sl] - rw).abs().max() > 1e-3, b
        else:
            assert (got[sl] - rw).abs().max() <= 1e-5 * max(rw.abs().max().item(), 1.0), b


def test_collinear_crystal_takes_the_pseudo_inverse():
    rng = np.random.default_rng(4)
    # atoms on a line along x: M = c (e_x e_x^T - I) has an exactly zero first column, so LU meets a zero pivot
    line = np.outer(np.linspace(-2.0, 3.0, 5), [1.0, 0.0, 0.0]) + np.array([0.5, -1.25, 2.0])
    pos = torch.from_numpy(np.concatenate([line, rng.normal(size=(6, 3))])).float()
    forces = torch.from_numpy(rng.normal(size=(11, 3))).float()
    off = torch.tensor([0, 5, 11], dtype=torch.int64)
    got = ops.remove_net_torque_per_crystal(pos.to(DEV), forces.to(DEV), off.to(DEV))
    assert torch.equal(got, _lone(pos.to(DEV), forces.to(DEV), off.to(DEV)))
    assert torch.isfinite(got).all()
    want = EO.remove_net_torque(pos[:5].double(), forces[:5].double(), [5])   # the oracle's pinv branch
    assert (got[:5].cpu().double() - want).abs().max() <= 1e-5 * want.abs().max().item()


def test_matches_the_fp64_oracle_per_crystal():
    # not 2 atoms: two points are collinear, and the rounding of M's tiny pivot decides the answer, in both
    sizes = [1, 3, 4, 255, 257, 1000]
    pos, forces, off = _batch(sizes, seed=2)
    got = ops.remove_net_torque_per_crystal(pos.to(DEV), forces.to(DEV), off.to(DEV)).cpu()
    want = torch.cat([EO.remove_net_torque(pos[int(off[b]):int(off[b + 1])].double(),
                                           forces[int(off[b]):int(off[b + 1])].double(), [n])
                      for b, n in enumerate(sizes)])
    # fp32 in and out: the kernel works in fp64 and rounds once at the end
    err = (got.double() - want).abs() - 2 ** -23 * want.abs()
    assert err.max().item() <= 1e-12, err.max().item()


def test_bad_arguments():
    lib = _lib.load()
    pos, forces, off = _batch([2, 3])
    pos, forces, off = pos.to(DEV), forces.to(DEV), off.to(DEV)
    out = torch.empty_like(forces)
    nb = int(lib.alignn_b200_remove_net_torque_per_crystal_workspace_bytes(2, 5))
    ws = torch.empty(nb, dtype=torch.uint8, device=DEV)
    st = _lib.stream_ptr()
    call = lambda p=pos.data_ptr(), f=forces.data_ptr(), o=off.data_ptr(), B=2, N=5, y=out.data_ptr(), w=ws.data_ptr(), n=nb: \
        lib.alignn_b200_remove_net_torque_per_crystal(p, f, o, B, N, y, w, n, st)   # noqa: E731
    assert call() == 0
    for kw in (dict(B=0), dict(B=-1), dict(N=-1), dict(p=None), dict(f=None), dict(o=None), dict(y=None), dict(w=None),
               dict(B=2 ** 31, N=5)):
        assert call(**kw) == -1, kw
    assert call(n=nb - 1) == -5
    assert lib.alignn_b200_remove_net_torque_per_crystal_workspace_bytes(0, 5) == 0
    assert lib.alignn_b200_remove_net_torque_per_crystal_workspace_bytes(2, -1) == 0
    assert lib.alignn_b200_remove_net_torque_per_crystal_workspace_bytes(1, 2 ** 40) == 0
    # offsets are device data: the kernel checks them and answers with NaN rows instead of reading out of range
    for bad in ([1, 2, 5], [0, 3, 2, 5], [0, 4, 3], [0, 2, 6], [0, 2, 4]):
        o = torch.tensor(bad, dtype=torch.int64, device=DEV)
        assert torch.isnan(ops.remove_net_torque_per_crystal(pos, forces, o)).all(), bad
    # an empty batch of crystals with no atoms is fine
    e = torch.zeros(0, 3, device=DEV)
    assert ops.remove_net_torque_per_crystal(e, e, torch.zeros(3, dtype=torch.int64, device=DEV)).shape == (0, 3)
    with pytest.raises(ValueError):
        ops.remove_net_torque_per_crystal(pos, forces, off.int())
