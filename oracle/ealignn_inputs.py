"""Seeded inputs of the eALIGNN fixtures (tests/golden/ealignn_small.npz), shared by oracle/make_golden_ealignn.py and
the tests.  Test infrastructure.

Small random periodic crystals, bonds from the periodic radius graph at 5 A (alignn/graphs.py:267-364, native host scan
`alignn_b200.neighbors.radius_graph`), so that the model's 4 A `inner_cutoff` removes bonds.  ndata: frac_coords, V,
atom_features; edata: r, images (integer cell offsets, as the reference stores them).  A crystal is redrawn until every
recomputed bond length (cart[dst] + images - cart[src], the reference's own formula) is at least 1e-4 A away from the
cutoff: at the boundary an fp32 length may round either way.
"""
from __future__ import annotations

import numpy as np
import torch

INNER_CUTOFF = 4.0
ATOM_FEATURES = 8
MARGIN = 1e-4


def _crystal(rng, n_atoms):
    lat = np.diag(rng.uniform(4.2, 5.2, 3)) + rng.uniform(-0.3, 0.3, (3, 3)) * (1 - np.eye(3))
    frac = rng.uniform(0.0, 1.0, (n_atoms, 3))
    return lat, frac


def _margin_ok(lat, frac, u, v, images):
    cart = torch.from_numpy(frac).float() @ torch.from_numpy(lat).float()
    r = (cart[torch.from_numpy(v)] + torch.from_numpy(images)) - cart[torch.from_numpy(u)]
    return bool((torch.norm(r.double(), dim=1) - INNER_CUTOFF).abs().min() >= MARGIN)


def crystals(seed: int = 7, sizes=(4, 5, 6)):
    """[(lattice [3,3] float64, frac [n,3] float64, u, v, r float32 [E,3], images float64 [E,3])] per crystal."""
    from alignn_b200 import neighbors
    rng = np.random.default_rng(seed)
    out = []
    for n in sizes:
        while True:
            lat, frac = _crystal(rng, n)
            u, v, r, images = neighbors.radius_graph(lat, frac @ lat, cutoff=5.0)
            if _margin_ok(lat, frac, u, v, images):
                break
        out.append((lat, frac, u, v, r, images))
    return out


def batch_arrays(seed: int = 7, sizes=(4, 5, 6)):
    """The batch as plain tensors: src, dst (int64), bnn, bne, lattices [B,3,3], frac, V, atom_features, r, images."""
    cs = crystals(seed, sizes)
    noff, src, dst = 0, [], []
    for lat, frac, u, v, _, _ in cs:
        src.append(torch.from_numpy(u) + noff)
        dst.append(torch.from_numpy(v) + noff)
        noff += frac.shape[0]
    feats = np.random.default_rng(seed + 1000).normal(size=(noff, ATOM_FEATURES))
    return dict(src=torch.cat(src), dst=torch.cat(dst),
                bnn=torch.tensor([c[1].shape[0] for c in cs]), bne=torch.tensor([len(c[2]) for c in cs]),
                lattice=torch.from_numpy(np.stack([c[0] for c in cs])),
                frac=torch.from_numpy(np.concatenate([c[1] for c in cs])),
                V=torch.cat([torch.full((c[1].shape[0],), abs(np.linalg.det(c[0]))) for c in cs]),
                atom_features=torch.from_numpy(feats).float(),
                r=torch.from_numpy(np.concatenate([c[4] for c in cs])),
                images=torch.from_numpy(np.concatenate([c[5] for c in cs])))


MODEL_CFG = dict(alignn_layers=2, gcn_layers=2, hidden_features=64, embedding_features=32,
                 atom_input_features=ATOM_FEATURES, stresswise_weight=0.1, stress_multiplier=10.0)
MODEL_SEED = 600


def torque_cases():
    """Inputs of the direct remove_net_torque fixtures (fp64): name -> (positions [N,3], forces [N,3], n_nodes [B])."""
    rng = np.random.default_rng(77)
    t = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float64))  # noqa: E731
    return {
        "one_crystal": (t(rng.normal(size=(7, 3)) * 2), t(rng.normal(size=(7, 3))), torch.tensor([7])),
        "batch": (t(rng.normal(size=(9, 3)) * 2), t(rng.normal(size=(9, 3))), torch.tensor([4, 3, 2])),
        "three_atoms": (t(rng.normal(size=(3, 3)) * 2), t(rng.normal(size=(3, 3))), torch.tensor([3])),
    }
