"""CPU oracle of eALIGNN (alignn/models/ealignn_atomwise.py): the structure rebuilt inside forward, the net-torque
removal and the energy / forces / stress, on the LayerNorm stack of oracle/alignn_oracle.py.

THIS IS TEST INFRASTRUCTURE, like alignn_oracle.py: only tests/ and oracle/make_golden_ealignn.py import it.  Every
function cites the reference file:line it follows; works in fp32 and fp64, pure torch on CPU.
"""
from __future__ import annotations

import numpy as np
import torch

from .alignn_oracle import ALIGNN, OGraph, avg_pool, bond_cosines, line_graph

def cartesian_coords(frac, lattice, bnn):
    """compute_cartesian_coordinates, alignn/models/utils.py:88-126: always fp32 (its dtype default)."""
    lat = lattice.to(torch.float32)
    if lat.dim() == 2:
        lat = lat.unsqueeze(0)
    gid = torch.repeat_interleave(torch.arange(len(lat)), torch.as_tensor(bnn))
    return torch.bmm(frac.to(torch.float32).unsqueeze(1), lat[gid]).squeeze(1)


def pair_vectors(cart, src, dst, images):
    """compute_pair_vector_and_distance, alignn/models/utils.py:47-55 (images are added as they are)."""
    return (cart[dst] + images) - cart[src]


def lightweight_filter(g: OGraph, r, inner_cutoff):
    """lightweight_line_graph(g, "bondlength", gt inner_cutoff), alignn/models/utils.py:129-222: keep the bonds with
    NOT |r| > inner_cutoff in order; edata filtered, ndata shared, edge_ids crystal-local when batch_size > 1."""
    keep = torch.logical_not(torch.gt(torch.norm(r, dim=1), inner_cutoff))
    eoff = np.concatenate([[0], np.cumsum(g.bne.numpy())])
    kept, eids = [], []
    for b in range(len(g.bne)):
        k = keep[eoff[b]:eoff[b + 1]]
        kept.append(int(k.sum()))
        eids.append(k.nonzero().reshape(-1) + (0 if len(g.bne) > 1 else int(eoff[b])))
    out = OGraph(g.src[keep], g.dst[keep], g.n, g.bnn.clone(), torch.tensor(kept))
    out.ndata = dict(g.ndata)
    out.edata = {k: v[keep] for k, v in g.edata.items()}
    out.edata["edge_ids"] = torch.cat(eids)
    return out


def remove_net_torque(positions, forces, bnn):
    """remove_net_torque, alignn/models/utils.py:295-398 with its quirks: batch-wide centre and torque, one solve per
    crystal with the same torque, the pseudo-inverse for the WHOLE batch when any system is singular, and torch.cross
    without `dim` (dim 0 for a batch of 3 atoms).  The reference's pseudo-inverse branch raises an IndexError
    (`b.unsqueeze(2)` on the 1-D torque); here it applies the pseudo-inverse to the torque of every crystal as meant.  Positions are cast to the forces' dtype (the reference itself
    fails in fp64 because its coordinates are fp32)."""
    n_nodes = torch.as_tensor(bnn)
    positions = positions.to(forces.dtype)
    cross = lambda a, b: torch.cross(a, b, dim=0 if a.shape[0] == 3 else 1)  # noqa: E731
    com = torch.sum(positions, dim=0) / n_nodes.float().sum()
    r = positions - com.repeat(positions.size(0), 1)
    tau = torch.sum(cross(r, forces), dim=0)
    r2 = torch.sum(r ** 2, dim=1)
    B = n_nodes.numel()
    s = torch.zeros(B, dtype=forces.dtype)
    S = torch.zeros(B, 3, 3, dtype=forces.dtype)
    outer = r.unsqueeze(2) @ r.unsqueeze(1)
    a = 0
    for i, n in enumerate(n_nodes.tolist()):
        s[i] = torch.sum(r2[a:a + n])
        S[i] = torch.sum(outer[a:a + n], dim=0)
        a += n
    M = S - s.view(-1, 1, 1) * torch.eye(3, dtype=forces.dtype).unsqueeze(0).expand(B, -1, -1)
    b = -tau
    try:
        mu = torch.linalg.solve(M, b)
    except RuntimeError:
        mu = torch.bmm(torch.linalg.pinv(M), b.expand(B, 3).unsqueeze(2)).squeeze(2)
    return forces + cross(r, torch.repeat_interleave(mu, n_nodes, dim=0))


def ealignn_forward(model: ALIGNN, g: OGraph, lattice, alignn_layers: int, inner_cutoff=4.0, remove_torque=True,
                    energy_mult_natoms=True, use_penalty=True, penalty_factor=0.1, penalty_threshold=1.0,
                    stresswise_weight=0.0, stress_multiplier=1.0, classification=False, create_graph=False):
    """eALIGNNAtomWise.forward, alignn/models/ealignn_atomwise.py:277-444, on the LayerNorm oracle stack (`model` built
    with norm="layernorm", output_features=1; same parameter names).  With ALIGNN layers: fp32 Cartesian coordinates,
    bond vectors with the images added as they are, bonds longer than inner_cutoff dropped, L(g) of the rest; pair forces
    = -dE/dr' * (atoms in the batch); forces = in-edge minus out-edge sums; net torque removed; virial from r'.
    Returns a dict: out, forces, pair_forces, stress, kept (per crystal), T (L(g) edges)."""
    x = model.atom_embedding(g.ndata["atom_features"])
    lg = z = None
    if alignn_layers > 0:
        cart = cartesian_coords(g.ndata["frac_coords"], lattice, g.bnn)
        g = lightweight_filter(g, pair_vectors(cart, g.src, g.dst, g.edata["images"]), inner_cutoff)
        r = pair_vectors(cart, g.src, g.dst, g.edata["images"]).detach().requires_grad_(True)
        lg = line_graph(g)
        z = model.angle_embedding(bond_cosines(r, lg.src, lg.dst))
        pos = cart
    else:
        r = g.edata["r"].detach().clone().requires_grad_(True)
        pos = g.ndata.get("cart_coords")
    bondlength = torch.norm(r, dim=1)
    y = model.edge_embedding(bondlength)
    x, y = model.conv_stack(g, lg, x, y, z)
    out = torch.squeeze(model.fc(avg_pool(g, x)))
    en = out * g.bnn.to(out.dtype) if energy_mult_natoms else out
    if use_penalty:
        pen = torch.where(bondlength < penalty_threshold, penalty_factor * (penalty_threshold - bondlength),
                          torch.zeros_like(bondlength))
        en = en + pen.sum()
        if not energy_mult_natoms:
            out = en
    (dr,) = torch.autograd.grad(en, r, grad_outputs=torch.ones_like(en), create_graph=create_graph)
    pair = -dr * g.n
    zeros = torch.zeros(g.n, 3, dtype=pair.dtype)
    forces = zeros.index_add(0, g.dst, pair) - zeros.index_add(0, g.src, pair)
    if remove_torque:
        forces = remove_net_torque(pos, forces, g.bnn)
    stress = None
    if stresswise_weight != 0:
        st, ce, cn = [], 0, 0
        for b in range(len(g.bne)):
            ne = int(g.bne[b])
            st.append(-1 * (160.21766208 * torch.matmul(r[ce:ce + ne].T, pair[ce:ce + ne]) / g.ndata["V"][cn]))
            ce += ne
            cn += int(g.bnn[b])
        stress = stress_multiplier * torch.stack(st)
    if classification:
        out = torch.sigmoid(out)
    res = dict(out=out, forces=forces, pair_forces=pair, stress=stress, kept=g.bne.clone(),
               T=0 if lg is None else lg.num_edges())
    if not create_graph:
        res = {k: (v.detach() if isinstance(v, torch.Tensor) else v) for k, v in res.items()}
    return res
