"""eALIGNN force field (mirror of alignn/models/ealignn_atomwise.py) on the CUDA conv stack.

Unlike ALIGNNAtomWise, the model rebuilds its graphs inside every forward (`compute_line_graph: false` in
examples/sample_data_ff/econfig_example_atomwise.json): Cartesian coordinates from `frac_coords` and the lattice, bond
vectors from those, the atom graph without the bonds longer than `inner_cutoff`, and L(g) of that graph -- all on the
device (csrc/ff_device.cu, csrc/graph_device.cu) -- and it removes the net torque from the forces afterwards.
"""
from __future__ import annotations

from typing import Literal

import torch
from pydantic_settings import BaseSettings, SettingsConfigDict
from torch import nn

from . import ops
from .alignn import RBFExpansion
from .alignn_atomwise import ALIGNNConv, EdgeGatedGraphConv, MLPLayer, virial_stress
from .conv import second_order
from .graph import Graph, as_graph, bond_cosines, lightweight_graph


class eALIGNNAtomWiseConfig(BaseSettings):
    """Field for field the reference schema (alignn/models/ealignn_atomwise.py:31-72).

    Fields the model reads like the reference does, and the ones it ignores like the reference does: `link`,
    `use_cutoff_function`, `multiply_cutoff`, `add_reverse_forces`, `batch_stress`, `lg_on_fly`, `grad_multiplier`,
    `force_mult_natoms`, `include_pos_deriv`, `zero_inflated` and `exponent` have no effect."""

    model_config = SettingsConfigDict(env_prefix="jv_model", extra="forbid")

    name: Literal["ealignn_atomwise"]
    alignn_layers: int = 2
    gcn_layers: int = 2
    atom_input_features: int = 1
    edge_input_features: int = 80
    triplet_input_features: int = 40
    embedding_features: int = 64
    hidden_features: int = 64
    output_features: int = 1
    calculate_gradient: bool = True
    atomwise_output_features: int = 0
    graphwise_weight: float = 1.0
    gradwise_weight: float = 1.0
    stresswise_weight: float = 0.0
    atomwise_weight: float = 0.0
    classification: bool = False
    energy_mult_natoms: bool = True
    remove_torque: bool = True
    inner_cutoff: float = 4
    use_penalty: bool = True
    extra_features: int = 0
    penalty_factor: float = 0.1
    penalty_threshold: float = 1
    additional_output_features: int = 0
    additional_output_weight: float = 0
    stress_multiplier: float = 1
    grad_multiplier: int = -1
    link: Literal["identity", "log", "logit"] = "identity"
    zero_inflated: bool = False
    force_mult_natoms: bool = False
    include_pos_deriv: bool = False
    use_cutoff_function: bool = False
    add_reverse_forces: bool = True
    lg_on_fly: bool = True
    batch_stress: bool = True
    multiply_cutoff: bool = False
    exponent: int = 5


def cartesian_coordinates(g: Graph, lat: torch.Tensor) -> torch.Tensor:
    """frac_coords @ lattice of each atom's crystal, in fp32 whatever the input precision (compute_cartesian_coordinates,
    alignn/models/utils.py:88-126, dtype=torch.float32 by default)."""
    frac = g.ndata["frac_coords"].to(torch.float32)
    lat = lat.to(device=frac.device, dtype=torch.float32)
    if lat.dim() == 2:
        lat = lat.unsqueeze(0)
    gid = torch.repeat_interleave(torch.arange(lat.shape[0], device=frac.device), g.batch_num_nodes_on_device(),
                                  output_size=frac.shape[0])
    return (frac.unsqueeze(2) * lat[gid]).sum(1)


def remove_net_torque_torch(pos: torch.Tensor, forces: torch.Tensor, batch_num_nodes: torch.Tensor) -> torch.Tensor:
    """`ops.remove_net_torque` from differentiable torch operators (force training differentiates through it).
    Same quirks: batch-wide centre and torque, per-crystal solve, pseudo-inverse for an exactly singular system, and
    dim 0 for the cross products of a 3-atom batch."""
    N, dev, dt = forces.shape[0], forces.device, forces.dtype
    dim = 0 if N == 3 else 1                  # torch.cross without `dim` takes the first dimension of size 3
    pos = pos.to(dt)
    r = pos - pos.sum(0) / N
    tau = torch.cross(r, forces, dim=dim).sum(0)
    bnn = batch_num_nodes.to(dev)
    B = bnn.numel()
    gid = torch.repeat_interleave(torch.arange(B, device=dev), bnn, output_size=N)
    s = torch.zeros(B, device=dev, dtype=dt).index_add(0, gid, (r * r).sum(1))
    S = torch.zeros(B, 9, device=dev, dtype=dt).index_add(0, gid, (r.unsqueeze(2) * r.unsqueeze(1)).reshape(N, 9)).view(B, 3, 3)
    eye = torch.eye(3, device=dev, dtype=dt)
    M = S - s.view(B, 1, 1) * eye
    b = (-tau).expand(B, 3)
    singular = (torch.linalg.solve_ex(M.detach(), b.detach())[1] != 0).view(B, 1)
    mu = torch.where(singular, (torch.linalg.pinv(M) @ b.unsqueeze(2)).squeeze(2),
                     torch.linalg.solve(torch.where(singular.view(B, 1, 1), eye, M), b))
    return forces + torch.cross(r, mu[gid], dim=dim)


class eALIGNNAtomWise(nn.Module):
    """Energy, forces and stress of eALIGNN (alignn/models/ealignn_atomwise.py:174-444) through the CUDA conv stack.

    `forward((g, lat))` or `forward((g, lg, lat))`; with ALIGNN layers a passed lg is ignored, because the reference
    rebuilds it.  With `alignn_layers > 0` the graph needs ndata `frac_coords` and edata `images`; the bonds that
    drive the model are the recomputed ones no longer than `inner_cutoff`.  Inference / MD run the filter, L(g), convs,
    pair-force scatter, torque removal and virial on the library's kernels; force / stress training (as in
    ALIGNNAtomWise) keeps the convs on the kernels and makes the embeddings, pooling, scatter, torque removal and virial
    differentiable torch operators.  Same state_dict names as the reference.
    """

    def __init__(self, config: eALIGNNAtomWiseConfig = eALIGNNAtomWiseConfig(name="ealignn_atomwise")):
        super().__init__()
        c = self.config = config
        if c.gradwise_weight == 0:                   # ealignn_atomwise.py:192-193
            c.calculate_gradient = False
        if c.extra_features != 0:
            raise NotImplementedError("alignn_b200.eALIGNNAtomWise: extra_features is outside the built hot path")
        self.classification = c.classification
        self.atom_embedding = MLPLayer(c.atom_input_features, c.hidden_features)
        self.edge_embedding = nn.Sequential(RBFExpansion(vmin=0, vmax=8.0, bins=c.edge_input_features),
                                            MLPLayer(c.edge_input_features, c.embedding_features),
                                            MLPLayer(c.embedding_features, c.hidden_features))
        self.angle_embedding = nn.Sequential(RBFExpansion(vmin=-1, vmax=1.0, bins=c.triplet_input_features),
                                             MLPLayer(c.triplet_input_features, c.embedding_features),
                                             MLPLayer(c.embedding_features, c.hidden_features))
        self.alignn_layers = nn.ModuleList([ALIGNNConv(c.hidden_features, c.hidden_features) for _ in range(c.alignn_layers)])
        self.gcn_layers = nn.ModuleList([EdgeGatedGraphConv(c.hidden_features, c.hidden_features) for _ in range(c.gcn_layers)])
        if c.atomwise_output_features > 0:
            self.fc_atomwise = nn.Linear(c.hidden_features, c.atomwise_output_features)
        if c.additional_output_features:
            self.fc_additional_output = nn.Linear(c.hidden_features, c.additional_output_features)
        if self.classification:
            self.fc = nn.Linear(c.hidden_features, 1)
            self.softmax = nn.Sigmoid()
        else:
            self.fc = nn.Linear(c.hidden_features, c.output_features)

    def forward(self, g):
        c = self.config
        second = bool(self.training and torch.is_grad_enabled() and c.calculate_gradient
                      and (c.gradwise_weight != 0 or c.stresswise_weight != 0))
        if second:
            with second_order():
                return self._forward(g, True)
        return self._forward(g, False)

    def _forward(self, inputs, second: bool):
        c = self.config
        g, lat = as_graph(inputs[0]), inputs[-1]
        x = self.atom_embedding(g.ndata["atom_features"])
        lg = z = None
        if len(self.alignn_layers) > 0:
            # :306-322 -- the structure is rebuilt from the coordinates: cutoff-filtered g, then its L(g)
            pos = cartesian_coordinates(g, lat)
            g, r = lightweight_graph(g, pos, c.inner_cutoff)
            lg = g.line_graph(shared=True)
        else:
            # :302-305 -- no filter: the stored bond vectors; torque removal reads the stored coordinates
            r = g.edata["r"].detach()
            pos = g.ndata["cart_coords"] if c.calculate_gradient and c.remove_torque else None
        if c.calculate_gradient:
            r = r.requires_grad_(True)        # a fresh leaf: grad(en_out, r) is the reference's grad w.r.t. the filtered r
        bondlength = torch.norm(r, dim=1)
        if lg is not None:
            z = self.angle_embedding(bond_cosines(r, lg))
        y = self.edge_embedding(bondlength)
        n_al, n_gcn = len(self.alignn_layers), len(self.gcn_layers)
        for i, layer in enumerate(self.alignn_layers):
            x, y, z = layer(g, lg, x, y, z, _need_z_out=(i + 1 < n_al))
        for i, layer in enumerate(self.gcn_layers):
            x, y = layer(g, x, y, _need_edge_out=(i + 1 < n_gcn))
        hpool = ops.segment_mean_any_order(x, g.node_graph_offsets(), second)
        out = torch.squeeze(self.fc(hpool))
        additional = torch.empty(1)
        if c.additional_output_features > 0:
            additional = self.fc_additional_output(hpool)
        atomwise_pred = torch.empty(1)
        if c.atomwise_output_features > 0 and c.atomwise_weight != 0:
            atomwise_pred = self.fc_atomwise(x)
        forces = torch.empty(1)
        stress = torch.empty(1)
        natoms = g.batch_num_nodes_on_device().to(out.dtype)
        en_out = out * natoms if c.energy_mult_natoms else out          # :364-366
        if c.use_penalty:                                               # :367-379
            pen = torch.where(bondlength < c.penalty_threshold, c.penalty_factor * (c.penalty_threshold - bondlength),
                              torch.zeros_like(bondlength))
            en_out = en_out + pen.sum()
            if not c.energy_mult_natoms:
                out = en_out                  # the in-place `en_out += total_penalty` also changes `out` (SURVEY App. D-12)
        result = {}
        if c.calculate_gradient:
            with ops.input_grads_only():
                (dr,) = torch.autograd.grad(en_out, r, grad_outputs=torch.ones_like(en_out),
                                            create_graph=second, retain_graph=second or self.training)
            pair_forces = -dr * g.num_nodes()                           # :384-394: the batch's total atom count
            if second:
                src, dst = g.index.src.long(), g.index.dst.long()
                zeros = torch.zeros(g.num_nodes(), 3, device=r.device, dtype=r.dtype)
                forces = zeros.index_add(0, dst, pair_forces) - zeros.index_add(0, src, pair_forces)   # :396-408
            else:
                forces = ops.pair_force_scatter(pair_forces, g.index, True)
            if c.remove_torque:                                         # :409-412
                if second:
                    forces = remove_net_torque_torch(pos.detach(), forces, g.batch_num_nodes())
                else:
                    forces = ops.remove_net_torque(pos.detach(), forces, g.node_graph_offsets().long())
            forces = torch.squeeze(forces)
            result["pair_forces"] = pair_forces
            if c.stresswise_weight != 0:                                # :415-435
                if second:
                    stress = virial_stress(r, pair_forces, g.node_graph_offsets(), g.batch_num_edges(), g.ndata["V"],
                                           c.stress_multiplier)
                else:
                    stress = ops.virial_stress(r.detach(), pair_forces, g.edge_graph_offsets64(),
                                               g.node_graph_offsets().long(), g.ndata["V"], c.stress_multiplier)
        if self.classification:
            out = self.softmax(out)
        result.update(out=out, additional=additional, grad=forces, stresses=stress, atomwise_pred=atomwise_pred)
        return result
