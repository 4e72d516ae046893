"""LayerNorm twins of the conv layers (mirror of alignn/models/alignn_atomwise.py:127-246).

`train.py` trains ALIGNNAtomWise, whose EdgeGatedGraphConv / ALIGNNConv / MLPLayer use
`nn.LayerNorm` where alignn.py uses `nn.BatchNorm1d`; parameter names are the same.
"""
from __future__ import annotations

from torch import nn

from .conv import ALIGNNConvBase, EdgeGatedGraphConvBase, second_order


class MLPLayer(nn.Module):
    """Linear -> LayerNorm -> SiLU (alignn/models/utils.py:277-292)."""

    def __init__(self, in_features: int, out_features: int):
        super().__init__()
        self.layer = nn.Sequential(nn.Linear(in_features, out_features), nn.LayerNorm(out_features), nn.SiLU())

    def forward(self, x):
        from .alignn import mlp_forward
        return mlp_forward(self.layer, x)


class EdgeGatedGraphConv(EdgeGatedGraphConvBase):
    """LayerNorm variant (alignn/models/alignn_atomwise.py:127-208)."""

    def __init__(self, input_features: int, output_features: int, residual: bool = True):
        super().__init__(input_features, output_features, residual, norm="layernorm")


class ALIGNNConv(ALIGNNConvBase):
    """alignn/models/alignn_atomwise.py:211-246."""

    conv_cls = EdgeGatedGraphConv


# --------------------------------------------------------------------------------------------------
# ALIGNN-FF shell (energy + per-atom forces) on the same conv stack
# --------------------------------------------------------------------------------------------------
from typing import Literal  # noqa: E402

import numpy as np  # noqa: E402
import torch  # noqa: E402
from pydantic_settings import BaseSettings, SettingsConfigDict  # noqa: E402

from . import ops  # noqa: E402
from .alignn import RBFExpansion  # noqa: E402
from .graph import as_graph, bond_cosines  # noqa: E402


class ALIGNNAtomWiseConfig(BaseSettings):
    """Field-for-field the reference schema (alignn/models/alignn_atomwise.py:28-79)."""

    model_config = SettingsConfigDict(env_prefix="jv_model", extra="forbid")

    name: Literal["alignn_atomwise"]
    alignn_layers: int = 2
    gcn_layers: int = 2
    atom_input_features: int = 1
    edge_input_features: int = 80
    triplet_input_features: int = 40
    embedding_features: int = 64
    hidden_features: int = 64
    output_features: int = 1
    grad_multiplier: int = -1
    calculate_gradient: bool = True
    atomwise_output_features: int = 0
    graphwise_weight: float = 1.0
    gradwise_weight: float = 1.0
    stresswise_weight: float = 0.0
    atomwise_weight: float = 0.0
    link: Literal["identity", "log", "logit"] = "identity"
    zero_inflated: bool = False
    classification: bool = False
    force_mult_natoms: bool = False
    energy_mult_natoms: bool = True
    include_pos_deriv: bool = False
    use_cutoff_function: bool = False
    inner_cutoff: float = 3
    stress_multiplier: float = 1
    add_reverse_forces: bool = True
    lg_on_fly: bool = True
    batch_stress: bool = True
    multiply_cutoff: bool = False
    use_penalty: bool = True
    extra_features: int = 0
    exponent: int = 5
    penalty_factor: float = 0.1
    penalty_threshold: float = 1
    additional_output_features: int = 0
    additional_output_weight: float = 0


def cutoff_function_based_edges(r: torch.Tensor, inner_cutoff: float = 4, exponent: int = 3) -> torch.Tensor:
    """Polynomial envelope 1 + c1 x^p + c2 x^(p+1) + c3 x^(p+2), x = r / inner_cutoff, zero beyond the cutoff
    (alignn/models/utils.py:58-86)."""
    p = exponent
    x = r / inner_cutoff
    c1, c2, c3 = -(p + 1) * (p + 2) / 2, p * (p + 2), -p * (p + 1) / 2
    env = 1 + c1 * x ** p + c2 * x ** (p + 1) + c3 * x ** (p + 2)
    return torch.where(r <= inner_cutoff, env, torch.zeros_like(r))


def bond_penalty(bondlength: torch.Tensor, config) -> torch.Tensor:
    """Per-bond penalty penalty_factor * (penalty_threshold - bondlength) for bonds shorter than penalty_threshold, zero
    otherwise (alignn_atomwise.py:498-510; the model adds its sum to every crystal's energy)."""
    c = config
    return torch.where(bondlength < c.penalty_threshold, c.penalty_factor * (c.penalty_threshold - bondlength),
                       torch.zeros_like(bondlength))


EV_PER_A3_IN_GPA = 160.21766208          # 1 eV/A^3 in GPa (alignn_atomwise.py:569)


def virial_stress(r: torch.Tensor, pair_forces: torch.Tensor, node_offsets: torch.Tensor, batch_num_edges,
                  V: torch.Tensor, multiplier: float = 1.0) -> torch.Tensor:
    """Per-crystal virial stress [B,3,3] = multiplier * -160.21766208 * (r_b^T @ F_b) / V_b, where r_b / F_b are the
    bond vectors and pair forces of crystal b and V_b is the volume stored on its FIRST atom
    (alignn_atomwise.py:610-635: the loop reads `g.ndata["V"][count_node + 0]`).
    One [E,9] outer product and one segment sum over the batch instead of the reference's per-graph matmul loop."""
    E = r.shape[0]
    bne = torch.as_tensor(batch_num_edges, device=r.device).long()
    B = bne.numel()
    gid = torch.repeat_interleave(torch.arange(B, device=r.device), bne, output_size=E)
    outer = (r.unsqueeze(2) * pair_forces.unsqueeze(1)).reshape(E, 9)
    virial = torch.zeros(B, 9, device=r.device, dtype=r.dtype).index_add_(0, gid, outer).view(B, 3, 3)
    vol = V.to(r.dtype)[node_offsets[:-1].long()].view(B, 1, 1)
    return multiplier * (-EV_PER_A3_IN_GPA * virial / vol)


class ALIGNNAtomWise(nn.Module):
    """Energy (+ forces by autograd through the CUDA conv stack) -- the inference path of ALIGNN-FF
    (alignn/models/alignn_atomwise.py:249-660, BASELINE config 4).

    Same constructor/`forward((g, lg, lat))`/result-dict surface and state_dict names as the reference.
    Forces come from autograd through the conv stack.  In training with a force or stress loss the force pass keeps the
    graph (`create_graph=True`, :530-539) and the loss's backward runs the convs' double backward on the CUDA kernels
    (alignn_b200_egc_backward_vjp); the embedding MLPs, pooling and force / virial reductions are torch operators there.
    Stress: the batched virial of :610-638 (`batch_stress=True`, the default) from the same pair forces.
    Cutoff envelope on the bond lengths (`use_cutoff_function`, both `multiply_cutoff` settings, :434-451).
    `forward((g, lat))` builds L(g) inside forward (:379-386; on the device for a CUDA graph).
    Not built (SURVEY.md section 8f): `batch_stress=False` (:573-590), include_pos_deriv.
    """

    def __init__(self, config: ALIGNNAtomWiseConfig = ALIGNNAtomWiseConfig(name="alignn_atomwise")):
        super().__init__()
        c = self.config = config
        if c.gradwise_weight == 0:                 # alignn_atomwise.py:267-268: property-only models skip the force pass
            c.calculate_gradient = False
        for flag, why in ((c.include_pos_deriv, "include_pos_deriv"),
                          (c.stresswise_weight != 0 and not c.batch_stress, "stresswise_weight != 0 with batch_stress=False"),
                          (c.stresswise_weight != 0 and not c.calculate_gradient, "stress without calculate_gradient"),
                          (c.extra_features != 0, "extra_features")):
            if flag:
                raise NotImplementedError(f"alignn_b200.ALIGNNAtomWise: {why} is outside the built hot path")
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
        if c.link == "log":
            self.fc.bias.data = torch.tensor(np.log(0.7), dtype=torch.float)

    def forward(self, g):
        c = self.config
        # Force / stress TRAINING differentiates through the force computation (create_graph=True, :530-539): the MLP
        # embeddings and the pooling then run as differentiable torch operators (conv.second_order) while the LayerNorm
        # convs keep the CUDA kernels, whose backward is differentiable once more; inference, MD and property-only
        # training use the first-order kernels throughout.
        second = bool(self.training and torch.is_grad_enabled() and c.calculate_gradient
                      and (c.gradwise_weight != 0 or c.stresswise_weight != 0))
        if second:
            with second_order():
                return self._forward(g, True)
        return self._forward(g, False)

    def _forward(self, g, second: bool):
        c = self.config
        if len(self.alignn_layers) > 0:
            if len(g) == 3:
                g, lg, lat = g
                lg = as_graph(lg)
            else:
                # (g, lat): L(g) built here (:379-386), on the device for a CUDA graph; its cosines come from r below
                if not c.lg_on_fly:
                    raise ValueError("ALIGNNAtomWise((g, lat)) builds L(g) inside forward and needs lg_on_fly=True for "
                                     "its bond angles; pass (g, lg, lat) otherwise")
                g, lat = g
                g = as_graph(g)
                lg = g.line_graph(shared=True)
        else:
            g, lat = g[0], g[-1]
            lg = None
        g = as_graph(g)
        result = {}
        x = self.atom_embedding(g.ndata["atom_features"])
        r = g.edata["r"]
        if c.calculate_gradient:
            r = r.detach().requires_grad_(True)                    # alignn_atomwise.py:416-420 (without mutating g)
        bondlength = torch.norm(r, dim=1)
        z = None
        if lg is not None:
            # lg_on_fly (:424-431): cosines recomputed from r so that the three-body terms are in the autograd graph
            h = bond_cosines(r, lg) if (c.lg_on_fly or c.calculate_gradient) else lg.edata["h"]
            z = self.angle_embedding(h)
        if c.use_cutoff_function:                                   # (:434-451)
            env = cutoff_function_based_edges(bondlength, inner_cutoff=c.inner_cutoff, exponent=c.exponent)
            if c.multiply_cutoff:
                y = self.edge_embedding(bondlength) * env.unsqueeze(1)
            else:
                bondlength = env        # the reference rebinds `bondlength`: the penalty below then sees the envelope
                y = self.edge_embedding(bondlength)
        else:
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
        en_out = out * natoms if c.energy_mult_natoms else out          # (:495-497)
        if c.use_penalty:                                               # (:498-510) zero for bonds >= threshold
            pen = bond_penalty(bondlength, c)
            en_out = en_out + pen.sum()
            if not c.energy_mult_natoms:
                # the reference does `en_out = out; en_out += total_penalty` in place, so the (whole-batch) penalty also
                # lands in result["out"] (SURVEY App. D-12); reproduced, not fixed
                out = en_out
        if c.calculate_gradient:
            # only d energy / d r leaves this call, so the kernels skip every parameter gradient (in force training the
            # parameter gradients come from the loss's backward through this graph)
            with ops.input_grads_only():
                (dr,) = torch.autograd.grad(en_out, r, grad_outputs=torch.ones_like(en_out),
                                            create_graph=second, retain_graph=second or self.training)
            pair_forces = c.grad_multiplier * dr                         # (:530-539)
            if c.force_mult_natoms:
                pair_forces = pair_forces * g.num_nodes()
            if second or not pair_forces.is_cuda:
                # force training: the reductions stay differentiable torch operators
                src, dst = g.index.src.long(), g.index.dst.long()
                zeros = torch.zeros(g.num_nodes(), 3, device=r.device, dtype=r.dtype)
                forces = zeros.index_add(0, dst, pair_forces)                # copy_e/sum over in-edges (:547-550)
                if c.add_reverse_forces:
                    forces = forces - zeros.index_add(0, src, pair_forces)   # ... minus over out-edges (:555-563)
            else:
                # inference / MD: one deterministic kernel for both reductions (csrc/graph_device.cu)
                forces = ops.pair_force_scatter(pair_forces, g.index, c.add_reverse_forces)
            forces = torch.squeeze(forces)
            result["pair_forces"] = pair_forces
            if c.stresswise_weight != 0:
                if second or not pair_forces.is_cuda:
                    stress = virial_stress(r if second else r.detach(), pair_forces, g.node_graph_offsets(),
                                           g.batch_num_edges(), g.ndata["V"], c.stress_multiplier)
                else:
                    stress = ops.virial_stress(r.detach(), pair_forces, g.edge_graph_offsets64(),
                                               g.node_graph_offsets().long(), g.ndata["V"], c.stress_multiplier)
        if c.link == "log":
            out = torch.exp(out)
        elif c.link == "logit":
            out = torch.sigmoid(out)
        if self.classification:
            out = self.softmax(out)
        result.update(out=out, additional=additional, grad=forces, stresses=stress, atomwise_pred=atomwise_pred)
        return result
