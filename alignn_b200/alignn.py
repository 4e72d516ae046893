"""ALIGNN property model on the H100 edge-gated conv kernels.

Host-side mirror of the reference module alignn/models/alignn.py: same public names
(`ALIGNNConfig`, `EdgeGatedGraphConv`, `ALIGNNConv`, `MLPLayer`, `ALIGNN`), same constructor
arguments, same `forward((g, lg, lat))` call, same state_dict keys (SURVEY.md App. A) -- so
`alignn/pretrained.py:293-300` style loading (`ALIGNN(ALIGNNConfig(**cfg)); load_state_dict(...)`)
works unchanged.  Graph arguments may be `alignn_b200.Graph` objects or anything DGLGraph-like.

Only the conv stack (alignn.py:317-322) is custom CUDA; the embedding MLPs and the final Linear
are plain library layers (they are rows "next" in SURVEY.md section 8f).
"""
from __future__ import annotations

from typing import Literal, Optional

import numpy as np
import torch
from pydantic_settings import BaseSettings, SettingsConfigDict
from torch import nn

from . import ops
from .conv import ALIGNNConvBase, EdgeGatedGraphConvBase, second_order
from .graph import as_graph


class ALIGNNConfig(BaseSettings):
    """Hyperparameter schema, field-for-field the reference's (alignn/models/alignn.py:19-45)."""

    model_config = SettingsConfigDict(env_prefix="jv_model")

    name: Literal["alignn"]
    alignn_layers: int = 4
    gcn_layers: int = 4
    atom_input_features: int = 92
    edge_input_features: int = 80
    triplet_input_features: int = 40
    embedding_features: int = 64
    hidden_features: int = 256
    output_features: int = 1
    link: Literal["identity", "log", "logit"] = "identity"
    zero_inflated: bool = False
    classification: bool = False
    num_classes: int = 2
    extra_features: int = 0


class RBFExpansion(nn.Module):
    """Gaussian radial basis on a uniform grid (alignn/models/utils.py:11-44).

    With lengthscale=None the width is gamma = 1 / mean(diff(centers)) -- not squared
    (utils.py:30-34) -- which pretrained weights depend on.
    """

    def __init__(self, vmin: float = 0, vmax: float = 8, bins: int = 40, lengthscale: Optional[float] = None):
        super().__init__()
        self.vmin, self.vmax, self.bins = vmin, vmax, bins
        self.register_buffer("centers", torch.linspace(vmin, vmax, bins))
        if lengthscale is None:
            self.lengthscale = float(np.diff(self.centers.numpy()).mean())
            self.gamma = 1.0 / self.lengthscale
        else:
            self.lengthscale = lengthscale
            self.gamma = 1.0 / (lengthscale ** 2)

    def forward(self, distance: torch.Tensor) -> torch.Tensor:
        delta = distance.unsqueeze(1) - self.centers
        return torch.exp(-self.gamma * delta * delta)


def mlp_forward(layer: nn.Sequential, x: torch.Tensor) -> torch.Tensor:
    """Linear -> norm -> SiLU.  On CUDA fp32 inputs the Linear (forward, data gradient, weight gradient) runs on
    the wgmma bf16x3 kernels when its shape is one the library supports (the angle/bond embeddings act on
    T = 276 480 rows per batch); train-mode BatchNorm, LayerNorm and (without autograd) eval-mode BatchNorm run fused with
    the SiLU on the library's row kernels (SURVEY.md section 8f row 3)."""
    lin, norm = layer[0], layer[1]
    if second_order.active:                 # force / stress training: everything must be differentiable twice
        return layer(x)
    if x.is_cuda and x.dtype == torch.float32 and x.dim() == 2 and ops.tc_linear_supported(lin.in_features, lin.out_features):
        if (isinstance(norm, nn.BatchNorm1d) and norm.training and norm.momentum is not None and norm.affine
                and torch.is_grad_enabled()):
            return ops.mlp_bn_train(x, lin, norm)        # Linear + batch statistics + normalise + SiLU on library kernels
        if (isinstance(norm, nn.LayerNorm) and norm.elementwise_affine and norm.bias is not None
                and tuple(norm.normalized_shape) == (lin.out_features,)):
            return ops.mlp_ln(x, lin, norm)              # Linear, then LayerNorm + SiLU in one row kernel each way
        h = ops.tc_linear(x, lin)
        if isinstance(norm, nn.BatchNorm1d) and not norm.training and norm.affine and norm.track_running_stats and not h.requires_grad:
            rstd = torch.rsqrt(norm.running_var + norm.eps)
            scale = norm.weight * rstd
            return ops.affine_silu_residual(h, None, scale, norm.bias - norm.running_mean * scale)
    else:
        h = lin(x)
    return layer[2](norm(h))


class MLPLayer(nn.Module):
    """Linear -> BatchNorm1d -> SiLU, submodule name `layer` (alignn.py:170-184)."""

    def __init__(self, in_features: int, out_features: int):
        super().__init__()
        self.layer = nn.Sequential(nn.Linear(in_features, out_features), nn.BatchNorm1d(out_features), nn.SiLU())

    def forward(self, x):
        return mlp_forward(self.layer, x)


class EdgeGatedGraphConv(EdgeGatedGraphConvBase):
    """BatchNorm1d variant (alignn/models/alignn.py:48-129)."""

    def __init__(self, input_features: int, output_features: int, residual: bool = True):
        super().__init__(input_features, output_features, residual, norm="batchnorm")


class ALIGNNConv(ALIGNNConvBase):
    """alignn/models/alignn.py:132-167."""

    conv_cls = EdgeGatedGraphConv


def _pool(g, x):
    return ops.segment_mean(x, g.node_graph_offsets())


class ALIGNN(nn.Module):
    """Atomistic line graph network: 4 ALIGNN + 4 gated-GCN layers by default (alignn.py:187-349)."""

    _mlp = MLPLayer
    _alignn_conv = ALIGNNConv
    _gcn_conv = EdgeGatedGraphConv

    def __init__(self, config: ALIGNNConfig = ALIGNNConfig(name="alignn")):
        super().__init__()
        self.config = config
        self.classification = config.classification
        c, mlp = config, self._mlp
        self.atom_embedding = mlp(c.atom_input_features, c.hidden_features)
        self.edge_embedding = nn.Sequential(
            RBFExpansion(vmin=0, vmax=8.0, bins=c.edge_input_features),
            mlp(c.edge_input_features, c.embedding_features),
            mlp(c.embedding_features, c.hidden_features))
        self.angle_embedding = nn.Sequential(
            RBFExpansion(vmin=-1, vmax=1.0, bins=c.triplet_input_features),
            mlp(c.triplet_input_features, c.embedding_features),
            mlp(c.embedding_features, c.hidden_features))
        self.alignn_layers = nn.ModuleList(
            [self._alignn_conv(c.hidden_features, c.hidden_features) for _ in range(c.alignn_layers)])
        self.gcn_layers = nn.ModuleList(
            [self._gcn_conv(c.hidden_features, c.hidden_features) for _ in range(c.gcn_layers)])
        if self.classification:
            self.fc = nn.Linear(c.hidden_features, c.num_classes)
            self.softmax = nn.LogSoftmax(dim=1)
        else:
            self.fc = nn.Linear(c.hidden_features, c.output_features)
        if c.extra_features != 0:           # Gong et al. arXiv:2208.05039 (alignn.py:250-266)
            w = c.extra_features + c.hidden_features
            self.extra_feature_embedding = mlp(c.extra_features, c.extra_features)
            self.fc3 = nn.Linear(w, c.output_features)
            self.fc1 = mlp(w, w)
            self.fc2 = mlp(w, w)
        self.link_name = c.link
        if c.link == "log":                 # bias starts at log(mean band gap), alignn.py:273-278
            self.fc.bias.data = torch.tensor(np.log(0.7), dtype=torch.float)

    # -- the hot path --------------------------------------------------------------------------
    def conv_stack(self, g, lg, x, y, z):
        """4x ALIGNNConv then 4x EdgeGatedGraphConv (alignn.py:317-322).

        The last ALIGNN layer's z and the last GCN layer's y are never read again
        (SURVEY.md App. D-11), so those two edge outputs are not materialised.
        """
        n_al, n_gcn = len(self.alignn_layers), len(self.gcn_layers)
        for i, layer in enumerate(self.alignn_layers):
            x, y, z = layer(g, lg, x, y, z, _need_z_out=(i + 1 < n_al))
        for i, layer in enumerate(self.gcn_layers):
            x, y = layer(g, x, y, _need_edge_out=(i + 1 < n_gcn))
        return x, y

    def refresh_images(self):
        """One table-driven launch rebuilds the bf16 operand images of every conv and embedding Linear whose weight
        changed since the last call (training: once per step; inference: once)."""
        dev = self.fc.weight.device
        if dev.type != "cuda":
            return
        tbl = getattr(self, "_alignn_b200_images", None)
        if tbl is None or tbl.device != dev:
            tbl = ops.ImageTable(dev)
            for m in self.modules():
                if isinstance(m, EdgeGatedGraphConvBase):
                    tbl.absorb(m.image_table())
                elif isinstance(m, nn.Sequential) and len(m) == 3 and isinstance(m[0], nn.Linear) and \
                        ops.tc_linear_supported(m[0].in_features, m[0].out_features):
                    tbl.absorb(ops.linear_table(m[0]))
            object.__setattr__(self, "_alignn_b200_images", tbl)
        tbl.refresh()

    def forward(self, g):
        """`g` is the 3-sequence (g, lg, lat) of alignn.py:294 (lat unused, as in the reference)."""
        self.refresh_images()
        z = lg = None
        if len(self.alignn_layers) > 0:
            g, lg, _lat = g
            lg = as_graph(lg)
            z = self.angle_embedding(lg.edata["h"])
        elif isinstance(g, (tuple, list)):
            g = g[0]
        g = as_graph(g)
        feats = None
        if self.config.extra_features != 0:
            feats = self.extra_feature_embedding(g.ndata["extra_features"])
        x = self.atom_embedding(g.ndata["atom_features"])
        y = self.edge_embedding(torch.norm(g.edata["r"], dim=1))
        x, y = self.conv_stack(g, lg, x, y, z)
        h = _pool(g, x)
        if feats is not None:
            h = torch.cat((h, _pool(g, feats)), 1)
            out = self.fc3(self.fc2(self.fc1(h)))
        else:
            out = self.fc(h)
        if self.link_name == "log":
            out = torch.exp(out)
        elif self.link_name == "logit":
            out = torch.sigmoid(out)
        if self.classification:
            out = self.softmax(out)
        return torch.squeeze(out)
