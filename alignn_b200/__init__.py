"""alignn_b200: H100-native (sm_90a) edge-gated graph-convolution hot path of ALIGNN.

Keeps the reference's ALIGNN / ALIGNNConfig / forward((g, lg, lat)) surface
(alignn/models/alignn.py) on top of hand-written CUDA kernels behind a C-ABI
library (include/alignn_b200.h).  See DESIGN.md.
"""
__version__ = "0.1.0"

from .graph import Graph, batch, unbatch, reverse, graph, as_graph, bond_cosines  # noqa: F401
from .ealignn_atomwise import eALIGNNAtomWise, eALIGNNAtomWiseConfig  # noqa: F401,E402
from .relax import relax_structures, RelaxResult, CellRelaxResult  # noqa: F401,E402
from .md import run_md, maxwell_boltzmann_momenta, upper_triangular, MDResult, NPTResult  # noqa: F401,E402
from .phonons import phonons, PhononResult  # noqa: F401,E402
from .eos import ev_curve, fit_eos, single_point, EOSFit, EVCurveResult, SinglePointResult  # noqa: F401,E402
