"""Generate tests/golden/ealignn_small.npz by running the UNMODIFIED reference eALIGNN
(alignn/models/ealignn_atomwise.py) on oracle/dgl_stub.  A separate entry point from make_golden.py, which would
rewrite every other fixture.  Run in the authoring container only (needs /root/reference, read-only, and the built
library for the radius graph of the inputs):

    python oracle/make_golden_ealignn.py

Stored: (1) an fp64 model run with remove_torque=False (the reference fails in fp64 with torque removal: its fp32
coordinates meet fp64 forces in torch.cross); (2) an fp32 run with remove_torque=True; (3) remove_net_torque called
directly in fp64 (default dtype fp64, since its buffers take the default dtype) on a one-crystal batch, a batch of
three crystals and a batch of 3 atoms in total; (4) the reference config's field names and defaults and the model's
state_dict keys.  A crystal with a single atom makes the reference's pseudo-inverse branch raise an IndexError, so that
case has no fixture; the tests check it against the oracle.  The oracle restatement is asserted to reproduce every
stored output before anything is written.
"""
import json
import os
import sys
from unittest import mock

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "dgl_stub"))
sys.path.insert(0, REF)

for name in ["jarvis", "jarvis.core", "jarvis.core.atoms", "jarvis.core.specie", "jarvis.core.utils",
             "jarvis.analysis", "jarvis.analysis.structure", "jarvis.analysis.structure.neighbors",
             "matplotlib", "matplotlib.pyplot"]:
    sys.modules.setdefault(name, mock.MagicMock(name=name))

import dgl  # noqa: E402  (the stub)

_stub_graph = dgl.graph


def _graph(data, num_nodes=None, device=None):
    """The reference calls `dgl.graph(..., device=...)` (alignn/models/utils.py:172-176, 208-212); the stub graph lives on
    the CPU, so the keyword is accepted and dropped."""
    return _stub_graph(data, num_nodes)


dgl.graph = _graph
from alignn.models import ealignn_atomwise as ref_e  # noqa: E402
from alignn.models import utils as ref_utils  # noqa: E402

from oracle import alignn_oracle as O  # noqa: E402
from oracle import ealignn_oracle as EO  # noqa: E402
from oracle import ealignn_inputs as EI  # noqa: E402
from oracle import golden_inputs as GI  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "ealignn_small.npz")


def graphs(a, dtype):
    f = lambda t: t.to(dtype)  # noqa: E731
    dg = dgl.DGLGraph(a["src"], a["dst"], int(a["bnn"].sum()), a["bnn"].clone(), a["bne"].clone())
    og = O.OGraph(a["src"], a["dst"], int(a["bnn"].sum()), a["bnn"], a["bne"])
    for g in (dg, og):
        g.ndata.update(frac_coords=f(a["frac"]), V=f(a["V"]), atom_features=f(a["atom_features"]))
        g.edata.update(r=f(a["r"]), images=f(a["images"]))
    return dg, og


def oracle_model(dtype):
    m = O.ALIGNN(norm="layernorm", alignn_layers=2, gcn_layers=2, hidden_features=64, embedding_features=32,
                 atom_input_features=EI.ATOM_FEATURES).to(dtype)
    return m


def main():
    a = EI.batch_arrays()
    store = {"in_crc": GI.checksum(a["src"], a["dst"], a["frac"], a["r"], a["images"], a["atom_features"])}
    for tag, dtype, torque, tol in (("f64", torch.float64, False, 1e-11), ("f32", torch.float32, True, 2e-5)):
        ref = ref_e.eALIGNNAtomWise(ref_e.eALIGNNAtomWiseConfig(name="ealignn_atomwise", remove_torque=torque,
                                                                **EI.MODEL_CFG)).to(dtype)
        GI.fill_state_dict(ref, EI.MODEL_SEED)
        ref.eval()
        dg, og = graphs(a, dtype)
        res = ref((dg, a["lattice"].to(dtype)))
        orc = oracle_model(dtype)
        orc.load_state_dict(ref.state_dict())
        o = EO.ealignn_forward(orc, og, a["lattice"].to(dtype), alignn_layers=2, remove_torque=torque,
                              stresswise_weight=0.1, stress_multiplier=10.0)
        for k, rk in (("out", "out"), ("forces", "grad"), ("stress", "stresses")):
            want = res[rk].detach()
            err = (o[k] - want).abs().max().item()
            assert err <= tol * max(1.0, want.abs().max().item()), (tag, k, err)
            store[f"{tag}.{k}"] = want.numpy()
        store[f"{tag}.pair_forces"] = o["pair_forces"].numpy()
        store[f"{tag}.kept"] = o["kept"].numpy()
        store[f"{tag}.T"] = np.asarray(o["T"])
        print(tag, "E =", int(a["bne"].sum()), "kept =", o["kept"].tolist(), "T =", o["T"])

    torch.set_default_dtype(torch.float64)
    for name, (pos, forces, nn_) in EI.torque_cases().items():
        g = dgl.graph((torch.zeros(0, dtype=torch.int64), torch.zeros(0, dtype=torch.int64)), num_nodes=pos.shape[0])
        g.ndata["cart_coords"] = pos
        want = ref_utils.remove_net_torque(g, forces, nn_)
        got = EO.remove_net_torque(pos, forces, nn_)
        assert (got - want).abs().max() <= 1e-12 * max(1.0, want.abs().max().item()), name
        store[f"torque.{name}"] = want.numpy()
    torch.set_default_dtype(torch.float32)

    cfg = ref_e.eALIGNNAtomWiseConfig(name="ealignn_atomwise")
    fields = {k: v for k, v in cfg.model_dump().items()}
    store["config_json"] = np.asarray(json.dumps(fields))
    store["config_fields"] = np.asarray(list(type(cfg).model_fields))
    store["state_dict_keys"] = np.asarray(list(ref_e.eALIGNNAtomWise(cfg).state_dict().keys()))
    np.savez_compressed(OUT, **store)
    print("written", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
