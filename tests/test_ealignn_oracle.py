"""CPU: the eALIGNN restatement (oracle) against the unmodified reference's outputs in tests/golden/ealignn_small.npz,
the product's config schema and parameter names against the reference's, and the net-torque removal's defining
property.  Inputs are regenerated from seeds (oracle/ealignn_inputs.py)."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import alignn_oracle as O
from oracle import ealignn_oracle as EO
from oracle import ealignn_inputs as EI
from oracle import golden_inputs as GI


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, "ealignn_small.npz"))


@pytest.fixture(scope="module")
def arrays(gold):
    a = EI.batch_arrays()
    assert GI.checksum(a["src"], a["dst"], a["frac"], a["r"], a["images"], a["atom_features"]) == int(gold["in_crc"])
    return a


def _oracle_graph(a, dtype):
    og = O.OGraph(a["src"], a["dst"], int(a["bnn"].sum()), a["bnn"], a["bne"])
    og.ndata.update(frac_coords=a["frac"].to(dtype), V=a["V"].to(dtype), atom_features=a["atom_features"].to(dtype))
    og.edata.update(r=a["r"].to(dtype), images=a["images"].to(dtype))
    return og


def _oracle_model(dtype):
    m = O.ALIGNN(norm="layernorm", alignn_layers=2, gcn_layers=2, hidden_features=64, embedding_features=32,
                 atom_input_features=EI.ATOM_FEATURES).to(dtype)
    GI.fill_state_dict(m, EI.MODEL_SEED)
    return m


@pytest.mark.parametrize("tag,dtype,torque,tol", [("f64", torch.float64, False, 1e-10), ("f32", torch.float32, True, 2e-5)])
def test_ealignn_oracle_matches_reference(gold, arrays, tag, dtype, torque, tol):
    o = EO.ealignn_forward(_oracle_model(dtype), _oracle_graph(arrays, dtype), arrays["lattice"].to(dtype), alignn_layers=2,
                          remove_torque=torque, stresswise_weight=0.1, stress_multiplier=10.0)
    for k in ("out", "forces", "pair_forces", "stress"):
        want = torch.from_numpy(gold[f"{tag}.{k}"])
        err = (o[k].double() - want.double()).abs().max().item()
        assert err <= tol * max(1.0, want.abs().max().item()), (k, err)
    assert np.array_equal(o["kept"].numpy(), gold[f"{tag}.kept"]) and o["T"] == int(gold[f"{tag}.T"])
    assert int(o["kept"].sum()) < int(arrays["bne"].sum())          # the 4 A cutoff removes bonds of the 5 A graph


@pytest.mark.parametrize("name", ["one_crystal", "batch", "three_atoms"])
def test_remove_net_torque_oracle_and_torch_composition_match_reference(gold, name):
    from alignn_b200.ealignn_atomwise import remove_net_torque_torch
    pos, forces, nn_ = EI.torque_cases()[name]
    want = torch.from_numpy(gold[f"torque.{name}"])
    for got in (EO.remove_net_torque(pos, forces, nn_), remove_net_torque_torch(pos, forces, nn_)):
        assert (got - want).abs().max().item() <= 1e-10 * max(1.0, want.abs().max().item())


def test_net_torque_is_zero_after_removal_one_crystal():
    from alignn_b200.ealignn_atomwise import remove_net_torque_torch
    pos, forces, nn_ = EI.torque_cases()["one_crystal"]
    r = pos - pos.mean(0)
    assert torch.cross(r, forces, dim=1).sum(0).abs().max() > 1e-3
    for f in (EO.remove_net_torque(pos, forces, nn_), remove_net_torque_torch(pos, forces, nn_)):
        assert torch.cross(r, f, dim=1).sum(0).abs().max().item() <= 1e-12 * max(1.0, forces.abs().max().item())


def test_singular_crystal_uses_the_pseudo_inverse():
    """A one-atom crystal whose offset from the batch centre lies on an axis has an exactly singular system; the
    torch composition (per crystal) and the oracle (whole batch) both fall back to the pseudo-inverse."""
    from alignn_b200.ealignn_atomwise import remove_net_torque_torch
    pos = torch.tensor([[0.0, 1.0, 0.0], [0.0, -1.0, 0.0], [1.0, 0.0, 0.5], [1.0, 0.0, -0.5], [4.0, 0.0, 0.0]],
                       dtype=torch.float64)
    forces = torch.from_numpy(np.random.default_rng(3).normal(size=(5, 3)))
    nn_ = torch.tensor([4, 1])
    want = EO.remove_net_torque(pos, forces, nn_)
    got = remove_net_torque_torch(pos, forces, nn_)
    assert torch.isfinite(want).all() and (got - want).abs().max().item() <= 1e-10 * want.abs().max().item()


def test_config_schema_and_state_dict_keys_match_reference(gold):
    from alignn_b200 import eALIGNNAtomWise, eALIGNNAtomWiseConfig
    cfg = eALIGNNAtomWiseConfig(name="ealignn_atomwise")
    assert list(type(cfg).model_fields) == [str(s) for s in gold["config_fields"]]
    assert cfg.model_dump() == json.loads(str(gold["config_json"]))
    assert list(eALIGNNAtomWise(cfg).state_dict().keys()) == [str(s) for s in gold["state_dict_keys"]]
    with pytest.raises(NotImplementedError):
        eALIGNNAtomWise(eALIGNNAtomWiseConfig(name="ealignn_atomwise", extra_features=4))
