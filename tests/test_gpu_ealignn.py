"""GPU (-m gpu): eALIGNN on the CUDA path -- the bond cutoff filter and the net-torque kernel of csrc/ff_device.cu
against torch / fp64 restatements, the filtered L(g), and eALIGNNAtomWise (inference and force + stress training)
against the fp64 oracle (oracle.ealignn_oracle.ealignn_forward)."""
import numpy as np
import pytest
import torch

from alignn_b200 import ops, synthetic
from alignn_b200.ealignn_atomwise import eALIGNNAtomWise, eALIGNNAtomWiseConfig
from alignn_b200.graph import Graph, lightweight_graph
from oracle import alignn_oracle as O
from oracle import ealignn_oracle as EO
from oracle import ealignn_inputs as EI
from oracle import golden_inputs as GI
from tests.helpers import assert_close, assert_dict_close

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _random_batch(sizes, k=6, seed=0, images_shift=None):
    """Random crystals: k random out-bonds per atom, coordinates in a 6 A box, integer images in {-1, 0, 1}."""
    rng = np.random.default_rng(seed)
    src, dst, imgs, noff = [], [], [], 0
    for b, n in enumerate(sizes):
        s = np.repeat(np.arange(n), k)
        d = rng.integers(0, n, n * k)
        im = rng.integers(-1, 2, (n * k, 3)).astype(np.float32)
        if images_shift is not None and b == images_shift:
            im += 100.0                                             # every bond of this crystal is far too long
        src.append(s + noff)
        dst.append(d + noff)
        imgs.append(im)
        noff += n
    g = Graph(np.concatenate(src), np.concatenate(dst), noff, torch.tensor(sizes), torch.tensor([n * k for n in sizes]))
    g.edata["images"] = torch.from_numpy(np.concatenate(imgs))
    g.edata["r"] = torch.from_numpy(rng.normal(size=(g.num_edges(), 3)).astype(np.float32))
    cart = torch.from_numpy(rng.uniform(0, 6, (noff, 3)).astype(np.float32))
    return g.to(DEV), cart.to(DEV)


def _filter_restatement(g, cart, cutoff):
    src, dst = g.index.src.long(), g.index.dst.long()
    r = (cart[dst] + g.edata["images"]) - cart[src]
    keep = torch.logical_not(torch.gt(torch.norm(r, dim=1), cutoff))
    eoff = g.edge_graph_offsets64().cpu()
    kept, eids = [], []
    for b in range(g.batch_size):
        kb = keep[eoff[b]:eoff[b + 1]]
        kept.append(int(kb.sum()))
        eids.append(kb.nonzero().reshape(-1) + (0 if g.batch_size > 1 else int(eoff[b])))
    return src[keep].int(), dst[keep].int(), r[keep], torch.cat(eids), torch.tensor(kept)


@pytest.mark.parametrize("case", ["nothing_removed", "one_crystal_loses_all", "none_kept", "one_crystal", "batch64"])
def test_bond_cutoff_filter_matches_mask_and_nonzero(case):
    sizes, cutoff, shift = {"nothing_removed": ([5, 7, 6], 1e4, None), "one_crystal_loses_all": ([5, 7, 6], 5.0, 1),
                            "none_kept": ([5, 7], 1e-3, None), "one_crystal": ([12], 5.0, None),
                            "batch64": ([28 + (b % 5) for b in range(64)], 5.0, None)}[case]
    g, cart = _random_batch(sizes, seed=len(case), images_shift=shift)
    src, dst, r, imgs, eids, kept = ops.bond_cutoff_filter(cart, g.index, g.edata["images"], g.edge_graph_offsets64(), cutoff)
    s_ref, d_ref, r_ref, e_ref, k_ref = _filter_restatement(g, cart, cutoff)
    assert torch.equal(src, s_ref) and torch.equal(dst, d_ref) and torch.equal(eids, e_ref)
    assert torch.equal(r, r_ref)                                     # bit-identical bond vectors
    assert torch.equal(kept, k_ref)
    if case == "nothing_removed":
        assert int(kept.sum()) == g.num_edges()
    if case == "one_crystal_loses_all":
        assert int(kept[1]) == 0 and int(kept.sum()) > 0
    if case == "none_kept":
        assert int(kept.sum()) == 0 and src.numel() == 0
    fg, r2 = lightweight_graph(g, cart, cutoff)
    assert torch.equal(r2, r) and torch.equal(fg.batch_num_edges(), kept)
    lg = fg.line_graph(shared=True)                                  # still valid when nothing is kept
    assert lg.num_nodes() == fg.num_edges()


def test_filtered_line_graph_equals_host_builder_and_carries_parent():
    g, cart = _random_batch([9, 11, 10], seed=5)
    fg, _ = lightweight_graph(g, cart, 5.0)
    assert 0 < fg.num_edges() < g.num_edges()
    lg = fg.line_graph(shared=True)
    host = Graph(fg.index.src.cpu(), fg.index.dst.cpu(), fg.num_nodes(), fg.batch_num_nodes(), fg.batch_num_edges())
    hlg = host.line_graph(shared=True)
    for a, b in zip(lg.edges(), hlg.edges()):
        assert torch.equal(a.cpu(), b)
    assert torch.equal(lg.batch_num_edges(), hlg.batch_num_edges())
    assert lg.index.parent is not None
    assert torch.equal(lg.ndata["images"], fg.edata["images"])


def _torque_cases():
    rng = np.random.default_rng(11)
    t = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float32))  # noqa: E731
    cases = {name: (p.float(), f.float(), n) for name, (p, f, n) in EI.torque_cases().items()}
    cases["batch64"] = (t(rng.normal(size=(2000, 3)) * 5), t(rng.normal(size=(2000, 3))), torch.tensor([31] * 64 + [16]))
    cases["singular"] = (t([[0, 1, 0], [0, -1, 0], [1, 0, 0.5], [1, 0, -0.5], [4, 0, 0]]), t(rng.normal(size=(5, 3))),
                         torch.tensor([4, 1]))
    cases["single_atom"] = (t([[1.0, 2.0, 3.0]]), t([[0.5, -1.0, 2.0]]), torch.tensor([1]))
    cases["three_atoms_two_crystals"] = (t([[0, 1, 0], [0, -1, 0], [3, 0, 0]]), t(rng.normal(size=(3, 3))), torch.tensor([2, 1]))
    return cases


@pytest.mark.parametrize("name", list(_torque_cases()))
def test_remove_net_torque_kernel_matches_fp64(name):
    pos, forces, nn_ = _torque_cases()[name]
    off = torch.zeros(nn_.numel() + 1, dtype=torch.int64)
    off[1:] = torch.cumsum(nn_, 0)
    got = ops.remove_net_torque(pos.to(DEV), forces.to(DEV), off.to(DEV)).cpu()
    want = EO.remove_net_torque(pos.double(), forces.double(), nn_)
    assert torch.isfinite(got).all()
    assert_close(got, want, tol=1e-5, what=f"torque {name}")


def _product_graph(a, cart_coords=False):
    g = Graph(a["src"], a["dst"], int(a["bnn"].sum()), a["bnn"], a["bne"])
    g.ndata.update(frac_coords=a["frac"].float(), V=a["V"].float(), atom_features=a["atom_features"])
    g.edata.update(r=a["r"], images=a["images"].float())
    if cart_coords:
        g.ndata["cart_coords"] = EO.cartesian_coords(a["frac"], a["lattice"], a["bnn"])
    return g.to(DEV)


def _oracle_graph(a, cart_coords=False):
    og = O.OGraph(a["src"], a["dst"], int(a["bnn"].sum()), a["bnn"], a["bne"])
    og.ndata.update(frac_coords=a["frac"], V=a["V"], atom_features=a["atom_features"].double())
    og.edata.update(r=a["r"].double(), images=a["images"])
    if cart_coords:
        og.ndata["cart_coords"] = EO.cartesian_coords(a["frac"], a["lattice"], a["bnn"]).double()
    return og


def _models(**kw):
    # Self-image bonds have recomputed length |image| (images are added as Angstrom), 1 A for a unit image: exactly on
    # the default penalty threshold, where fp32 and fp64 may disagree on whether the penalty applies.  1.05 A keeps the
    # fp64 comparison away from that step.
    cfg = {**EI.MODEL_CFG, "penalty_threshold": 1.05, **kw}
    m = eALIGNNAtomWise(eALIGNNAtomWiseConfig(name="ealignn_atomwise", **cfg))
    GI.fill_state_dict(m, EI.MODEL_SEED)
    orc = O.ALIGNN(norm="layernorm", alignn_layers=cfg["alignn_layers"], gcn_layers=cfg["gcn_layers"], hidden_features=64,
                   embedding_features=32, atom_input_features=EI.ATOM_FEATURES).double()
    orc.load_state_dict({k: v.double() for k, v in m.state_dict().items()})
    return m.to(DEV), orc, cfg


@pytest.mark.parametrize("variant", ["default", "no_torque", "no_alignn_layers", "no_alignn_layers_no_torque",
                                     "energy_not_mult_natoms", "classification"])
def test_ealignn_eval_matches_fp64_oracle(variant):
    kw = {"default": {}, "no_torque": dict(remove_torque=False), "no_alignn_layers": dict(alignn_layers=0),
          "no_alignn_layers_no_torque": dict(alignn_layers=0, remove_torque=False),
          "energy_not_mult_natoms": dict(energy_mult_natoms=False, penalty_threshold=3.0),
          "classification": dict(classification=True)}[variant]
    a = EI.batch_arrays()
    m, orc, cfg = _models(**kw)
    m.eval()
    cart = cfg["alignn_layers"] == 0
    res = m((_product_graph(a, cart), a["lattice"].to(DEV)))
    o = EO.ealignn_forward(orc, _oracle_graph(a, cart), a["lattice"].double(), alignn_layers=cfg["alignn_layers"],
                          remove_torque=cfg.get("remove_torque", True), energy_mult_natoms=cfg.get("energy_mult_natoms", True),
                          penalty_threshold=cfg["penalty_threshold"], stresswise_weight=0.1, stress_multiplier=10.0,
                          classification=cfg.get("classification", False))
    assert_close(res["out"], o["out"], what=f"{variant} out")
    assert_close(res["pair_forces"], o["pair_forces"], what=f"{variant} pair forces")
    assert_close(res["grad"], o["forces"], what=f"{variant} forces")
    assert_close(res["stresses"], o["stress"], tol=1e-3, what=f"{variant} stress")


def test_ealignn_force_stress_training_gradients_match_oracle_double_backward():
    a = EI.batch_arrays()
    m, orc, _ = _models()
    m.train()
    tgt = GI.features(31, int(a["bnn"].sum()), 3)
    res = m((_product_graph(a), a["lattice"].to(DEV)))
    assert res["grad"].requires_grad
    ((res["grad"] - tgt.to(DEV)).abs().mean() + res["out"].abs().mean() + res["stresses"].abs().mean()).backward()
    o = EO.ealignn_forward(orc, _oracle_graph(a), a["lattice"].double(), alignn_layers=2, penalty_threshold=1.05,
                          stresswise_weight=0.1, stress_multiplier=10.0, create_graph=True)
    ((o["forces"] - tgt.double()).abs().mean() + o["out"].abs().mean() + o["stress"].abs().mean()).backward()
    got = {"g." + n: (p.grad if p.grad is not None else torch.zeros_like(p)) for n, p in m.named_parameters()}
    want = {"g." + n: (p.grad if p.grad is not None else torch.zeros_like(p)) for n, p in orc.named_parameters()}
    assert_dict_close(got, want, tol=1e-3, what="eALIGNN force+stress training gradients")


def test_ealignn_repeated_forwards_bitwise_identical():
    a = EI.batch_arrays()
    m, _, _ = _models()
    m.eval()
    g, lat = _product_graph(a), a["lattice"].to(DEV)
    r1, r2 = m((g, lat)), m((g, g, lat))                            # a passed lg is ignored with ALIGNN layers
    for k in ("out", "grad", "pair_forces", "stresses"):
        assert torch.equal(r1[k], r2[k]), k


def test_atomwise_g_lat_call_equals_passing_the_line_graph():
    from alignn_b200.alignn_atomwise import ALIGNNAtomWise, ALIGNNAtomWiseConfig
    g, _, lat, _ = synthetic.make_batch(batch_size=3, atoms=8, k=12, seed=41, vary_atoms=True)
    g.ndata["V"] = GI.cell_volumes(g.batch_num_nodes())
    m = ALIGNNAtomWise(ALIGNNAtomWiseConfig(name="alignn_atomwise", alignn_layers=2, gcn_layers=2, hidden_features=64,
                                            embedding_features=32, atom_input_features=92, stresswise_weight=0.1))
    GI.fill_state_dict(m, 400)
    m.to(DEV).eval()
    gd, latd = g.to(DEV), lat.to(DEV)
    r1 = m((gd, latd))
    r2 = m((gd, gd.line_graph(shared=True), latd))
    for k in ("out", "grad", "pair_forces", "stresses"):
        assert torch.equal(r1[k], r2[k]), k
    m.config.lg_on_fly = False
    with pytest.raises(ValueError):
        m((gd, latd))
