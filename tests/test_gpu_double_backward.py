"""GPU (-m gpu): the double backward of the LayerNorm edge-gated conv on the library kernels (create_graph=True through
_EdgeGatedConvFn, alignn_b200_egc_backward_vjp) against the explicit fp64 restatement of
tests/test_double_backward_math.py, and ALIGNN-FF force / stress training on it against the fp64 oracle."""
import os
import sys

import numpy as np
import pytest
import torch

from alignn_b200 import conv as CV
from alignn_b200 import dp, ops, synthetic
from alignn_b200.alignn import EdgeGatedGraphConv as ConvBN
from alignn_b200.alignn_atomwise import ALIGNNAtomWise, ALIGNNAtomWiseConfig
from alignn_b200.alignn_atomwise import EdgeGatedGraphConv as ConvLN
from alignn_b200.graph import Graph
from oracle import alignn_oracle as O
from oracle import golden_inputs as GI
from tests.helpers import assert_close, assert_dict_close, rel_err, to_oracle
from tests.test_double_backward_math import PARAMS, double_backward_reference, ragged_hub_graph

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
from bench_force_training import use_torch_ops_convs  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _inputs(g, d, seed):
    Nn, Ne = g.num_nodes(), g.num_edges()
    f = lambda k, n: GI.features(seed + k, n, d)  # noqa: E731
    return f(1, Nn), f(2, Ne), f(3, Nn), f(4, Ne), f(5, Nn), f(6, Ne)


def _kernel_double_backward(conv, g, x, y, wx, wy, vx, vy, need_edge_out=True, transposed=False):
    """(gx, gy) = grad(<x_out, wx> + <y_out, wy>, (x, y), create_graph=True); then the gradients of <gx, vx> + <gy, vy>
    with respect to x, y, wx (gx_out), wy (gy_out) and every parameter.  transposed=True hands the conv non-contiguous
    (column-major) views of x and y."""
    xi = x.to(DEV).clone().requires_grad_(True)
    yi = y.to(DEV).clone().requires_grad_(True)
    wxi = wx.to(DEV).clone().requires_grad_(True)
    wyi = wy.to(DEV).clone().requires_grad_(True)
    xa, ya = (xi.t().contiguous().t(), yi.t().contiguous().t()) if transposed else (xi, yi)
    if transposed and min(x.shape) > 1:
        assert not xa.is_contiguous()
    xo, yo = conv(g.to(DEV), xa, ya, _need_edge_out=need_edge_out)
    first = (xo * wxi).sum() + ((yo * wyi).sum() if need_edge_out else 0.0)
    gx, gy = torch.autograd.grad(first, (xi, yi), create_graph=True)
    second = (gx * vx.to(DEV)).sum() + (gy * vy.to(DEV)).sum()
    params = dict(conv.named_parameters())
    grads = torch.autograd.grad(second, [xi, yi, wxi, wyi] + [params[k] for k in PARAMS], allow_unused=True)
    out = {"x": grads[0], "y": grads[1], "gx_out": grads[2]}
    if need_edge_out:
        out["gy_out"] = torch.zeros_like(wyi) if grads[3] is None else grads[3]
    for k, gr in zip(PARAMS, grads[4:]):
        out["g." + k] = torch.zeros_like(params[k]) if gr is None else gr
    return out


def _check_conv(g, d, seed, residual=True, need_edge_out=True, transposed=False):
    conv = ConvLN(d, d, residual=residual)
    GI.fill_state_dict(conv, seed)
    ref_mod = ConvLN(d, d, residual=residual)
    GI.fill_state_dict(ref_mod, seed)
    ref_mod = ref_mod.double()
    x, y, wx, wy, vx, vy = _inputs(g, d, seed)
    got = _kernel_double_backward(conv.to(DEV), g, x, y, wx, wy, vx, vy, need_edge_out, transposed)
    want = double_backward_reference(ref_mod, g.index.src, g.index.dst, x.double(), y.double(), wx.double(),
                                     wy.double() if need_edge_out else None, vx.double(), vy.double())
    assert set(got) == set(want)
    assert_dict_close(got, want, what=f"double backward d={d} residual={residual} edge_out={need_edge_out}")
    return got


@pytest.mark.parametrize("d", [32, 64, 128, 256])
def test_double_backward_ragged_graph_all_widths(d):
    g, _, _, _ = synthetic.make_batch(batch_size=3, atoms=9, k=8, seed=d, regular=False, vary_atoms=True)
    _check_conv(g, d, 7)


@pytest.mark.parametrize("residual,need_edge_out", [(False, True), (True, False), (False, False)])
def test_double_backward_residual_and_dead_edge_output(residual, need_edge_out):
    g, _, _, _ = synthetic.make_batch(batch_size=2, atoms=8, k=8, seed=3, regular=False, vary_atoms=True)
    _check_conv(g, 64, 11, residual, need_edge_out)


def test_double_backward_isolated_nodes_and_hub():
    got = _check_conv(ragged_hub_graph(), 64, 5)
    assert all(bool(torch.isfinite(v).all()) for v in got.values())


def test_double_backward_non_contiguous_features():
    """Column-major x and y (a transposed copy, as a slice or permute would give) reach x_bar, y_bar like contiguous ones."""
    g, _, _, _ = synthetic.make_batch(batch_size=2, atoms=8, k=8, seed=6, regular=False, vary_atoms=True)
    got = _check_conv(g, 64, 19, transposed=True)
    assert float(got["x"].abs().max()) > 0 and float(got["y"].abs().max()) > 0


def test_parameter_gradients_of_a_create_graph_backward_refuse_a_second_derivative():
    g = ragged_hub_graph(seed=2)
    conv = ConvLN(64, 64)
    GI.fill_state_dict(conv, 23)
    conv.to(DEV)
    x, y, wx, wy, _, _ = _inputs(g, 64, 23)
    xi = x.to(DEV).requires_grad_(True)
    xo, yo = conv(g.to(DEV), xi, y.to(DEV))
    (gw,) = torch.autograd.grad((xo * wx.to(DEV)).sum() + (yo * wy.to(DEV)).sum(), conv.src_gate.weight,
                                create_graph=True)
    assert gw.requires_grad
    with pytest.raises(NotImplementedError, match="cannot be differentiated again"):
        torch.autograd.grad((gw * gw).sum(), xi)


def test_double_backward_edgeless_graph():
    g = Graph(np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.int64), 5)
    got = _check_conv(g, 64, 13)
    assert got["y"].shape == (0, 64)


def test_double_backward_is_bitwise_repeatable():
    g = ragged_hub_graph(seed=1)
    conv = ConvLN(128, 128)
    GI.fill_state_dict(conv, 21)
    conv.to(DEV)
    args = _inputs(g, 128, 21)
    a = _kernel_double_backward(conv, g, *args)
    b = _kernel_double_backward(conv, g, *args)
    for k in a:
        assert torch.equal(a[k], b[k]), k


def test_batchnorm_conv_create_graph_behaves_as_before():
    """BatchNorm convs have no double backward on the kernels: their create_graph backward stays once-differentiable
    (its result is a constant, as before), and under `second_order` they still run as the torch-operator composition."""
    g, _, _, _ = synthetic.make_batch(batch_size=2, atoms=6, k=6, seed=4)
    conv = ConvBN(64, 64)
    GI.fill_state_dict(conv, 3)
    conv.to(DEV).train()
    x = GI.features(1, g.num_nodes(), 64).to(DEV).requires_grad_(True)
    y = GI.features(2, g.num_edges(), 64).to(DEV).requires_grad_(True)
    gd = g.to(DEV)
    xo, yo = conv(gd, x, y)
    gx, _ = torch.autograd.grad(xo.sum() + yo.sum(), (x, y), create_graph=True)
    assert not gx.requires_grad
    conv.eval()                  # running statistics unchanged by the two evaluations below
    with CV.second_order():
        xo, yo = conv(gd, x, y)
    xr, yr = CV._torch_ops_forward(conv, gd.index, x, y, True)
    assert_close(xo, xr, tol=1e-6, what="x_out")            # (index_add on CUDA sums in no fixed order)
    assert_close(yo, yr, tol=1e-6, what="y_out")
    assert "EdgeGatedConvFn" not in type(xo.grad_fn).__name__


# ---- ALIGNN-FF force and stress training --------------------------------------------------------------------------
FF_CFG = dict(alignn_layers=4, gcn_layers=4, hidden_features=256, atom_input_features=92)


def _ff_batch():
    g, lg, lat, _ = synthetic.make_batch(batch_size=8, atoms=12, k=12, seed=51, vary_atoms=True)
    g.ndata["V"] = GI.cell_volumes(g.batch_num_nodes())
    return g, lg, lat


def _ff_loss(res, tgt_e, tgt_f, tgt_s, gradwise=1.0, stresswise=0.1):
    return ((res["out"] - tgt_e).abs().mean() + gradwise * (res["grad"] - tgt_f).abs().mean()
            + stresswise * (res["stresses"] - tgt_s).abs().mean())


def _ff_model(seed=500):
    m = ALIGNNAtomWise(ALIGNNAtomWiseConfig(name="alignn_atomwise", stresswise_weight=0.1, **FF_CFG))
    GI.fill_state_dict(m, seed)
    return m.to(DEV).train()


def _ff_targets(g):
    B = len(g.batch_num_nodes())
    return GI.features(61, 1, B)[0], GI.features(62, g.num_nodes(), 3), 10 * GI.features(63, B, 9).view(B, 3, 3)


def _ff_step(m, batch, targets):
    g, lg, lat = batch
    for p in m.parameters():
        p.grad = None
    res = m((g.to(DEV), lg.to(DEV), lat.to(DEV)))
    loss = _ff_loss(res, *(t.to(DEV) for t in targets))
    loss.backward()
    return {"g." + n: (p.grad.clone() if p.grad is not None else torch.zeros_like(p)) for n, p in m.named_parameters()}


def test_force_and_stress_training_step_matches_fp64_oracle():
    batch = _ff_batch()
    g, lg, lat = batch
    targets = _ff_targets(g)
    m = _ff_model()
    ops.TIMER = ops.KernelTimer()
    try:
        got = _ff_step(m, batch, targets)
        torch.cuda.synchronize()
        launches = ops.TIMER.summary().get("egc_backward_vjp", {}).get("launches", 0)
    finally:
        ops.TIMER = None
    assert launches == 12, launches                   # every conv of the 4+4 stack took the kernel double backward
    aten = _ff_step(use_torch_ops_convs(_ff_model()), batch, targets)
    orc = O.ALIGNN(norm="layernorm", alignn_layers=4, gcn_layers=4, hidden_features=256).double().train()
    orc.load_state_dict({k: v.double().cpu() for k, v in _ff_model().state_dict().items()})
    og, olg = to_oracle(g, torch.float64), to_oracle(lg, torch.float64)
    out, forces, pair = O.energy_and_forces(orc, og, olg, create_graph=True)
    stress = O.virial_stress(og, pair, g.ndata["V"].double(), 1.0)
    te, tf, ts = (t.double() for t in targets)
    ((out - te).abs().mean() + (forces - tf).abs().mean() + 0.1 * (stress - ts).abs().mean()).backward()
    want = {"g." + n: (p.grad if p.grad is not None else torch.zeros_like(p)) for n, p in orc.named_parameters()}
    worst = lambda d: max(rel_err(d[k], want[k]) for k in want if want[k].abs().max() > 0)  # noqa: E731
    print(f"\n[force training] largest relative gradient error vs fp64: kernels {worst(got):.3e}, "
          f"torch-operator convs {worst(aten):.3e}")
    assert_dict_close(got, want, tol=1e-3, what="force/stress training gradients (kernel double backward vs fp64)")


def test_force_training_step_with_flat_gradient_buffer():
    batch = _ff_batch()
    targets = _ff_targets(batch[0])
    m = _ff_model()
    plain = _ff_step(m, batch, targets)
    red = dp.FlatGradAllReducer(m.parameters())
    red.gather()
    red.zero_grad()
    g, lg, lat = batch
    with red.deferring():
        _ff_loss(m((g.to(DEV), lg.to(DEV), lat.to(DEV))), *(t.to(DEV) for t in targets)).backward()
    red.gather()
    for n, p in m.named_parameters():
        if plain["g." + n].abs().max() > 0:
            assert_close(p.grad, plain["g." + n], tol=1e-5, what=n)
