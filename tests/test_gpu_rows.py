"""GPU (-m gpu): the row kernels around the conv stack (csrc/row_kernels.cu) against torch in fp64.

LayerNorm + SiLU: fp32 arithmetic with two-pass row statistics; outputs agree with the fp64 composition to ~1e-6 of the
output scale (tolerance 1e-5), the parameter-gradient sums over n rows to 1e-5 of their scale.
AdamW: same operation order as torch.optim.AdamW's fused kernel; tolerance 1e-6 relative per step."""
import pytest
import torch

from alignn_b200 import _lib, dp, ops
from alignn_b200.alignn import mlp_forward

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _ln_silu_ref(h, gamma, beta, eps):
    return torch.nn.functional.silu(torch.nn.functional.layer_norm(h, (h.shape[1],), gamma, beta, eps))


@pytest.mark.parametrize("n,d", [(1, 32), (7, 64), (1000, 128), (4737, 256), (276480, 64), (100003, 256)])
def test_ln_silu_forward_backward_match_fp64(n, d):
    lib = _lib.load()
    g = torch.Generator(device="cpu").manual_seed(n + d)
    h = (torch.randn(n, d, generator=g) * 3 + 0.5).to(DEV)
    gamma = (torch.rand(d, generator=g) + 0.5).to(DEV)
    beta = torch.randn(d, generator=g).to(DEV)
    go = torch.randn(n, d, generator=g).to(DEV)
    eps = 1e-5
    out = torch.empty_like(h)
    rowstat = torch.empty(n, 2, device=DEV)
    _lib.check(lib.alignn_b200_ln_silu_forward(h.data_ptr(), gamma.data_ptr(), beta.data_ptr(), eps, n, d, out.data_ptr(),
                                                rowstat.data_ptr(), None), "fwd")
    hd = h.double().requires_grad_(True)
    gd, bd = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    ref = _ln_silu_ref(hd, gd, bd, eps)
    assert (out.double() - ref).abs().max().item() <= 1e-5 * max(ref.abs().max().item(), 1.0)
    assert (rowstat[:, 0].double() - h.double().mean(1)).abs().max().item() <= 1e-5
    gh_ref, gg_ref, gb_ref = torch.autograd.grad(ref, (hd, gd, bd), go.double())
    rows = ops.partial_rows(n, d)
    gh = torch.empty_like(h)
    part = torch.empty(rows, 2 * d, device=DEV)
    _lib.check(lib.alignn_b200_ln_silu_backward(h.data_ptr(), go.data_ptr(), rowstat.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
                                                 n, d, gh.data_ptr(), part.data_ptr(), rows, None), "bwd")
    assert (gh.double() - gh_ref).abs().max().item() <= 2e-5 * max(gh_ref.abs().max().item(), 1e-3)
    s = ops.colsum(part).double()
    assert (s[:d] - gg_ref).abs().max().item() <= 1e-5 * max(gg_ref.abs().max().item(), 1.0) * max(1.0, n ** 0.5 / 30)
    assert (s[d:] - gb_ref).abs().max().item() <= 1e-5 * max(gb_ref.abs().max().item(), 1.0) * max(1.0, n ** 0.5 / 30)
    # wrong workspace size is refused, not overrun
    assert lib.alignn_b200_ln_silu_backward(h.data_ptr(), go.data_ptr(), rowstat.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
                                            n, d, gh.data_ptr(), part.data_ptr(), rows + 1, None) != 0


@pytest.mark.parametrize("n,fin,fout", [(500, 40, 64), (3000, 64, 256), (1201, 92, 256), (20000, 80, 64)])
def test_mlp_layernorm_layer_matches_torch_layers(n, fin, fout):
    """Linear -> LayerNorm -> SiLU (alignn_atomwise.py:249-268) through mlp_forward: output, input gradient and all four
    parameter gradients against the same layers evaluated by torch in fp64."""
    torch.manual_seed(n + fin)
    layer = torch.nn.Sequential(torch.nn.Linear(fin, fout), torch.nn.LayerNorm(fout), torch.nn.SiLU()).to(DEV)
    with torch.no_grad():
        layer[1].weight.uniform_(0.5, 1.5)
        layer[1].bias.normal_()
    x = torch.randn(n, fin, device=DEV, requires_grad=True)
    go = torch.randn(n, fout, device=DEV)
    out = mlp_forward(layer, x)
    assert type(out.grad_fn).__name__.startswith("_MLPLNFn")
    grads = torch.autograd.grad(out, [x] + list(layer.parameters()), go)
    ref_layer = torch.nn.Sequential(torch.nn.Linear(fin, fout), torch.nn.LayerNorm(fout), torch.nn.SiLU()).to(DEV).double()
    ref_layer.load_state_dict({k: v.double() for k, v in layer.state_dict().items()})
    xd = x.detach().double().requires_grad_(True)
    ref = ref_layer(xd)
    ref_grads = torch.autograd.grad(ref, [xd] + list(ref_layer.parameters()), go.double())
    assert (out.double() - ref).abs().max().item() <= 1e-4 * ref.abs().max().item()
    for a, b in zip(grads, ref_grads):
        assert a.shape == b.shape
        assert (a.double() - b).abs().max().item() <= 1e-4 * max(b.abs().max().item(), 1e-6)
    # forces-only backward: parameter gradients are skipped, the input gradient is unchanged
    out2 = mlp_forward(layer, x)
    with ops.input_grads_only():
        (gx2,) = torch.autograd.grad(out2, [x], go)
    assert torch.equal(gx2, grads[0])


def test_mlp_eval_batchnorm_without_autograd_matches_torch():
    torch.manual_seed(3)
    layer = torch.nn.Sequential(torch.nn.Linear(64, 256), torch.nn.BatchNorm1d(256), torch.nn.SiLU()).to(DEV)
    with torch.no_grad():
        layer[1].running_mean.normal_()
        layer[1].running_var.uniform_(0.5, 2.0)
        layer[1].weight.uniform_(0.5, 1.5)
        layer[1].bias.normal_()
    layer.eval()
    x = torch.randn(2000, 64, device=DEV)
    with torch.no_grad():
        out = mlp_forward(layer, x)
        ref = layer.double()(x.double())
    assert (out.double() - ref).abs().max().item() <= 1e-4 * ref.abs().max().item()


@pytest.mark.parametrize("n", [5, 1024, 4_100_003])
def test_adamw_flat_matches_torch_adamw(n):
    lib = _lib.load()
    g = torch.Generator(device="cpu").manual_seed(n)
    p0 = torch.randn(n, generator=g).to(DEV)
    p = p0.clone()
    ref_p = torch.nn.Parameter(p0.clone().double())
    ref = torch.optim.AdamW([ref_p], lr=1e-2, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2)
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    step = torch.zeros(1, dtype=torch.int64, device=DEV)
    ticket = torch.zeros(1, dtype=torch.int32, device=DEV)
    for it in range(5):
        grad = torch.randn(n, generator=g).to(DEV)
        gbuf = grad.clone()
        ref_p.grad = grad.double()
        ref.step()
        _lib.check(lib.alignn_b200_adamw_flat(p.data_ptr(), gbuf.data_ptr(), m.data_ptr(), v.data_ptr(), n, 1e-2, 0.9, 0.999, 1e-8,
                                               1e-2, int(it % 2), step.data_ptr(), ticket.data_ptr(), None), "adamw")
        assert step.item() == it + 1 and ticket.item() == 0
        assert (gbuf.abs().max().item() == 0.0) == bool(it % 2)
        assert (p.double() - ref_p.detach()).abs().max().item() <= 2e-6 * (it + 1) * max(ref_p.abs().max().item(), 1.0)


def test_flat_adamw_replays_inside_a_cuda_graph():
    """The device step counter advances on every replay: 3 replays == 3 eager steps of torch.optim.AdamW."""
    torch.manual_seed(0)

    def make():
        torch.manual_seed(1)
        return torch.nn.Sequential(torch.nn.Linear(64, 32), torch.nn.SiLU(), torch.nn.Linear(32, 8)).to(DEV)
    a, b = make(), make()
    x, y = torch.randn(128, 64, device=DEV), torch.randn(128, 8, device=DEV)
    ref_opt = torch.optim.AdamW(a.parameters(), lr=1e-2)
    red = dp.FlatGradAllReducer(b.parameters())
    red.zero_grad()
    (b(x) - y).abs().mean().backward()
    red.gather()
    opt = dp.FlatAdamW(red, lr=1e-2)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())

    def one():
        red.zero_grad()
        (b(x) - y).abs().mean().backward()
        red.gather()
        opt.step()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr, stream=side):
        one()
    for _ in range(3):
        ref_opt.zero_grad(set_to_none=True)
        (a(x) - y).abs().mean().backward()
        ref_opt.step()
        gr.replay()
    torch.cuda.synchronize()
    assert opt.step_count.item() == 3
    for pa, pb in zip(a.parameters(), b.parameters()):
        assert torch.allclose(pa, pb, rtol=1e-5, atol=1e-6)


# ---- ring-staged edge kernels (cp.async into shared memory) are the register-staged kernels, bit for bit -------------
@pytest.mark.parametrize("d", [32, 64, 128, 256])
@pytest.mark.parametrize("mode", ["bn_train", "layernorm", "affine_inference"])
def test_forward_ring_kernel_is_bit_identical_to_register_kernel(d, mode):
    from alignn_b200._lib import NORM_AFFINE, NORM_LAYER, NORM_STATS
    from alignn_b200.graph import Graph
    lib = _lib.load()
    gen = torch.Generator(device="cpu").manual_seed(d)
    Nn = 301
    # ragged in-degrees: empty nodes, one node with 70 in-edges (> one 32-edge chunk), edges in random order (in_eid used)
    deg = torch.randint(0, 9, (Nn,), generator=gen)
    deg[5] = 70
    deg[0] = 0
    deg[Nn - 1] = 0
    dst = torch.repeat_interleave(torch.arange(Nn), deg)
    perm = torch.randperm(dst.numel(), generator=gen)
    dst = dst[perm]
    src = torch.randint(0, Nn, (dst.numel(),), generator=gen)
    for sort in (False, True):
        if sort:
            order = torch.argsort(dst, stable=True)
            src, dst = src[order], dst[order]
        gr = Graph(src.numpy(), dst.numpy(), Nn).to(DEV)
        ix = gr.index
        Ne = dst.numel()
        rnd = lambda *s: torch.randn(*s, generator=gen).to(DEV)  # noqa: E731
        x, y, G, P = rnd(Nn, d), rnd(Ne, d), rnd(Ne, d), rnd(Nn, 4 * d)
        vec = [torch.rand(d, generator=gen).to(DEV) + 0.5 for _ in range(4)]
        nn_, ne_, save = {"bn_train": (NORM_STATS, NORM_AFFINE, True), "layernorm": (NORM_LAYER, NORM_LAYER, True),
                          "affine_inference": (NORM_AFFINE, NORM_AFFINE, False)}[mode]
        res = {}
        try:
            for flag in (1, 0):
                lib.alignn_b200_debug_egc_flags(flag)
                res[flag] = ops.egc_forward(ix, x, y, G, P, *vec, norm_nodes=nn_, norm_edges=ne_, residual=True, save=save,
                                            need_edge_out=True, gate_is_m=True)
        finally:
            lib.alignn_b200_debug_egc_flags(0)
        for k in ("x_out", "y_out", "XP", "S", "H", "partials"):
            a, b = res[0][k], res[1][k]
            assert (a is None) == (b is None), k
            if a is not None:
                assert torch.equal(a, b), (k, sort)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_kernels_follow_the_tensors_device_not_the_current_device():
    """A model on cuda:1 in a process whose current device is cuda:0 (plain `model.to('cuda:1')`, no set_device) gives the
    same numbers as on cuda:0: every wrapper launches on the device and stream of its operands (ADVICE r1)."""
    from alignn_b200 import synthetic
    from alignn_b200.alignn import ALIGNN, ALIGNNConfig
    outs = []
    for dev in ("cuda:0", "cuda:1"):
        torch.manual_seed(0)
        model = ALIGNN(ALIGNNConfig(name="alignn", alignn_layers=1, gcn_layers=1, hidden_features=64, embedding_features=32)).to(dev).train()
        g, lg, lat, tgt = (t.to(dev) for t in synthetic.make_batch(4, 8, 12, seed=2, vary_atoms=True))
        red = dp.FlatGradAllReducer(model.parameters())
        assert torch.cuda.current_device() == 0
        for _ in range(2):
            red.zero_grad()
            with red.deferring():
                (model((g, lg, lat)) - tgt).abs().mean().backward()
            red.gather()
        torch.cuda.synchronize(dev)
        outs.append(red.flat.cpu())
    assert torch.equal(outs[0], outs[1])
