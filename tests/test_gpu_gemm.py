"""GPU (-m gpu): the wgmma bf16x3 Linear kernel against an fp64 matmul.

Tolerance 2e-5 relative to the output scale: the bf16x3 split drops terms of relative size
<= 3*2^-18 per product (tc_common.cuh), ~4e-6 rms on a K=256 dot product."""
import pytest
import torch

from alignn_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _ref(A, W, bias, R):
    out = A.double() @ W.double().t()
    if bias is not None:
        out += bias.double()
    if R is not None:
        out += R.double()
    return out


@pytest.mark.parametrize("M,N,K", [(128, 128, 32), (128, 256, 256), (1000, 256, 256), (1920, 1024, 256),
                                   (23040, 256, 1024), (333, 64, 64), (77, 32, 32), (5000, 128, 128)])
def test_gemm_nt_matches_fp64(M, N, K):
    g = torch.Generator(device="cpu").manual_seed(M + N + K)
    A = torch.randn(M, K, generator=g).to(DEV)
    W = (torch.randn(N, K, generator=g) / K ** 0.5).to(DEV)
    bias = torch.randn(N, generator=g).to(DEV)
    R = torch.randn(M, N, generator=g).to(DEV)
    img = ops.WeightImage(W)
    for b, r in ((None, None), (bias, None), (bias, R)):
        out = ops.gemm_nt(A, img, b, r)
        ref = _ref(A, W, b, r)
        err = (out.double() - ref).abs().max().item()
        assert err <= 2e-5 * ref.abs().max().item(), (M, N, K, err, ref.abs().max().item())


def test_gemm_transposed_weight_and_strided_input():
    """Data-gradient form: C = G[M,N'] @ W[N',K'] uses the image of W^T; A may be a column slice."""
    g = torch.Generator(device="cpu").manual_seed(5)
    G = torch.randn(700, 1024, generator=g).to(DEV)
    W = (torch.randn(256, 256, generator=g) / 16).to(DEV)            # Linear weight [out, in]
    img_t = ops.WeightImage(W, transpose=True)                        # acts as W^T: N = in, K = out
    A = G[:, 256:512]                                                 # row stride 1024
    out = ops.gemm_nt(A, img_t)
    ref = A.double() @ W.double()
    assert (out.double() - ref).abs().max().item() <= 2e-5 * ref.abs().max().item()


def test_gemm_extreme_magnitudes():
    """bf16 has fp32's exponent range: large / tiny activations keep the same relative accuracy."""
    g = torch.Generator(device="cpu").manual_seed(9)
    for scale in (1e-20, 1e12):
        A = (torch.randn(256, 256, generator=g) * scale).to(DEV)
        W = (torch.randn(256, 256, generator=g) / 16).to(DEV)
        out = ops.gemm_nt(A, ops.WeightImage(W))
        ref = A.double() @ W.double().t()
        assert (out.double() - ref).abs().max().item() <= 2e-5 * ref.abs().max().item()


def test_gemm_rejects_bad_shapes():
    W = torch.zeros(48, 64, device=DEV)
    with pytest.raises(RuntimeError):
        ops.WeightImage(W)
    img = ops.WeightImage(torch.zeros(64, 64, device=DEV))
    with pytest.raises(RuntimeError):
        ops.gemm_nt(torch.zeros(8, 32, device=DEV), img)


@pytest.mark.parametrize("K,D,groups", [(32, 256, 1), (1000, 256, 1), (23040, 256, 4), (276480, 256, 1), (5000, 128, 4),
                                        (777, 64, 1), (130, 32, 4), (3, 256, 1)])
def test_wgrad_matches_fp64(K, D, groups):
    g = torch.Generator(device="cpu").manual_seed(K + D)
    A = torch.randn(K, groups * D, generator=g).to(DEV)
    B = torch.randn(K, D, generator=g).to(DEV)
    out = ops.wgrad(A, B, groups)
    ref = A.double().t() @ B.double()
    err = (out.double() - ref).abs().max().item()
    assert err <= 2e-5 * ref.abs().max().item(), (K, D, groups, err, ref.abs().max().item())
    assert torch.equal(out, ops.wgrad(A, B, groups))          # deterministic split-K


@pytest.mark.parametrize("K,DA,DB", [(276480, 256, 64), (23040, 256, 96), (5000, 64, 96), (777, 64, 32), (777, 32, 64),
                                     (5000, 32, 96)])
def test_wgrad_rectangular_matches_fp64(K, DA, DB):
    """Embedding-MLP weight gradients: [out, in_padded] with out != in."""
    g = torch.Generator(device="cpu").manual_seed(K + DA + DB)
    A = torch.randn(K, DA, generator=g).to(DEV)
    B = torch.randn(K, DB, generator=g).to(DEV)
    out = ops.wgrad(A, B, 1)
    ref = A.double().t() @ B.double()
    assert out.shape == (DA, DB)
    assert (out.double() - ref).abs().max().item() <= 2e-5 * ref.abs().max().item()
    assert not ops.wgrad_supported(48, 64)


# ---- gemm_gather: Linear with gather-add epilogue and column statistics (csrc/gemm_tc.cu) ----------------------------
@pytest.mark.parametrize("M,N,K", [(1, 32, 32), (127, 64, 64), (128, 256, 256), (129, 128, 96), (1000, 256, 256),
                                   (1920, 1024, 256), (23040, 256, 1024), (5000, 64, 96), (276480, 256, 256)])
def test_gemm_gather_plain_matches_fp64_and_gemm_nt(M, N, K):
    g = torch.Generator(device="cpu").manual_seed(M + N + K)
    A = torch.randn(M, K, generator=g).to(DEV)
    W = (torch.randn(N, K, generator=g) / K ** 0.5).to(DEV)
    bias = torch.randn(N, generator=g).to(DEV)
    img = ops.WeightImage(W)
    for b in (None, bias):
        out = ops.gemm_gather(A, img, b)
        ref = _ref(A, W, b, None)
        err = (out.double() - ref).abs().max().item()
        assert err <= 2e-5 * ref.abs().max().item(), (M, N, K, err, ref.abs().max().item())
        # same operand split, same MMA order, same epilogue association: bit-identical to the register-fed kernel
        assert torch.equal(out, ops.gemm_nt(A, img, b))


@pytest.mark.parametrize("M,Nn,d", [(5, 3, 32), (384, 32, 64), (1000, 77, 128), (23040, 1920, 256), (70001, 5000, 256)])
def test_gemm_gather_edge_gate_matches_fp64(M, Nn, d):
    """m = e_src[src] + e_dst[dst] + edge_gate(y) and its column sums (alignn.py:98-101, 123)."""
    g = torch.Generator(device="cpu").manual_seed(M + Nn + d)
    y = torch.randn(M, d, generator=g).to(DEV)
    W = (torch.randn(d, d, generator=g) / d ** 0.5).to(DEV)
    P = torch.randn(Nn, 4 * d, generator=g).to(DEV)
    src = torch.randint(0, Nn, (M,), generator=g).to(torch.int32).to(DEV)
    dst = torch.randint(0, Nn, (M,), generator=g).to(torch.int32).to(DEV)
    img = ops.WeightImage(W)
    out, part = ops.gemm_gather(y, img, None, add0=P[:, 0:d], idx0=src, add1=P[:, 2 * d:3 * d], idx1=dst, stats=True)
    ref = y.double() @ W.double().t() + P[:, 0:d].double()[src.long()] + P[:, 2 * d:3 * d].double()[dst.long()]
    scale = ref.abs().max().item()
    assert (out.double() - ref).abs().max().item() <= 2e-5 * scale
    s = part.double().sum(0)
    assert (s[0] - ref.sum(0)).abs().max().item() <= 1e-5 * ref.abs().sum(0).max().item()
    assert (s[1] - (ref * ref).sum(0)).abs().max().item() <= 1e-5 * (ref * ref).sum(0).max().item()
    # deterministic
    out2, part2 = ops.gemm_gather(y, img, None, add0=P[:, 0:d], idx0=src, add1=P[:, 2 * d:3 * d], idx1=dst, stats=True)
    assert torch.equal(out, out2) and torch.equal(part, part2)


def test_gemm_gather_residual_and_strided_views():
    """Data-gradient form with the residual in the epilogue: gy = GM W + gy_out; A a column slice of a wider matrix."""
    g = torch.Generator(device="cpu").manual_seed(11)
    G = torch.randn(3000, 1024, generator=g).to(DEV)
    W = (torch.randn(256, 256, generator=g) / 16).to(DEV)
    R = torch.randn(3000, 256, generator=g).to(DEV)
    img_t = ops.WeightImage(W, transpose=True)
    A = G[:, 512:768]
    out = ops.gemm_gather(A, img_t, None, add0=R)
    ref = A.double() @ W.double() + R.double()
    assert (out.double() - ref).abs().max().item() <= 2e-5 * ref.abs().max().item()


# ---- wgrad_batch: many square weight gradients in one launch (csrc/wgrad_tc.cu, alignn_b200_wgrad_batch) ------------
@pytest.mark.parametrize("d", [256, 64, 32])
def test_wgrad_batch_matches_fp64_and_is_deterministic(d):
    g = torch.Generator(device="cpu").manual_seed(d)
    Ks = [0, 1, 31, 33, 1920, 1920, 23040, 5000, 70001, 128, 276480 if d == 256 else 40000]
    problems, refs = [], []
    for i, K in enumerate(Ks):
        wide = torch.randn(K, 4 * d, generator=g).to(DEV)                 # A is a column block of a wider matrix (GP)
        A = wide[:, (i % 4) * d:(i % 4 + 1) * d]
        B = torch.randn(K, d, generator=g).to(DEV)
        out = torch.full((d, d), float("nan"), device=DEV)
        problems.append((A, B, out))
        refs.append(A.double().t() @ B.double())
    ops.wgrad_batch(problems)
    first = [p[2].clone() for p in problems]
    for (A, B, out), ref, K in zip(problems, refs, Ks):
        assert torch.isfinite(out).all()
        err = (out.double() - ref).abs().max().item()
        assert err <= 2e-5 * max(ref.abs().max().item(), 1e-30) + (0 if K else 0), (K, err)
        if K:
            # same products as the single-problem kernel up to the order of the split-K partial sums
            single = ops.wgrad(A.contiguous(), B, 1)
            assert (out - single).abs().max().item() <= 2e-5 * ref.abs().max().item()
    ops.wgrad_batch(problems)
    for a, (_, _, out) in zip(first, problems):
        assert torch.equal(a, out)


def test_wgrad_batch_more_problems_than_one_launch_holds():
    g = torch.Generator(device="cpu").manual_seed(1)
    d = 64
    problems, refs = [], []
    for i in range(ops.WGRAD_BATCH_MAX + 7):
        K = 50 + 13 * i
        A, B = torch.randn(K, d, generator=g).to(DEV), torch.randn(K, d, generator=g).to(DEV)
        problems.append((A, B, torch.empty(d, d, device=DEV)))
        refs.append(A.double().t() @ B.double())
    ops.wgrad_batch(problems)
    for (_, _, out), ref in zip(problems, refs):
        assert (out.double() - ref).abs().max().item() <= 2e-5 * ref.abs().max().item()


def test_deferred_weight_gradients_equal_immediate_ones():
    """FlatGradAllReducer.deferring(): the conv layers queue their weight gradients, gather() computes them with one
    batched launch into the flat buffer.  Same gradients as the launch-by-launch path (split-K order differs)."""
    from alignn_b200 import dp, synthetic
    from alignn_b200.alignn import ALIGNN, ALIGNNConfig
    g, lg, lat, tgt = (t.to(DEV) for t in synthetic.make_batch(6, 9, 12, seed=5, vary_atoms=True))
    flats = []
    launches = []
    for deferred in (False, True):
        torch.manual_seed(0)
        model = ALIGNN(ALIGNNConfig(name="alignn", alignn_layers=2, gcn_layers=2, hidden_features=64, embedding_features=32)).to(DEV).train()
        red = dp.FlatGradAllReducer(model.parameters())
        for it in range(2):                                            # the first backward discovers the trainable set
            red.zero_grad()
            loss = (model((g, lg, lat)) - tgt).abs().mean()
            from alignn_b200 import _lib
            l0 = _lib.launch_count()
            if deferred:
                with red.deferring():
                    loss.backward()
            else:
                loss.backward()
            red.gather()
            l1 = _lib.launch_count()
        flats.append(red.flat.clone())
        launches.append(l1 - l0)
        assert all(p.grad is not None and p.grad.data_ptr() == v.data_ptr() for p, v in zip(red.active, red.views))
    a, b = flats
    assert (a - b).abs().max().item() <= 2e-5 * a.abs().max().item()
    assert launches[1] < launches[0] - 10                               # 4 convs x (2 launches -> 0) + ... -> 1 batched launch
