"""Train-mode BatchNorm backward statistics taken in the epilogue of the consumer's data-gradient GEMM.

`gemm_gather(..., bn_bwd=(R, scale, shift, mean, rstd))` leaves the per-CTA partial sums of gu and gu * xhat over its
output C (the incoming gradient of the BatchNorm + SiLU whose input is R), and the autograd Functions hand them from
consumer to producer (ops.bn_fold_offer / bn_fold_take / bn_backward_stats).  Checked here:
  - the epilogue sums against fp64 at the bench's shapes, C bitwise unchanged by the request, bitwise repeatable;
  - a bench-shaped BatchNorm-train step runs one bn_backward_reduce (the last GCN's node BatchNorm, whose gradient
    comes from the pool) and matches the path with the fold switched off; CUDA-graph replay equals eager;
  - every case where the producer cannot use the partials falls back to bn_backward_reduce and gives bitwise the
    result of the path without the fold.
The compile check of the new kernel instantiations runs without a GPU."""
import gc
import os
import re
import shutil
import subprocess
import weakref

import pytest
import torch

from alignn_b200 import ops, synthetic
from alignn_b200.alignn import ALIGNN, ALIGNNConfig, MLPLayer

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "alignn_b200", "csrc")


def _nvcc():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    return nvcc if os.path.exists(nvcc) else shutil.which("nvcc")


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not available")
def test_bn_bwd_kernels_no_spills_stack_or_serialized_wgmma(tmp_path):
    cmd = [_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-cubin",
           "-I" + os.path.join(ROOT, "include"), "-I" + CSRC, "-o", str(tmp_path / "gemm_tc.cubin"),
           os.path.join(CSRC, "gemm_tc.cu")]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    report, current = {}, None
    for line in res.stderr.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            current = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and current is not None:
            report[current] = tuple(int(v) for v in m.groups())
            current = None
    bnb = {name: v for name, v in report.items() if "gemm_bf16x3_bn_bwd_kernel" in name}
    assert sorted(re.search(r"ILi(\d+)E", n).group(1) for n in bnb) == ["128", "32", "64"], report
    assert all(v == (0, 0, 0) for v in bnb.values()), bnb
    serialized = [line for line in res.stderr.splitlines() if "wgmma.mma_async instructions are serialized" in line]
    assert not serialized, serialized


# ---- the epilogue mode ------------------------------------------------------------------------------------------------
def _bn_operands(M, N, K, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    A = torch.randn(M, K, generator=g).to(DEV)
    W = (torch.randn(N, K, generator=g) / K ** 0.5).to(DEV)
    R = (torch.randn(M, N, generator=g) * 1.5 + 0.3).to(DEV)
    mean = R.double().mean(0).float()
    rstd = torch.rsqrt(R.double().var(0, unbiased=False) + 1e-5).float()
    gamma = (1.0 + 0.2 * torch.randn(N, generator=g)).to(DEV)
    beta = (0.1 * torch.randn(N, generator=g)).to(DEV)
    scale = gamma * rstd
    shift = beta - mean * scale
    return g, A, W, R, (R, scale.contiguous(), shift.contiguous(), mean.contiguous(), rstd.contiguous())


def _fp64_sums(C, vecs):
    R, scale, shift, mean, rstd = (t.double() for t in vecs)
    u = R * scale + shift
    s = torch.sigmoid(u)
    gu = C.double() * (s * (1 + u * (1 - s)))
    xhat = (R - mean) * rstd
    return gu.sum(0), (gu * xhat).sum(0), gu.abs().sum(0), (gu * xhat).abs().sum(0)


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K,residual", [(276480, 256, 256, True), (23040, 256, 256, False), (1920, 256, 1024, True),
                                            (276480, 64, 256, False), (2 * 132 * 128 + 77, 128, 64, True),
                                            (1001, 32, 32, True)])
def test_epilogue_sums_match_fp64(M, N, K, residual):
    g, A, W, R, vecs = _bn_operands(M, N, K, M + N + K)
    img = ops.WeightImage(W)
    add0 = torch.randn(M, N, generator=g).to(DEV) if residual else None
    plain = ops.gemm_gather(A, img, add0=add0)
    C, part = ops.gemm_gather(A, img, add0=add0, bn_bwd=vecs)
    assert torch.equal(C, plain)                                         # C bitwise what the plain call writes
    s = part.double().sum(0)
    s1, s2, a1, a2 = _fp64_sums(C, vecs)
    assert ((s[0] - s1).abs() <= 1e-5 * a1).all()
    assert ((s[1] - s2).abs() <= 1e-5 * a2).all()
    C2, part2 = ops.gemm_gather(A, img, add0=add0, bn_bwd=vecs)
    assert torch.equal(C, C2) and torch.equal(part, part2)
    # and what bn_backward_reduce makes of the same gradient
    c1, c2 = ops.bn_backward_reduce(R, C, *vecs[1:])
    c = ops.colsum(part.view(part.shape[0], 2 * N), 1.0 / M)
    assert ((c[:N].double() - c1.double()).abs() <= 1e-5 * a1 / M).all()
    assert ((c[N:].double() - c2.double()).abs() <= 1e-5 * a2 / M).all()


@pytest.mark.gpu
def test_epilogue_rejections():
    _, A, W, R, vecs = _bn_operands(300, 64, 64, 1)
    img = ops.WeightImage(W)
    with pytest.raises(RuntimeError):
        ops.gemm_gather(A, img, stats=True, bn_bwd=vecs)                 # forward and backward statistics at once
    with pytest.raises(RuntimeError):
        ops.gemm_gather(A, img, add1=R, bn_bwd=vecs)
    with pytest.raises(RuntimeError):
        ops.gemm_gather(A, img, out=R.clone(), bn_bwd=(vecs[0][:, :32],) + vecs[1:])
    with pytest.raises(RuntimeError):
        ops.gemm_gather(A, img, out=R, bn_bwd=vecs)                      # R overlaps C


# ---- the hand-off in a model step -------------------------------------------------------------------------------------
class _CountReduce:
    def __init__(self, monkeypatch):
        self.calls = 0
        orig = ops.bn_backward_reduce

        def counted(*a):
            self.calls += 1
            return orig(*a)
        monkeypatch.setattr(ops, "bn_backward_reduce", counted)


def _reset(model):
    for mod in model.modules():
        if isinstance(mod, torch.nn.BatchNorm1d):
            mod.reset_running_stats()
    for p in model.parameters():
        p.grad = None


def _state(model):
    out = {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}
    out.update({n: b.clone() for n, b in model.named_buffers() if b.dtype.is_floating_point})
    return out


def _run(model, fn, fold):
    prev = ops.bn_fold.enabled
    ops.bn_fold.enabled = fold
    try:
        _reset(model)
        fn()
        torch.cuda.synchronize()
        return _state(model)
    finally:
        ops.bn_fold.enabled = prev


# Linear biases whose gradient is zero in exact arithmetic: src_update feeds the node BatchNorm directly, dst_update
# through the gated mean sum(sigma Bh) / (sum(sigma) + 1e-6), whose weights sum to 1 up to 1e-6; the embedding
# Linears' biases feed their BatchNorm.  What the kernels return for them is rounding noise.
_ZERO_GRAD = re.compile(r"(src_update|dst_update)\.bias$|layer\.0\.bias$")


def _assert_close(a, b, tol=1e-4):
    """Within tol of each tensor's scale.  The biases of _ZERO_GRAD get the scale floor 1e-3 of the largest gradient
    of the model; every other tensor is held to its own scale."""
    assert set(a) == set(b)
    floor = 1e-3 * max(b[n].abs().max().item() for n in b)
    bad = []
    for n in a:
        scale = b[n].abs().max().item()
        if _ZERO_GRAD.search(n):
            scale = max(scale, floor)
        err = (a[n] - b[n]).abs().max().item()
        if err > tol * scale:
            bad.append((n, err, scale))
    assert not bad, bad


@pytest.mark.gpu
def test_bench_step_one_reduce_and_matches_unfused(monkeypatch):
    g, lg, lat, tgt = synthetic.make_batch(batch_size=64, atoms=30, k=12, seed=123)
    g, lg, lat, tgt = g.to(DEV), lg.to(DEV), lat.to(DEV), tgt.to(DEV)
    torch.manual_seed(123)
    model = ALIGNN(ALIGNNConfig(name="alignn")).to(DEV).train()

    def step():
        (model((g, lg, lat)) - tgt).abs().mean().backward()
    count = _CountReduce(monkeypatch)
    ref = _run(model, step, fold=False)
    assert count.calls == 27                                             # 12 node, 10 live edge, 5 embedding BatchNorms
    count.calls = 0
    got = _run(model, step, fold=True)
    assert count.calls == 1                                              # the last GCN's node BatchNorm (pool gradient)
    _assert_close(got, ref)


@pytest.mark.gpu
def test_cuda_graph_replay_bitwise_equal_to_eager(monkeypatch):
    g, lg, lat, tgt = synthetic.make_batch(batch_size=8, atoms=12, k=12, seed=7)
    g, lg, lat, tgt = g.to(DEV), lg.to(DEV), lat.to(DEV), tgt.to(DEV)
    torch.manual_seed(5)
    m = ALIGNN(ALIGNNConfig(name="alignn", alignn_layers=2, gcn_layers=2, hidden_features=64,
                            embedding_features=32)).to(DEV).train()
    count = _CountReduce(monkeypatch)

    def fwd_bwd():
        for p in m.parameters():
            p.grad = None
        loss = (m((g, lg, lat)) - tgt).abs().mean()
        loss.backward()
        return loss
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            fwd_bwd()
    torch.cuda.current_stream().wait_stream(side)
    def grads():
        return {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None}
    _reset(m)
    count.calls = 0
    loss_eager = fwd_bwd().item()
    assert count.calls == 1
    eager = grads()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        loss_g = fwd_bwd()
    gr.replay()
    torch.cuda.synchronize()
    assert loss_g.item() == loss_eager
    graph = grads()
    assert set(graph) == set(eager)
    for n in eager:
        assert torch.equal(eager[n], graph[n]), n


# ---- fallbacks: the producer cannot use the partials and runs bn_backward_reduce ------------------------------------
def _mlps(seed):
    torch.manual_seed(seed)
    return torch.nn.ModuleDict({"a": MLPLayer(40, 64), "b": MLPLayer(64, 256)}).to(DEV).train()


def _inputs(seed, rows=3000):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return torch.randn(rows, 40, generator=g).to(DEV), torch.randn(rows, 256, generator=g).to(DEV)


@pytest.mark.gpu
def test_chain_uses_fold(monkeypatch):
    m = _mlps(1)
    x, w = _inputs(1)
    count = _CountReduce(monkeypatch)
    ref = _run(m, lambda: (m["b"](m["a"](x)) * w).sum().backward(), fold=False)
    count.calls = 0
    got = _run(m, lambda: (m["b"](m["a"](x)) * w).sum().backward(), fold=True)
    assert count.calls == 1                                              # only "b", whose output goes to user code
    _assert_close(got, ref)


def _fallback_case(monkeypatch, fn, expected_calls):
    m = _mlps(2)
    x, w = _inputs(2)
    count = _CountReduce(monkeypatch)
    ref = _run(m, lambda: fn(m, x, w), fold=False)
    count.calls = 0
    got = _run(m, lambda: fn(m, x, w), fold=True)
    assert count.calls == expected_calls
    assert set(got) == set(ref)
    for n in ref:
        assert torch.equal(got[n], ref[n]), n


@pytest.mark.gpu
def test_fallback_tensor_consumed_twice(monkeypatch):
    def fn(m, x, w):
        h = m["a"](x)
        ((m["b"](h) * w).sum() + (h * h).sum()).backward()             # autograd sums two gradients of h
    _fallback_case(monkeypatch, fn, 2)


@pytest.mark.gpu
def test_fallback_hook_scales_gradient_in_place(monkeypatch):
    def fn(m, x, w):
        h = m["a"](x)
        h.register_hook(lambda gr: gr.mul_(2.0))
        (m["b"](h) * w).sum().backward()
    _fallback_case(monkeypatch, fn, 2)


@pytest.mark.gpu
def test_fallback_hook_replaces_gradient(monkeypatch):
    def fn(m, x, w):
        h = m["a"](x)
        h.register_hook(lambda gr: gr * 0.5)
        (m["b"](h) * w).sum().backward()
    _fallback_case(monkeypatch, fn, 2)


@pytest.mark.gpu
def test_retain_graph_two_backwards(monkeypatch):
    m = _mlps(3)
    x, w = _inputs(3)

    def fn():
        loss = (m["b"](m["a"](x)) * w).sum()
        loss.backward(retain_graph=True)
        loss.backward()
    count = _CountReduce(monkeypatch)
    ref = _run(m, fn, fold=False)
    count.calls = 0
    got = _run(m, fn, fold=True)
    assert count.calls == 3          # the first backward folds "a"; the fold is used once, so the second one reduces
    _assert_close(got, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("fold", [True, False])
def test_bn_inputs_freed_by_backward_while_loss_is_kept(monkeypatch, fold):
    """The hand-off keeps no BatchNorm input R alive past backward: with the caller still holding `loss` (and so the
    graph), every R is gone, and the allocator holds what it holds without the fold."""
    g, lg, lat, tgt = synthetic.make_batch(batch_size=8, atoms=12, k=12, seed=11)
    g, lg, lat, tgt = g.to(DEV), lg.to(DEV), lat.to(DEV), tgt.to(DEV)
    torch.manual_seed(11)
    m = ALIGNN(ALIGNNConfig(name="alignn", alignn_layers=2, gcn_layers=2, hidden_features=64,
                            embedding_features=32)).to(DEV).train()
    refs = []
    orig = ops.bn_fold_offer

    def offer(out, R, *vecs):
        refs.append(weakref.ref(R))
        return orig(out, R, *vecs)
    monkeypatch.setattr(ops, "bn_fold_offer", offer)

    def kept_after_backward(on):
        prev = ops.bn_fold.enabled
        ops.bn_fold.enabled = on
        try:
            _reset(m)
            refs.clear()
            loss = (m((g, lg, lat)) - tgt).abs().mean()
            loss.backward()
            gc.collect()
            torch.cuda.synchronize()
            alive = [r for r in refs if r() is not None]
            return loss, len(refs), len(alive), torch.cuda.memory_allocated()
        finally:
            ops.bn_fold.enabled = prev
    loss_off, n_off, alive_off, mem_off = kept_after_backward(False)
    del loss_off
    loss_on, n_on, alive_on, mem_on = kept_after_backward(fold)
    assert n_on == n_off == 5 + 6 + 4              # 5 embedding, 6 node and 4 live edge BatchNorms offered
    assert alive_off == 0 and alive_on == 0
    assert mem_on <= mem_off + 16 * 1024           # less than the smallest R (96 nodes x 64 x 4 bytes)
    del loss_on


@pytest.mark.gpu
def test_layernorm_model_unchanged(monkeypatch):
    from alignn_b200 import alignn_atomwise as AW

    class Model(ALIGNN):
        _mlp, _alignn_conv, _gcn_conv = AW.MLPLayer, AW.ALIGNNConv, AW.EdgeGatedGraphConv
    g, lg, lat, tgt = synthetic.make_batch(batch_size=4, atoms=10, k=12, seed=9)
    g, lg, lat, tgt = g.to(DEV), lg.to(DEV), lat.to(DEV), tgt.to(DEV)
    torch.manual_seed(9)
    m = Model(ALIGNNConfig(name="alignn", alignn_layers=2, gcn_layers=2, hidden_features=64,
                           embedding_features=32)).to(DEV).train()
    count = _CountReduce(monkeypatch)

    def step():
        (m((g, lg, lat)) - tgt).abs().mean().backward()
    ref = _run(m, step, fold=False)
    got = _run(m, step, fold=True)
    assert count.calls == 0
    for n in ref:
        assert torch.equal(got[n], ref[n]), n
