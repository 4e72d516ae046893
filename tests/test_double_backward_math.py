"""CPU: the double backward of the LayerNorm edge-gated conv (alignn_b200_egc_backward_vjp), written out as explicit
torch code in fp64, against `torch.autograd.grad` through the torch-operator composition `conv._torch_ops_forward`;
plus the C ABI of the new entry point (struct layout, argument checks, no spills).  `double_backward_reference` is
also the fp64 reference of the GPU tests in tests/test_gpu_double_backward.py."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from alignn_b200 import _lib
from alignn_b200 import conv as CV
from alignn_b200.alignn_atomwise import EdgeGatedGraphConv as ConvLN
from alignn_b200.graph import Graph
from oracle import golden_inputs as GI

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PARAMS = ("src_gate.weight", "src_gate.bias", "dst_gate.weight", "dst_gate.bias", "edge_gate.weight", "edge_gate.bias",
          "bn_edges.weight", "bn_edges.bias", "src_update.weight", "src_update.bias", "dst_update.weight",
          "dst_update.bias", "bn_nodes.weight", "bn_nodes.bias")


def _ln_silu_parts(m, w, b, eps):
    mu = m.mean(1, keepdim=True)
    rho = 1.0 / torch.sqrt(((m - mu) ** 2).mean(1, keepdim=True) + eps)
    xh = (m - mu) * rho
    u = xh * w + b
    s = torch.sigmoid(u)
    return rho, xh, s * (1 + u * (1 - s)), s * (1 - s) * (2 + u * (1 - 2 * s))


def _ln_silu_backward(m, gout, w, b, eps):
    """Row gradient gm = d/dm [gout . silu(LayerNorm(m) w + b)] (the first backward)."""
    rho, xh, s1, _ = _ln_silu_parts(m, w, b, eps)
    gxh = gout * s1 * w
    return rho * (gxh - gxh.mean(1, keepdim=True) - xh * (gxh * xh).mean(1, keepdim=True))


def _ln_silu_backward_vjp(m, gout, w, b, eps, gam):
    """VJP of (m, gout, w, b) -> gm with cotangent gam: (m_bar, gout_bar, w_bar, b_bar)."""
    rho, xh, s1, s2 = _ln_silu_parts(m, w, b, eps)
    gu = gout * s1
    gxh = gu * w
    c = (gxh * xh).mean(1, keepdim=True)
    gm = rho * (gxh - gxh.mean(1, keepdim=True) - xh * c)
    gp = rho * gam
    p, q = gp.mean(1, keepdim=True), (gp * xh).mean(1, keepdim=True)
    gxh_bar = gp - p - xh * q
    xh_bar = -c * gp - q * gxh
    gu_bar = gxh_bar * w
    gout_bar = gu_bar * s1
    u_bar = gu_bar * gout * s2
    xh_bar = xh_bar + u_bar * w
    w_bar = (gxh_bar * gu + u_bar * xh).sum(0)
    m_bar = rho * (xh_bar - xh_bar.mean(1, keepdim=True) - xh * (xh_bar * xh).mean(1, keepdim=True)) \
        - rho * (gam * gm).mean(1, keepdim=True) * xh
    return m_bar, gout_bar, w_bar, u_bar.sum(0)


def double_backward_reference(mod, src, dst, x, y, gx_out, gy_out, gx_bar, gy_bar):
    """Cotangents of the first backward's inputs, (x, y, gx_out, gy_out, parameters), given the cotangents gx_bar,
    gy_bar of its outputs gx, gy.  gy_out None: dead edge output.  Follows the formulas of csrc/egc_vjp.cu."""
    d = x.shape[1]
    Nn = x.shape[0]
    s, t = src.long(), dst.long()
    p = {k: v.detach() for k, v in mod.named_parameters()}
    Wcat = torch.cat([p["src_gate.weight"], p["dst_update.weight"], p["dst_gate.weight"], p["src_update.weight"]])
    bcat = torch.cat([p["src_gate.bias"], p["dst_update.bias"], p["dst_gate.bias"] + p["edge_gate.bias"],
                      p["src_update.bias"]])
    Weg = p["edge_gate.weight"]
    nw, nb, ew, eb = p["bn_nodes.weight"], p["bn_nodes.bias"], p["bn_edges.weight"], p["bn_edges.bias"]
    eps_n, eps_e = mod.bn_nodes.eps, mod.bn_edges.eps

    def seg(v, idx):
        return torch.zeros(Nn, d, dtype=x.dtype).index_add(0, idx, v)
    # forward
    P = x @ Wcat.T + bcat
    A, C, B, D = P.split(d, 1)
    M = y @ Weg.T + A[s] + B[t]
    sg = torch.sigmoid(M)
    sp = sg * (1 - sg)
    spp = sp * (1 - 2 * sg)
    S = seg(sg, t)
    r = 1.0 / (S + CV.GATE_EPS)
    H = seg(C[s] * sg, t) * r
    XP = D + H
    # first backward
    gXP = _ln_silu_backward(XP, gx_out, nw, nb, eps_n)
    gM = _ln_silu_backward(M, gy_out, ew, eb, eps_e) if gy_out is not None else torch.zeros_like(M)
    gSh, gS = gXP * r, -gXP * H * r
    gM = gM + (gSh[t] * C[s] + gS[t]) * sp
    GP = torch.cat([seg(gM, s), seg(gSh[t] * sg, s), seg(gM, t), gXP], 1)
    # second backward: through gx = GP Wcat (+ gx_out), gy = gM W_eg (+ gy_out)
    GPb = gx_bar @ Wcat.T
    gAb, gCb, gBb, gDb = GPb.split(d, 1)
    Wcat_bar = GP.T @ gx_bar
    Weg_bar = gM.T @ gy_bar
    Gam = gy_bar @ Weg.T + gAb[s] + gBb[t]
    out = {"gx_out": gx_bar.clone() if mod.residual else torch.zeros_like(gx_bar)}
    zero = torch.zeros(d, dtype=x.dtype)
    if gy_out is not None:
        Mb, gyo_b, ew_b, eb_b = _ln_silu_backward_vjp(M, gy_out, ew, eb, eps_e, Gam)
        out["gy_out"] = gyo_b + (gy_bar if mod.residual else 0)
    else:
        Mb, ew_b, eb_b = torch.zeros_like(M), zero, zero
    Mb = Mb + Gam * (gSh[t] * C[s] + gS[t]) * spp + gCb[s] * gSh[t] * sp
    gShb, gSb = seg(Gam * C[s] * sp + gCb[s] * sg, t), seg(Gam * sp, t)
    gXPb = gDb + (gShb - gSb * H) * r
    XPb, gxo_b, nw_b, nb_b = _ln_silu_backward_vjp(XP, gx_out, nw, nb, eps_n, gXPb)
    out["gx_out"] = out["gx_out"] + gxo_b
    Hb = XPb - gSb * gXP * r
    Shb = Hb * r
    Sb = -Hb * H * r - (gShb - gSb * H) * gXP * r * r
    Mb = Mb + (Shb[t] * C[s] + Sb[t]) * sp
    Pb = torch.cat([seg(Mb, s), seg(Gam * gSh[t] * sp + Shb[t] * sg, s), seg(Mb, t), XPb], 1)
    # through the forward GEMMs
    out["x"], out["y"] = Pb @ Wcat, Mb @ Weg
    Wcat_bar = Wcat_bar + Pb.T @ x
    Weg_bar = Weg_bar + Mb.T @ y
    bcat_bar = Pb.sum(0)
    for i, name in enumerate(("src_gate", "dst_update", "dst_gate", "src_update")):
        out[f"g.{name}.weight"] = Wcat_bar[i * d:(i + 1) * d]
        out[f"g.{name}.bias"] = bcat_bar[i * d:(i + 1) * d]
    out["g.edge_gate.weight"], out["g.edge_gate.bias"] = Weg_bar, bcat_bar[2 * d:3 * d]
    out["g.bn_nodes.weight"], out["g.bn_nodes.bias"] = nw_b, nb_b
    out["g.bn_edges.weight"], out["g.bn_edges.bias"] = ew_b, eb_b
    return out


def double_backward_autograd(mod, g, x, y, gx_out, gy_out, gx_bar, gy_bar, need_edge_out=True):
    """The same cotangents from torch.autograd through `conv._torch_ops_forward`."""
    x, y, gx_out = (t.clone().requires_grad_(True) for t in (x, y, gx_out))
    gy_out = gy_out.clone().requires_grad_(True) if need_edge_out else None
    xo, yo = CV._torch_ops_forward(mod, g.index, x, y, need_edge_out)
    first = (xo * gx_out).sum() + ((yo * gy_out).sum() if need_edge_out else 0.0)
    gx, gy = torch.autograd.grad(first, (x, y), create_graph=True)
    second = (gx * gx_bar).sum() + (gy * gy_bar).sum()
    params = dict(mod.named_parameters())
    inputs = [x, y, gx_out] + ([gy_out] if need_edge_out else []) + [params[k] for k in PARAMS]
    grads = list(torch.autograd.grad(second, inputs, allow_unused=True))
    out = {"x": grads.pop(0), "y": grads.pop(0), "gx_out": grads.pop(0)}
    if need_edge_out:
        out["gy_out"] = grads.pop(0)
    for k, gr in zip(PARAMS, grads):
        out["g." + k] = torch.zeros_like(params[k]) if gr is None else gr
    return out


def ragged_hub_graph(n=12, seed=0):
    """Multigraph with isolated nodes (0-2, 8-11 receive nothing) and a hub with 70 in-edges (three 32-edge chunks)."""
    rng = np.random.default_rng(seed)
    src = np.concatenate([rng.integers(0, n, 70), rng.integers(0, n, 20)])
    dst = np.concatenate([np.full(70, 3), rng.integers(4, 8, 20)])
    return Graph(src, dst, n)


def make_case(g, d, seed, residual=True, dtype=torch.float64):
    mod = ConvLN(d, d, residual=residual)
    GI.fill_state_dict(mod, seed)
    mod = mod.to(dtype)
    Nn, Ne = g.num_nodes(), g.num_edges()
    f = lambda k, n: GI.features(seed + k, n, d).to(dtype)  # noqa: E731
    return mod, f(1, Nn), f(2, Ne), f(3, Nn), f(4, Ne), f(5, Nn), f(6, Ne)


CASES = [("residual", True, True), ("no_residual", False, True), ("dead_edge_out", True, False)]


@pytest.mark.parametrize("tag,residual,need_edge_out", CASES)
@pytest.mark.parametrize("d", [32, 64])
def test_explicit_double_backward_matches_autograd(tag, residual, need_edge_out, d):
    g = ragged_hub_graph()
    mod, x, y, gxo, gyo, gxb, gyb = make_case(g, d, 17, residual)
    want = double_backward_autograd(mod, g, x, y, gxo, gyo, gxb, gyb, need_edge_out)
    got = double_backward_reference(mod, g.index.src, g.index.dst, x, y, gxo, gyo if need_edge_out else None, gxb, gyb)
    assert set(got) == set(want)
    for k in want:
        err = (got[k] - want[k]).abs().max().item()
        scale = max(want[k].abs().max().item(), 1e-30)
        assert err <= 1e-10 * scale, f"{tag} d={d} {k}: {err:.3e} vs scale {scale:.3e}"


def test_explicit_double_backward_edgeless_graph():
    g = Graph(np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.int64), 5)
    mod, x, y, gxo, gyo, gxb, gyb = make_case(g, 32, 3)
    want = double_backward_autograd(mod, g, x, y, gxo, gyo, gxb, gyb)
    got = double_backward_reference(mod, g.index.src, g.index.dst, x, y, gxo, gyo, gxb, gyb)
    for k in want:
        assert got[k].shape == want[k].shape and torch.isfinite(got[k]).all(), k
        if got[k].numel():
            assert (got[k] - want[k]).abs().max().item() <= 1e-10 * max(want[k].abs().max().item(), 1e-30), k


def test_vjp_struct_matches_c_layout(tmp_path):
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "alignn_b200.h"\n'
                   'int main(){printf("%zu %zu %zu %zu %zu\\n", sizeof(alignn_b200_egc_bwd_vjp_args),'
                   'offsetof(alignn_b200_egc_bwd_vjp_args, P), offsetof(alignn_b200_egc_bwd_vjp_args, GPbar),'
                   'offsetof(alignn_b200_egc_bwd_vjp_args, partials_src), offsetof(alignn_b200_egc_bwd_vjp_args, stream));'
                   'return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(t) for t in subprocess.check_output([str(exe)]).split()]
    A = _lib.EgcBwdVjpArgs
    assert got == [ctypes.sizeof(A), A.P.offset, A.GPbar.offset, A.partials_src.offset, A.stream.offset]


def test_vjp_bad_arguments_are_rejected_without_touching_the_gpu():
    lib = _lib.load()
    size = ctypes.sizeof(_lib.EgcBwdVjpArgs)
    call = lambda **kw: lib.alignn_b200_egc_backward_vjp(ctypes.byref(_lib.EgcBwdVjpArgs(**kw)))  # noqa: E731
    assert call(struct_size=1) == -3
    assert call(struct_size=size, d=48, Nn=4, Ne=4, norm=_lib.NORM_LAYER) == -2
    assert call(struct_size=size, d=64, Nn=4, Ne=4, norm=_lib.NORM_LAYER) == -1           # NULL pointers
    # the norm mode is checked first: an empty graph is a no-op for LayerNorm and an error for the BatchNorm modes
    assert call(struct_size=size, d=64, Nn=0, Ne=0, norm=_lib.NORM_LAYER) == 0
    assert call(struct_size=size, d=64, Nn=0, Ne=0, norm=_lib.NORM_AFFINE) == -1
    assert call(struct_size=size, d=64, Nn=0, Ne=0, norm=_lib.NORM_STATS) == -1


def _nvcc():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    return nvcc if os.path.exists(nvcc) else shutil.which("nvcc")


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not available")
def test_vjp_kernels_do_not_spill(tmp_path):
    csrc = os.path.join(ROOT, "alignn_b200", "csrc")
    cmd = [_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-cubin",
           "-I" + os.path.join(ROOT, "include"), "-I" + csrc, "-o", str(tmp_path / "egc_vjp.cubin"),
           os.path.join(csrc, "egc_vjp.cu")]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    report, current = {}, None
    for line in res.stderr.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            current = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and current is not None:
            report[current] = (int(m.group(1)), int(m.group(2)))
            current = None
    for kernel in ("egc_vjp_dst_kernel", "egc_vjp_src_kernel"):
        found = {n: sp for n, sp in report.items() if kernel in n}
        assert sorted(int(re.search(r"ILi(\d+)E", n).group(1)) for n in found) == [32, 64, 128, 256], report
        assert all(sp == (0, 0) for sp in found.values()), found
