"""Tensor-level wrappers over the C ABI (include/alignn_b200.h).  Device memory, streams
and the autograd glue are PyTorch plumbing; all arithmetic of the edge-gated conv stage
runs in libalignn_b200.so.  Every function raises if the tensors are not fp32/int32 CUDA
tensors or if the library reports an error -- there is no fallback path.
"""
from __future__ import annotations

import ctypes as C
import functools
import math
import weakref
from typing import Optional, Tuple

import torch

from . import _lib
from ._lib import NORM_AFFINE, NORM_LAYER, NORM_STATS, ptr, require_cuda, stream_ptr  # noqa: F401
from .graph import EdgeIndex


def _on_tensor_device(fn):
    """Launch on the device the operands live on, whatever the current device is (a model on cuda:1 in a process whose
    current device is cuda:0 would otherwise enqueue on the wrong device and stream)."""
    @functools.wraps(fn)
    def wrapper(*args, **kw):
        dev = None
        for a in args:
            if isinstance(a, EdgeIndex):
                a = a.src
            elif isinstance(a, (list, tuple)) and a and isinstance(a[0], (list, tuple)) and a[0]:
                a = a[0][0]
            if isinstance(a, torch.Tensor) and a.is_cuda:
                dev = a.device
                break
        if dev is None or dev.index == torch.cuda.current_device():
            return fn(*args, **kw)
        with torch.cuda.device(dev):
            return fn(*args, **kw)
    return wrapper


class KernelTimer:
    """Optional CUDA-event timing of individual library calls (used by bench.py for the roofline
    of the dominant kernel: events are recorded on the launching stream, inside the timed region)."""

    def __init__(self, min_edges: int = 0):
        self.min_edges = min_edges
        self.records = {}      # name -> list of (start_event, end_event, algorithmic_bytes)

    def span(self, name: str, nbytes: int):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        self.records.setdefault(name, []).append((s, e, nbytes))
        return s, e

    def summary(self):
        """name -> launches, total_ms, total algorithmic bytes; plus the same for the largest launches alone
        (`big_*`: the L(g)-sized calls, bytes >= half of the largest)."""
        out = {}
        for name, rec in self.records.items():
            ms = [s.elapsed_time(e) for s, e, _ in rec]
            by = [b for _, _, b in rec]
            top = max(by)
            big = [(m, b) for m, b in zip(ms, by) if 2 * b >= top]
            out[name] = dict(launches=len(ms), total_ms=sum(ms), total_bytes=sum(by), big_launches=len(big),
                             big_ms=sum(m for m, _ in big), big_bytes=sum(b for _, b in big))
        return out


TIMER: Optional[KernelTimer] = None


class _span:
    """`with _span(name, nbytes): <library call>` -- CUDA events around the call on the launching stream when a
    KernelTimer is installed (bench.py); free otherwise."""
    __slots__ = ("ev",)

    def __init__(self, name: str, nbytes: int):
        self.ev = TIMER.span(name, int(nbytes)) if TIMER is not None else None

    def __enter__(self):
        if self.ev is not None:
            self.ev[0].record()

    def __exit__(self, *exc):
        if self.ev is not None:
            self.ev[1].record()


def _check_d(d: int) -> None:
    if d not in _lib.SUPPORTED_D:
        raise RuntimeError(f"alignn_b200: unsupported feature width {d}; supported: {_lib.SUPPORTED_D}")


def partial_rows(num_nodes: int, d: int) -> int:
    return int(_lib.load().alignn_b200_egc_partial_rows(num_nodes, d))


@_on_tensor_device
def egc_forward(ix: EdgeIndex, x, y, G, P, n_w, n_b, e_w, e_b, *, norm_nodes: int, norm_edges: int,
                residual: bool, save: bool, need_edge_out: bool, gate_eps: float = 1e-6, ln_eps: float = 1e-5,
                gate_is_m: bool = False):
    """Everything of EdgeGatedGraphConv.forward after the Linear layers (alignn.py:100-127).

    gate_is_m: G already holds the pre-activation gate m (from `gemm_gather` with the e_src / e_dst addends); the
    kernel then only applies the edge norm / SiLU / residual and reduces the gated messages (second pass over the edges).

    Returns dict(x_out, y_out, M, XP, S, H, partials)."""
    lib = _lib.load()
    Nn, d = x.shape
    Ne = y.shape[0]
    _check_d(d)
    require_cuda(x, y, G, P, n_w, n_b, e_w, e_b, ix.src, ix.in_ptr, ix.in_eid)
    stats = norm_nodes == NORM_STATS or norm_edges == NORM_STATS
    save = save or stats
    dev = x.device
    new = lambda *s: torch.empty(*s, device=dev, dtype=torch.float32)  # noqa: E731
    x_out = None if norm_nodes == NORM_STATS else new(Nn, d)
    y_out = new(Ne, d) if (need_edge_out and norm_edges != NORM_STATS) else None
    if gate_is_m and norm_edges == NORM_STATS and need_edge_out:
        raise RuntimeError("egc_forward(gate_is_m=True): finalize the batch statistics of m first and pass NORM_AFFINE")
    M = (G if gate_is_m else new(Ne, d)) if save else None
    XP, S, H = (new(Nn, d), new(Nn, d), new(Nn, d)) if save else (None, None, None)
    partials = new(partial_rows(Nn, d), 4, d) if stats else None
    a = _lib.EgcFwdArgs(
        struct_size=C.sizeof(_lib.EgcFwdArgs), Nn=Nn, Ne=Ne, d=d, norm_nodes=norm_nodes, norm_edges=norm_edges,
        residual=int(residual), gate_is_m=int(gate_is_m), gate_eps=gate_eps, ln_eps=ln_eps,
        x=ptr(x), y=ptr(y), G=ptr(G), P=ptr(P), src=ptr(ix.src), in_ptr=ptr(ix.in_ptr),
        in_eid=None if ix.dst_sorted else ptr(ix.in_eid),
        n_w=ptr(n_w), n_b=ptr(n_b), e_w=ptr(e_w), e_b=ptr(e_b),
        x_out=ptr(x_out), y_out=ptr(y_out), M=None if gate_is_m else ptr(M), XP=ptr(XP), S=ptr(S), H=ptr(H),
        partials=ptr(partials),
        stream=stream_ptr())
    # compulsory bytes of THIS kernel: read G (or m), P (each element once), indices; residual rows; what it writes
    nb = 4 * d * (Ne + 4 * Nn) + 4 * Ne + 4 * (Nn + 1)
    nb += 4 * d * Ne * (M is not None and not gate_is_m) + 4 * d * Nn * 3 * (XP is not None)
    nb += 4 * d * Ne * (1 + int(residual)) * (y_out is not None) + 4 * d * Nn * (1 + int(residual)) * (x_out is not None)
    with _span("egc_forward" + ("<gate_is_m>" if gate_is_m else ""), nb):
        _lib.check(lib.alignn_b200_egc_forward(C.byref(a)), "alignn_b200_egc_forward")
    return dict(x_out=x_out, y_out=y_out, M=M, XP=XP, S=S, H=H, partials=partials)


@_on_tensor_device
def bn_finalize(partials, which: int, count: int, gamma, beta, eps: float, momentum: float,
                running_mean: Optional[torch.Tensor], running_var: Optional[torch.Tensor]):
    """Batch statistics -> (scale, shift, mean, rstd); updates running stats in place."""
    lib = _lib.load()
    rows, nq, d = partials.shape
    require_cuda(partials, gamma, beta, running_mean, running_var)
    out = torch.empty(4, d, device=partials.device, dtype=torch.float32)
    _lib.check(lib.alignn_b200_bn_finalize(ptr(partials), rows, nq * d, which, count, d, ptr(gamma), ptr(beta), eps,
                                            momentum, ptr(running_mean), ptr(running_var), ptr(out[0]), ptr(out[1]),
                                            ptr(out[2]), ptr(out[3]), stream_ptr()), "alignn_b200_bn_finalize")
    return out[0], out[1], out[2], out[3]


@_on_tensor_device
def affine_silu_residual(R, res, scale, shift):
    lib = _lib.load()
    n, d = R.shape
    _check_d(d)
    require_cuda(R, res, scale, shift)
    out = torch.empty_like(R)
    with _span("affine_silu_residual", 4 * n * d * (2 + (res is not None))):
        _lib.check(lib.alignn_b200_affine_silu_residual(ptr(R), ptr(res), ptr(scale), ptr(shift), ptr(out), n, d,
                                                         stream_ptr()), "alignn_b200_affine_silu_residual")
    return out


@_on_tensor_device
def colsum(a: torch.Tensor, alpha: float = 1.0) -> torch.Tensor:
    """Deterministic fp64-accumulated column sum of a 2-D fp32 tensor (used on partial buffers)."""
    lib = _lib.load()
    require_cuda(a)
    rows, cols = a.shape
    out = torch.empty(cols, device=a.device, dtype=torch.float32)
    _lib.check(lib.alignn_b200_colsum(ptr(a), rows, cols, cols, alpha, ptr(out), stream_ptr()), "alignn_b200_colsum")
    return out


@_on_tensor_device
def bn_backward_reduce(R, g_out, scale, shift, mean, rstd) -> Tuple[torch.Tensor, torch.Tensor]:
    """c1 = mean(gu), c2 = mean(gu*xhat) per channel (BatchNorm train-mode backward, pass 1)."""
    lib = _lib.load()
    n, d = R.shape
    _check_d(d)
    require_cuda(R, g_out, scale, shift, mean, rstd)
    rows = partial_rows(n, d)
    partials = torch.empty(rows, 2 * d, device=R.device, dtype=torch.float32)
    with _span("bn_backward_reduce", 8 * n * d):
        _lib.check(lib.alignn_b200_bn_backward_reduce(ptr(R), ptr(g_out), ptr(scale), ptr(shift), ptr(mean), ptr(rstd), n, d,
                                                       ptr(partials), rows, stream_ptr()), "alignn_b200_bn_backward_reduce")
    c = colsum(partials, 1.0 / n)
    return c[:d], c[d:]


@_on_tensor_device
def egc_backward(ix: EdgeIndex, P, M, XP, S, H, gx_out, gy_out, n, e, *, reduce: bool = True, norm_nodes: int, norm_edges: int,
                 gate_eps: float = 1e-6, ln_eps: float = 1e-5, keep_gsh: bool = False):
    """n / e: dicts with keys w, b, mean, rstd, c1, c2 (entries may be None).

    Returns GM [Ne,d], GP [Nn,4d], vec_dst [6,d], vec_src [2,d] (column sums of the partials); with reduce=False the
    per-block partial rows [rows, 6d] and [rows, 2d] themselves.  keep_gsh=True appends the workspace GSh = dL/dSh
    [Nn,d], which the double backward (`egc_backward_vjp`) reads."""
    lib = _lib.load()
    Nn, d = XP.shape
    Ne = M.shape[0]
    _check_d(d)
    require_cuda(P, M, XP, S, H, gx_out, gy_out, ix.src, ix.dst, ix.in_ptr, ix.in_eid, ix.out_ptr, ix.out_eid,
                 *[t for dct in (n, e) for t in dct.values()])
    dev = XP.device
    new = lambda *s: torch.empty(*s, device=dev, dtype=torch.float32)  # noqa: E731
    GM, GP, GSh = new(Ne, d), new(Nn, 4 * d), new(Nn, d)
    rows = partial_rows(Nn, d)
    part, part_src = new(rows, 6 * d), new(rows, 2 * d)
    g = lambda dct, k: ptr(dct.get(k))  # noqa: E731
    a = _lib.EgcBwdArgs(
        struct_size=C.sizeof(_lib.EgcBwdArgs), Nn=Nn, Ne=Ne, d=d, norm_nodes=norm_nodes, norm_edges=norm_edges,
        gate_eps=gate_eps, ln_eps=ln_eps, P=ptr(P), M=ptr(M), XP=ptr(XP), S=ptr(S), H=ptr(H),
        src=ptr(ix.src), dst=ptr(ix.dst), in_ptr=ptr(ix.in_ptr), in_eid=None if ix.dst_sorted else ptr(ix.in_eid),
        out_ptr=ptr(ix.out_ptr), out_eid=ptr(ix.out_eid),
        n_w=g(n, "w"), n_b=g(n, "b"), n_mean=g(n, "mean"), n_rstd=g(n, "rstd"),
        e_w=g(e, "w"), e_b=g(e, "b"), e_mean=g(e, "mean"), e_rstd=g(e, "rstd"),
        n_c1=g(n, "c1"), n_c2=g(n, "c2"), e_c1=g(e, "c1"), e_c2=g(e, "c2"),
        gx_out=ptr(gx_out), gy_out=ptr(gy_out), GM=ptr(GM), GP=ptr(GP), GSh=ptr(GSh),
        partials=ptr(part), partials_src=ptr(part_src), stream=stream_ptr())
    if ix.parent is not None:
        # L(g) of a parent graph: one pass per parent atom (include/alignn_b200.h).  Compulsory bytes: M, gy_out read
        # and GM written once; node rows XP, gx_out, S, H, Bh read and GP [4d], GSh written; parent CSR + L(g) in_ptr.
        pin, peid, pout, poeid = ix.parent
        require_cuda(pin, peid, pout, poeid)
        a.parent_in_ptr, a.parent_in_eid, a.parent_out_ptr, a.parent_out_eid = ptr(pin), ptr(peid), ptr(pout), ptr(poeid)
        a.parent_Nn = pin.numel() - 1
        name = "egc_backward(line)"
        nb = 4 * d * (Ne * (2 + (gy_out is not None)) + 10 * Nn) + 4 * (2 * pin.numel() + 2 * Nn + Nn + 1)
    else:
        # destination-keyed pass reads M, gy_out, node rows and writes GM, GP; source-keyed pass reads GM, M: SURVEY 8d
        name = "egc_backward(dst+src)"
        nb = 4 * d * (Ne * (2 + (gy_out is not None)) + 9 * Nn) + 12 * Ne + 4 * d * 2 * Ne
    with _span(name, nb):
        _lib.check(lib.alignn_b200_egc_backward(C.byref(a)), "alignn_b200_egc_backward")
    extra = (GSh,) if keep_gsh else ()
    if not reduce:              # the caller sums the per-block partial rows itself (WgradQueue: one batched launch per backward)
        return (GM, GP, part, part_src) + extra
    return (GM, GP, colsum(part).view(6, d), colsum(part_src).view(2, d)) + extra


@_on_tensor_device
def egc_backward_vjp(ix: EdgeIndex, P, M, XP, S, H, gx_out, gy_out, GSh, GPbar, GMbar, gx_bar_res, gy_bar_res,
                     n_w, n_b, e_w, e_b, *, gate_eps: float = 1e-6, ln_eps: float = 1e-5):
    """Double backward of a LayerNorm conv (include/alignn_b200.h, alignn_b200_egc_backward_vjp): the cotangents of
    the first backward's inputs, given GPbar = gx_bar Wcat^T and GMbar = gy_bar W_eg^T (None: zero).  gx_bar_res /
    gy_bar_res are added to the gx_out / gy_out cotangents (the residual), None to skip.

    Returns Pbar [Nn,4d], Mbar [Ne,d], gx_out_bar [Nn,d], gy_out_bar [Ne,d] (None when gy_out is None), and the column
    sums vec_dst [6,d] = {e_w, e_b, n_w, n_b cotangents, sum Pbar_D, sum Pbar_B}, vec_src [2,d] = {sum Pbar_A,
    sum Pbar_C}."""
    lib = _lib.load()
    Nn, d = XP.shape
    Ne = M.shape[0]
    _check_d(d)
    require_cuda(P, M, XP, S, H, gx_out, gy_out, GSh, GPbar, GMbar, gx_bar_res, gy_bar_res, n_w, n_b, e_w, e_b,
                 ix.src, ix.dst, ix.in_ptr, ix.in_eid, ix.out_ptr, ix.out_eid)
    dev = XP.device
    new = lambda *s: torch.empty(*s, device=dev, dtype=torch.float32)  # noqa: E731
    Pbar, Mbar, gxo_bar = new(Nn, 4 * d), new(Ne, d), new(Nn, d)
    gyo_bar = new(Ne, d) if gy_out is not None else None
    Gamma, Shbar = new(Ne, d), new(Nn, d)
    rows = partial_rows(Nn, d)
    part, part_src = new(rows, 6 * d), new(rows, 2 * d)
    a = _lib.EgcBwdVjpArgs(
        struct_size=C.sizeof(_lib.EgcBwdVjpArgs), Nn=Nn, Ne=Ne, d=d, norm=NORM_LAYER, gate_eps=gate_eps, ln_eps=ln_eps,
        P=ptr(P), M=ptr(M), XP=ptr(XP), S=ptr(S), H=ptr(H),
        src=ptr(ix.src), dst=ptr(ix.dst), in_ptr=ptr(ix.in_ptr), in_eid=None if ix.dst_sorted else ptr(ix.in_eid),
        out_ptr=ptr(ix.out_ptr), out_eid=ptr(ix.out_eid),
        n_w=ptr(n_w), n_b=ptr(n_b), e_w=ptr(e_w), e_b=ptr(e_b),
        gx_out=ptr(gx_out), gy_out=ptr(gy_out), GSh=ptr(GSh),
        GPbar=ptr(GPbar), GMbar=ptr(GMbar), gx_bar_res=ptr(gx_bar_res), gy_bar_res=ptr(gy_bar_res),
        Pbar=ptr(Pbar), Mbar=ptr(Mbar), gx_out_bar=ptr(gxo_bar), gy_out_bar=ptr(gyo_bar), Gamma=ptr(Gamma),
        Shbar=ptr(Shbar), partials=ptr(part), partials_src=ptr(part_src), stream=stream_ptr())
    # compulsory bytes: every input row read once and every output row written once; gathered node rows (C, GPbar_A,
    # GPbar_C) count once per node.  node rows: read XP, gx_out, S, H, GSh, the C block of P, GPbar (4 blocks) and
    # gx_bar_res; write Pbar (4 blocks) and gx_out_bar.  edge rows: read M, GMbar, gy_out, gy_bar_res; write Mbar,
    # gy_out_bar; plus the src / dst / eid indices and both pointer arrays.  The workspaces Gamma and Shbar and the
    # re-reads of M and Mbar in the second sweep and the source pass are not compulsory.
    live = gy_out is not None
    nb = 4 * d * Nn * (6 + 4 + (gx_bar_res is not None) + 4 + 1)
    nb += 4 * d * Ne * (1 + (GMbar is not None) + live + (gy_bar_res is not None) + 1 + live) + 12 * Ne + 8 * (Nn + 1)
    with _span("egc_backward_vjp", nb):
        _lib.check(lib.alignn_b200_egc_backward_vjp(C.byref(a)), "alignn_b200_egc_backward_vjp")
    return Pbar, Mbar, gxo_bar, gyo_bar, colsum(part).view(6, d), colsum(part_src).view(2, d)


@_on_tensor_device
def gather_segment_sum(ix: EdgeIndex, Bh, sigma):
    """Sh[v] = sum_{e->v} Bh[src e] * sigma[e];  S[v] = sum_{e->v} sigma[e]  (alignn.py:105-108)."""
    lib = _lib.load()
    Nn, d = Bh.shape
    Ne = sigma.shape[0]
    _check_d(d)
    require_cuda(Bh, sigma, ix.src, ix.in_ptr, ix.in_eid)
    Sh, S = torch.empty_like(Bh), torch.empty_like(Bh)
    _lib.check(lib.alignn_b200_gather_segment_sum(ptr(Bh), ptr(sigma), ptr(ix.src), ptr(ix.in_ptr),
                                                   None if ix.dst_sorted else ptr(ix.in_eid), Nn, Ne, d, ptr(Sh), ptr(S),
                                                   stream_ptr()), "alignn_b200_gather_segment_sum")
    return Sh, S


@_on_tensor_device
def pair_force_scatter(pair_forces: torch.Tensor, ix: EdgeIndex, add_reverse: bool = True) -> torch.Tensor:
    """forces[v] = sum over in-edges of pair_forces - (add_reverse ? sum over out-edges : 0): DGL's
    update_all(copy_e, sum) on g and on dgl.reverse(g) (alignn_atomwise.py:547-563) in one deterministic kernel."""
    lib = _lib.load()
    pf = pair_forces.contiguous()
    require_cuda(pf, ix.in_ptr, ix.in_eid, ix.out_ptr, ix.out_eid)
    Nn = ix.in_ptr.numel() - 1
    out = torch.empty(Nn, 3, device=pf.device, dtype=torch.float32)
    _lib.check(lib.alignn_b200_pair_force_scatter(ptr(pf), ptr(ix.in_ptr), None if ix.dst_sorted else ptr(ix.in_eid), ptr(ix.out_ptr),
                                                  ptr(ix.out_eid), Nn, int(add_reverse), ptr(out), stream_ptr()),
               "alignn_b200_pair_force_scatter")
    return out


@_on_tensor_device
def virial_stress(r: torch.Tensor, pair_forces: torch.Tensor, edge_offsets64: torch.Tensor, node_offsets64: torch.Tensor,
                  V: torch.Tensor, multiplier: float = 1.0) -> torch.Tensor:
    """stress[b] = multiplier * -160.21766208 * (r_b^T F_b) / V[first atom of b], one block per crystal
    (alignn_atomwise.py:610-635)."""
    lib = _lib.load()
    r, pf, V = r.contiguous(), pair_forces.contiguous(), V.contiguous().to(torch.float32)
    B = edge_offsets64.numel() - 1
    out = torch.empty(B, 3, 3, device=r.device, dtype=torch.float32)
    _lib.check(lib.alignn_b200_virial_stress(ptr(r), ptr(pf), edge_offsets64.data_ptr(), node_offsets64.data_ptr(), ptr(V), B,
                                             float(multiplier), ptr(out), stream_ptr()), "alignn_b200_virial_stress")
    return out


@_on_tensor_device
def bond_cutoff_filter(cart: torch.Tensor, ix: EdgeIndex, images: torch.Tensor, edge_offsets64: torch.Tensor,
                       cutoff: float):
    """Bonds of `ix` no longer than `cutoff`, with r = (cart[dst] + images) - cart[src] recomputed in fp32
    (`lightweight_line_graph` + `compute_pair_vector_and_distance`, alignn/models/utils.py:47-55, 129-222).
    Returns (src', dst', r', images', edge_ids, kept bonds per crystal as a host int64 tensor); one read-back of the
    B+1 kept-bond boundaries sizes the outputs."""
    lib = _lib.load()
    cart, images = cart.contiguous(), images.contiguous().to(torch.float32)
    require_cuda(cart, images, ix.src, ix.dst)
    E, dev, B = ix.src.numel(), cart.device, edge_offsets64.numel() - 1
    r = torch.empty(E, 3, device=dev, dtype=torch.float32)
    off = torch.empty(E + 1, device=dev, dtype=torch.int32)
    nb = int(lib.alignn_b200_bond_cutoff_workspace_bytes(E))
    if nb == 0:
        raise ValueError("graph too large for int32 edge index")
    ws = torch.empty(nb, device=dev, dtype=torch.uint8)
    st = stream_ptr()
    _lib.check(lib.alignn_b200_bond_cutoff_offsets(ptr(cart), ptr(ix.src), ptr(ix.dst), ptr(images), E, float(cutoff), ptr(r),
                                                   ptr(off), ptr(ws), nb, st), "alignn_b200_bond_cutoff_offsets")
    at = off[edge_offsets64].cpu()                            # kept bonds before each crystal's first bond; last = E'
    Ek = int(at[-1])
    i32 = lambda: torch.empty(Ek, device=dev, dtype=torch.int32)  # noqa: E731
    src, dst = i32(), i32()
    r_k, img_k = (torch.empty(Ek, 3, device=dev, dtype=torch.float32) for _ in range(2))
    eids = torch.empty(Ek, device=dev, dtype=torch.int64)
    _lib.check(lib.alignn_b200_bond_cutoff_fill(ptr(ix.src), ptr(ix.dst), ptr(r), ptr(images), ptr(off), edge_offsets64.data_ptr(),
                                                B, E, ptr(src), ptr(dst), ptr(r_k), ptr(img_k), eids.data_ptr(), st),
               "alignn_b200_bond_cutoff_fill")
    return src, dst, r_k, img_k, eids, (at[1:] - at[:-1]).long()


@_on_tensor_device
def remove_net_torque(pos: torch.Tensor, forces: torch.Tensor, node_offsets64: torch.Tensor) -> torch.Tensor:
    """Forces with the batch's net torque removed (`remove_net_torque`, alignn/models/utils.py:295-398; batch-wide
    centre and torque, one 3x3 solve per crystal in double, pseudo-inverse for an exactly singular system).  A batch of
    exactly 3 atoms crosses along dim 0, as torch.cross without `dim` does there."""
    lib = _lib.load()
    pos, forces = pos.contiguous(), forces.contiguous()
    require_cuda(pos, forces)
    N, B = forces.shape[0], node_offsets64.numel() - 1
    out = torch.empty(N, 3, device=forces.device, dtype=torch.float32)
    nb = int(lib.alignn_b200_remove_net_torque_workspace_bytes(B))
    ws = torch.empty(nb, device=forces.device, dtype=torch.uint8)
    _lib.check(lib.alignn_b200_remove_net_torque(ptr(pos), ptr(forces), node_offsets64.data_ptr(), B, N, int(N == 3), ptr(out),
                                                 ptr(ws), nb, stream_ptr()), "alignn_b200_remove_net_torque")
    return out


@_on_tensor_device
def remove_net_torque_per_crystal(pos: torch.Tensor, forces: torch.Tensor, node_offsets64: torch.Tensor) -> torch.Tensor:
    """Forces with each crystal's own net torque removed, the crystal's centre and torque taken over its atoms only:
    bit for bit `remove_net_torque` of every crystal as a one-crystal batch (a 3-atom crystal crosses along dim 0), in
    one set of launches for the batch and without a read-back.  node_offsets64 [B+1] int64 on the device; offsets that
    do not start at 0, decrease or do not end at N give NaN forces."""
    lib = _lib.load()
    pos, forces = pos.contiguous(), forces.contiguous()
    require_cuda(pos, forces)
    if node_offsets64.dtype != torch.int64 or node_offsets64.device != forces.device:
        raise ValueError("node_offsets64 must be an int64 tensor on the forces' device")
    N, B = forces.shape[0], node_offsets64.numel() - 1
    if pos.shape != (N, 3) or forces.shape != (N, 3):
        raise ValueError(f"pos and forces must both be [N,3], got {tuple(pos.shape)} and {tuple(forces.shape)}")
    out = torch.empty(N, 3, device=forces.device, dtype=torch.float32)
    nb = int(lib.alignn_b200_remove_net_torque_per_crystal_workspace_bytes(B, N))
    ws = torch.empty(max(nb, 1), device=forces.device, dtype=torch.uint8)
    _lib.check(lib.alignn_b200_remove_net_torque_per_crystal(ptr(pos), ptr(forces), node_offsets64.contiguous().data_ptr(),
                                                             B, N, ptr(out), ptr(ws), nb, stream_ptr()),
               "alignn_b200_remove_net_torque_per_crystal")
    return out


FIRE_DEFAULTS = dict(maxstep=0.2, dtmax=1.0, n_min=5, finc=1.1, fdec=0.5, astart=0.1, fa=0.99)   # ase FIRE defaults
FIRE_DT0, FIRE_A0 = 0.1, 0.1                                                                    # its initial dt and a
FIRE_BAD_INPUT = 3            # istate status of a crystal whose batch slice does not match its atom count
FIRE_MAX_STEPS = 2 ** 31 - 1  # steps travels as an int32


def _operands(name, want, device) -> None:
    """The device, dtype and contiguity checks of the wrapper `name`: every (tensor, dtype or tuple of dtypes) pair of
    `want` is a contiguous CUDA tensor of that dtype on `device`."""
    for t, dt in want:
        if not isinstance(t, torch.Tensor) or not t.is_cuda or t.device != device:
            got = t.device if isinstance(t, torch.Tensor) else type(t).__name__
            raise RuntimeError(f"{name} needs all operands on one CUDA device; got {got} and {device}")
        if (t.dtype not in dt if isinstance(dt, tuple) else t.dtype != dt) or not t.is_contiguous():
            raise RuntimeError(f"{name}: expected a contiguous {dt} tensor, got {t.dtype}")


def _check_int(name, what, v, lo, hi, hi_text=None) -> None:
    """v is an integer in [lo, hi] (hi_text: how the message names hi)."""
    if isinstance(v, bool) or int(v) != v or not lo <= int(v) <= hi:
        raise ValueError(f"{name}: {what} must be an integer in [{lo}, {hi_text or hi}], got {v!r}")


def _md_counts(name, steps, evaluation) -> None:
    _check_int(name, "steps", steps, 1, FIRE_MAX_STEPS)
    _check_int(name, "evaluation", evaluation, 0, int(steps), "steps")


def _fire_params(name, fire, fmax, steps, force_multiplier):
    """The FireParams of one FIRE step: FIRE_DEFAULTS overridden by `fire`."""
    par = dict(FIRE_DEFAULTS, **fire)
    _check_int(name, "steps", steps, 1, FIRE_MAX_STEPS)
    _check_int(name, "n_min", par["n_min"], 0, FIRE_MAX_STEPS)
    return _lib.FireParams(float(par["maxstep"]), float(par["dtmax"]), float(par["finc"]), float(par["fdec"]),
                           float(par["astart"]), float(par["fa"]), float(fmax), int(par["n_min"]), int(steps),
                           float(force_multiplier))


@_on_tensor_device
def fire_step(grad: torch.Tensor, active: torch.Tensor, batch_offsets: torch.Tensor, atom_offsets: torch.Tensor,
              positions: torch.Tensor, velocities: torch.Tensor, forces: torch.Tensor, fstate: torch.Tensor,
              istate: torch.Tensor, *, fmax: float, steps: int, force_multiplier: float = 1.0, **fire) -> None:
    """One FIRE step (ASE 3.22.1 `FIRE.step` with `Optimizer.converged` and the step limit of `Dynamics.irun`) for the
    running crystals listed in `active`, in place, one launch (csrc/fire_device.cu, alignn_b200_fire_step).

    grad [M,3] fp32: the model's forces for the crystals of `active` in that order (batch_offsets [A+1] int32; slice j
    must hold exactly the atoms of crystal active[j]); atom_offsets [B+1] int64 with atom_offsets[B] == N; positions /
    velocities [N,3] float64; forces [N,3] fp32 (written: the scaled forces of this evaluation); fstate [B,2] float64 =
    {dt, a}; istate [B,4] int32 = {Nsteps, first step pending, steps taken, status (0 running, 1 converged, 2 step limit,
    FIRE_BAD_INPUT: slice j is not crystal active[j]'s atoms or lies outside grad -- nothing else is read or written for
    that crystal)}.  Enqueue only: the statuses are the caller's to read back.  `fire` overrides FIRE_DEFAULTS."""
    lib = _lib.load()
    _operands("fire_step", ((grad, torch.float32), (active, torch.int32), (batch_offsets, torch.int32),
                            (atom_offsets, torch.int64), (positions, torch.float64), (velocities, torch.float64),
                            (forces, torch.float32), (fstate, torch.float64), (istate, torch.int32)), grad.device)
    B, A = atom_offsets.numel() - 1, active.numel()
    N = positions.numel() // 3
    if (velocities.numel() != 3 * N or forces.numel() != 3 * N or fstate.numel() != 2 * B or istate.numel() != 4 * B
            or batch_offsets.numel() != A + 1 or grad.dim() != 2 or grad.shape[1] != 3):
        raise ValueError("fire_step: inconsistent operand shapes")
    p = _fire_params("fire_step", fire, fmax, steps, force_multiplier)
    _lib.check(lib.alignn_b200_fire_step(C.byref(p), active.data_ptr(), A, atom_offsets.data_ptr(), batch_offsets.data_ptr(),
                                         B, grad.data_ptr(), grad.shape[0], positions.data_ptr(), velocities.data_ptr(), forces.data_ptr(),
                                         fstate.data_ptr(), istate.data_ptr(), stream_ptr()), "alignn_b200_fire_step")


FIRE_CELL_DEGENERATE = 4      # istate status of a crystal whose cell lost its volume or whose expm(L) is not finite


@_on_tensor_device
def fire_cell_step(grad: torch.Tensor, stress: torch.Tensor, active: torch.Tensor, batch_offsets: torch.Tensor,
                   atom_offsets: torch.Tensor, positions: torch.Tensor, velocities: torch.Tensor, forces: torch.Tensor,
                   cells0: torch.Tensor, logdef: torch.Tensor, defgrad: torch.Tensor, cells: torch.Tensor,
                   cell_velocities: torch.Tensor, cell_forces: torch.Tensor, stress_out: torch.Tensor, fstate: torch.Tensor,
                   istate: torch.Tensor, *, fmax: float, steps: int, force_multiplier: float = 1.0, stress_wt: float = 1.0,
                   **fire) -> None:
    """One FIRE step on ASE 3.22.1's `ExpCellFilter` (atoms and cell together) for the running crystals listed in
    `active`, in place, one launch (csrc/fire_cell_device.cu, alignn_b200_fire_cell_step).

    As `fire_step`, plus: stress [A,3,3] fp32, the model's stress of crystal active[j] in row j; stress_out [B,6] fp32
    (written: the calculator's Voigt stress, eV/A^3); cell_forces [B,3,3] float64 (written: the filter's cell rows);
    the filter state, [B,3,3] float64 each: cells0 (the starting cells), logdef (L, initially 0), defgrad (F = expm(L),
    initially I), cells (C = C0 F^T, initially cells0), cell_velocities (initially 0).  Status FIRE_CELL_DEGENERATE:
    the cell's volume is not finite and > 0, or expm(L) is not finite; the crystal is frozen."""
    lib = _lib.load()
    _operands("fire_cell_step",
              ((grad, torch.float32), (stress, torch.float32), (active, torch.int32), (batch_offsets, torch.int32),
               (atom_offsets, torch.int64), (positions, torch.float64), (velocities, torch.float64),
               (forces, torch.float32), (cells0, torch.float64), (logdef, torch.float64), (defgrad, torch.float64),
               (cells, torch.float64), (cell_velocities, torch.float64), (cell_forces, torch.float64),
               (stress_out, torch.float32), (fstate, torch.float64), (istate, torch.int32)), grad.device)
    B, A = atom_offsets.numel() - 1, active.numel()
    N = positions.numel() // 3
    if (velocities.numel() != 3 * N or forces.numel() != 3 * N or fstate.numel() != 2 * B or istate.numel() != 4 * B
            or batch_offsets.numel() != A + 1 or grad.dim() != 2 or grad.shape[1] != 3
            or stress.numel() != 9 * A or stress_out.numel() != 6 * B
            or any(t.numel() != 9 * B for t in (cells0, logdef, defgrad, cells, cell_velocities, cell_forces))):
        raise ValueError("fire_cell_step: inconsistent operand shapes")
    p = _lib.FireCellParams(_fire_params("fire_cell_step", fire, fmax, steps, force_multiplier), float(stress_wt))
    _lib.check(lib.alignn_b200_fire_cell_step(C.byref(p), active.data_ptr(), A, atom_offsets.data_ptr(), batch_offsets.data_ptr(),
                                              B, grad.data_ptr(), grad.shape[0], stress.data_ptr(), A, positions.data_ptr(),
                                              velocities.data_ptr(), forces.data_ptr(), cells0.data_ptr(), logdef.data_ptr(),
                                              defgrad.data_ptr(), cells.data_ptr(), cell_velocities.data_ptr(),
                                              cell_forces.data_ptr(), stress_out.data_ptr(), fstate.data_ptr(),
                                              istate.data_ptr(), stream_ptr()), "alignn_b200_fire_cell_step")


LBFGS_DEFAULTS = dict(maxstep=0.2, memory=100, damping=1.0, alpha=70.0)   # ase LBFGS defaults (no line search)
BFGS_DEFAULTS = dict(maxstep=0.2, alpha=70.0)                             # ase BFGS defaults
QN_BREAKDOWN = 5              # istate status of a crystal whose quasi-Newton update or step is not finite


def _qn_operands(name, grad, stress, active, batch_offsets, atom_offsets, positions, forces, cell_ops, rows_ops, istate,
                 steps):
    """The operand checks lbfgs_step and bfgs_update share.  Returns (B, A, N, rows, cell)."""
    cell = stress is not None
    want = [(grad, torch.float32), (active, torch.int32), (batch_offsets, torch.int32), (atom_offsets, torch.int64),
            (positions, torch.float64), (forces, torch.float32), (istate, torch.int32)]
    want += [(t, torch.float64) for t in rows_ops]
    if cell:
        want += [(stress, torch.float32), (cell_ops[-1], torch.float32)] + [(t, torch.float64) for t in cell_ops[:-1]]
    _operands(name, want, grad.device)
    B, A = atom_offsets.numel() - 1, active.numel()
    N = positions.numel() // 3
    rows = N + 3 * B if cell else N
    if (forces.numel() != 3 * N or istate.numel() != 4 * B or batch_offsets.numel() != A + 1 or grad.dim() != 2
            or grad.shape[1] != 3 or any(t.numel() != 3 * rows for t in rows_ops[:4])
            or (cell and (stress.numel() != 9 * A or cell_ops[-1].numel() != 6 * B
                          or any(t.numel() != 9 * B for t in cell_ops[:-1])))):
        raise ValueError(f"{name}: inconsistent operand shapes")
    _check_int(name, "steps", steps, 1, FIRE_MAX_STEPS)
    return B, A, N, rows, cell


def _cell_ptrs(cell, cell_ops):
    return [t.data_ptr() for t in cell_ops] if cell else [None] * 6


@_on_tensor_device
def lbfgs_step(grad: torch.Tensor, stress, active: torch.Tensor, batch_offsets: torch.Tensor, atom_offsets: torch.Tensor,
               positions: torch.Tensor, forces: torch.Tensor, cells0, logdef, defgrad, cells, cell_forces, stress_out,
               r0: torch.Tensor, f0: torch.Tensor, work: torch.Tensor, s_ring: torch.Tensor, y_ring: torch.Tensor,
               history: torch.Tensor, istate: torch.Tensor, *, fmax: float, steps: int, force_multiplier: float = 1.0,
               stress_wt: float = 1.0, **lbfgs) -> None:
    """One LBFGS step (ASE 3.22.1 `LBFGS.step` with `Optimizer.converged` and the step limit of `Dynamics.irun`) for the
    running crystals listed in `active`, in place, one launch (csrc/qn_device.cu, alignn_b200_lbfgs_step).

    As `fire_step` for grad, active, batch_offsets, atom_offsets, positions and forces.  stress None: the atoms alone;
    else ExpCellFilter as `fire_cell_step` (stress, cells0, logdef, defgrad, cells, cell_forces, stress_out; no cell
    velocities).  Per-row state, [rows, 3] float64 with rows = N (+ 3B with the filter): r0, f0, work; the history ring
    s_ring, y_ring [slots * rows * 3] float64 and history [B, 2 * slots] float64, slots >= min(memory, steps); istate
    [B,4] int32 = {iteration, pairs used, steps taken, status (0 running, 1 converged, 2 step limit, FIRE_BAD_INPUT,
    FIRE_CELL_DEGENERATE, QN_BREAKDOWN)}, initially zero.  `lbfgs` overrides LBFGS_DEFAULTS."""
    lib = _lib.load()
    par = dict(LBFGS_DEFAULTS, **lbfgs)
    cell_ops = (cells0, logdef, defgrad, cells, cell_forces, stress_out)
    B, A, N, rows, cell = _qn_operands("lbfgs_step", grad, stress, active, batch_offsets, atom_offsets, positions, forces,
                                       cell_ops, (r0, f0, work, work, s_ring, y_ring, history), istate, steps)
    slots = s_ring.numel() // max(3 * rows, 1)
    if (s_ring.numel() != slots * 3 * rows or y_ring.numel() != s_ring.numel() or history.numel() != 2 * slots * B
            or slots < 1):
        raise ValueError("lbfgs_step: inconsistent operand shapes")
    memory = par["memory"]
    _check_int("lbfgs_step", "memory", memory, 1, FIRE_MAX_STEPS)
    p = _lib.LbfgsParams(float(par["maxstep"]), float(par["alpha"]), float(par["damping"]), float(fmax), int(memory),
                         int(slots), int(steps), int(cell), float(force_multiplier), float(stress_wt))
    c0, ld, dg, ce, cf, so = _cell_ptrs(cell, cell_ops)
    _lib.check(lib.alignn_b200_lbfgs_step(C.byref(p), active.data_ptr(), A, atom_offsets.data_ptr(), batch_offsets.data_ptr(),
                                          B, grad.data_ptr(), grad.shape[0], stress.data_ptr() if cell else None,
                                          A if cell else 0, positions.data_ptr(), forces.data_ptr(), c0, ld, dg, ce, cf, so,
                                          r0.data_ptr(), f0.data_ptr(), work.data_ptr(), s_ring.data_ptr(),
                                          y_ring.data_ptr(), history.data_ptr(), istate.data_ptr(), stream_ptr()),
               "alignn_b200_lbfgs_step")


@_on_tensor_device
def bfgs_update(grad: torch.Tensor, stress, active: torch.Tensor, batch_offsets: torch.Tensor, atom_offsets: torch.Tensor,
                positions: torch.Tensor, forces: torch.Tensor, cells0, logdef, defgrad, cells, cell_forces, stress_out,
                h_offsets: torch.Tensor, H: torch.Tensor, r0: torch.Tensor, f0: torch.Tensor, r: torch.Tensor,
                f: torch.Tensor, work: torch.Tensor, istate: torch.Tensor, *, max_dim: int, fmax: float, steps: int,
                force_multiplier: float = 1.0, stress_wt: float = 1.0, **bfgs) -> None:
    """The first half of a BFGS step (ASE 3.22.1 `BFGS.step` up to `update`), in place (csrc/qn_device.cu,
    alignn_b200_bfgs_update): forces, decision, this evaluation's rows r and f, and H's rank-2 update.

    Operands as `lbfgs_step`, plus: h_offsets [B+1] int64 (crystal c's H, [3m, 3m] row-major, at H[h_offsets[c]:]),
    H float64, initially alpha I per crystal; r, f [rows, 3] float64; work [3, rows, 3] float64; istate = {r0 and f0 set,
    update pending, steps taken, status}, initially zero; max_dim >= 3m for every crystal of `active`.  `bfgs`
    overrides BFGS_DEFAULTS."""
    lib = _lib.load()
    par = dict(BFGS_DEFAULTS, **bfgs)
    cell_ops = (cells0, logdef, defgrad, cells, cell_forces, stress_out)
    B, A, N, rows, cell = _qn_operands("bfgs_update", grad, stress, active, batch_offsets, atom_offsets, positions, forces,
                                       cell_ops, (r0, f0, r, f, work, H), istate, steps)
    if work.numel() != 9 * rows or h_offsets.dtype != torch.int64 or h_offsets.numel() != B + 1 or not h_offsets.is_cuda:
        raise ValueError("bfgs_update: inconsistent operand shapes")
    p = _lib.BfgsParams(float(par["maxstep"]), float(par["alpha"]), float(fmax), int(steps), int(cell),
                        float(force_multiplier), float(stress_wt))
    c0, ld, dg, ce, cf, so = _cell_ptrs(cell, cell_ops)
    _lib.check(lib.alignn_b200_bfgs_update(C.byref(p), active.data_ptr(), A, atom_offsets.data_ptr(), batch_offsets.data_ptr(),
                                           B, int(max_dim), grad.data_ptr(), grad.shape[0],
                                           stress.data_ptr() if cell else None, A if cell else 0, positions.data_ptr(),
                                           forces.data_ptr(), c0, ld, dg, ce, cf, so, h_offsets.data_ptr(), H.data_ptr(),
                                           r0.data_ptr(), f0.data_ptr(), r.data_ptr(), f.data_ptr(), work.data_ptr(),
                                           istate.data_ptr(), stream_ptr()), "alignn_b200_bfgs_update")


@_on_tensor_device
def bfgs_apply(group: torch.Tensor, omega: torch.Tensor, eigenvectors: torch.Tensor, atom_offsets: torch.Tensor,
               positions: torch.Tensor, cells0, logdef, defgrad, cells, r0: torch.Tensor, f0: torch.Tensor,
               r: torch.Tensor, f: torch.Tensor, work: torch.Tensor, istate: torch.Tensor, *, cell: bool, **bfgs) -> None:
    """The second half of a BFGS step (csrc/qn_device.cu, alignn_b200_bfgs_apply) for a group of crystals with the same
    3m, after omega, V = torch.linalg.eigh(H) of their blocks (row g: crystal group[g]): dr = V ((f V) / |omega|), the
    longest-row cap, set_positions, r0 = r, f0 = f.  Crystals of the group that are not running are ignored; a
    crystal whose update broke down gets QN_BREAKDOWN.  Operands as `bfgs_update`."""
    lib = _lib.load()
    par = dict(BFGS_DEFAULTS, **bfgs)
    G, dim = group.numel(), int(omega.shape[-1]) if omega.dim() == 2 else 0
    B = atom_offsets.numel() - 1
    rows = r.numel() // 3
    want = [(group, torch.int32), (omega, torch.float64), (eigenvectors, torch.float64), (atom_offsets, torch.int64),
            (positions, torch.float64), (r0, torch.float64), (f0, torch.float64), (r, torch.float64), (f, torch.float64),
            (work, torch.float64), (istate, torch.int32)]
    want += [(t, torch.float64) for t in (cells0, logdef, defgrad, cells)] if cell else []
    _operands("bfgs_apply", want, r.device)
    if (omega.dim() != 2 or omega.shape[0] != G or tuple(eigenvectors.shape) != (G, dim, dim) or work.numel() != 9 * rows
            or any(t.numel() != 3 * rows for t in (r0, f0, f)) or istate.numel() != 4 * B):
        raise ValueError("bfgs_apply: inconsistent operand shapes")
    p = _lib.BfgsParams(float(par["maxstep"]), float(par["alpha"]), 0.0, 1, int(bool(cell)), 1.0, 1.0)
    cp = [t.data_ptr() for t in (cells0, logdef, defgrad, cells)] if cell else [None] * 4
    _lib.check(lib.alignn_b200_bfgs_apply(C.byref(p), group.data_ptr(), G, dim, omega.data_ptr(), eigenvectors.data_ptr(),
                                          atom_offsets.data_ptr(), B, rows, positions.data_ptr(), *cp, r0.data_ptr(),
                                          f0.data_ptr(), r.data_ptr(), f.data_ptr(), work.data_ptr(), istate.data_ptr(),
                                          stream_ptr()), "alignn_b200_bfgs_apply")


MD_NVE, MD_NVT_BERENDSEN = 0, 1   # alignn_b200_md_params.ensemble
MD_BAD_INPUT = 3                  # status of a crystal whose atom slice does not lie inside the batch


@_on_tensor_device
def md_step(grad: torch.Tensor, atom_offsets: torch.Tensor, masses: torch.Tensor,
            target_temperature: Optional[torch.Tensor], positions: torch.Tensor, momenta: torch.Tensor,
            forces: torch.Tensor, kinetic_energy: torch.Tensor, temperature: torch.Tensor, status: torch.Tensor, *,
            evaluation: int, steps: int, dt: float, kB: float, ensemble: int, taut: float = 0.0,
            force_multiplier: float = 1.0) -> None:
    """Evaluation `evaluation` of an MD run of `steps` steps (ASE 3.22.1 `VelocityVerlet` / `NVTBerendsen` with
    `MolecularDynamics.irun`) for every crystal, in place, one launch (csrc/md_device.cu, alignn_b200_md_step): the
    forces, the second half-kick of the previous step (evaluation >= 1), ekin and T of this evaluation, and unless
    evaluation == steps the first half of the next step up to the drift.

    grad [M,3] fp32: the model's forces for all crystals in order; atom_offsets [B+1] int64; masses [N] float64 (amu);
    target_temperature [B] float64 (K; Berendsen only, may be None for NVE); positions / momenta [N,3] float64; forces
    [N,3] fp32 (written); kinetic_energy / temperature [B] float64 (written: this evaluation's log row); status [B] int32
    (0 ok, MD_BAD_INPUT: the crystal's slice does not lie inside grad -- nothing else is read or written for it).
    dt and taut in ASE time units, kB in eV/K.  Enqueue only: the statuses are the caller's to read back."""
    lib = _lib.load()
    want = [(grad, torch.float32), (atom_offsets, torch.int64), (masses, torch.float64), (positions, torch.float64),
            (momenta, torch.float64), (forces, torch.float32), (kinetic_energy, torch.float64),
            (temperature, torch.float64), (status, torch.int32)]
    if target_temperature is not None:
        want.append((target_temperature, torch.float64))
    _operands("md_step", want, grad.device)
    B = atom_offsets.numel() - 1
    N = positions.numel() // 3
    if (B < 1 or positions.numel() != 3 * N or momenta.numel() != 3 * N or forces.numel() != 3 * N
            or masses.numel() != N or kinetic_energy.numel() != B or temperature.numel() != B or status.numel() != B
            or grad.dim() != 2 or grad.shape[1] != 3 or grad.shape[0] > N
            or (target_temperature is not None and target_temperature.numel() != B)):
        raise ValueError("md_step: inconsistent operand shapes")
    if ensemble == MD_NVT_BERENDSEN and target_temperature is None:
        raise ValueError("md_step: NVT Berendsen needs target_temperature")
    _md_counts("md_step", steps, evaluation)
    p = _lib.MdParams(float(dt), float(taut), float(kB), int(evaluation), int(steps), int(ensemble), float(force_multiplier))
    _lib.check(lib.alignn_b200_md_step(C.byref(p), atom_offsets.data_ptr(), B, grad.data_ptr(), grad.shape[0],
                                       masses.data_ptr(),
                                       None if target_temperature is None else target_temperature.data_ptr(),
                                       positions.data_ptr(), momenta.data_ptr(), forces.data_ptr(),
                                       kinetic_energy.data_ptr(), temperature.data_ptr(), status.data_ptr(),
                                       stream_ptr()), "alignn_b200_md_step")


MD_NVT_LANGEVIN, MD_NVT_ANDERSEN = 2, 3   # alignn_b200_md_thermostat_params.ensemble, also the noise stream's tags
MD_ONE_ATOM = 6                           # status of a one-atom crystal under Langevin (ASE divides by n - 1)


@_on_tensor_device
def md_thermostat_step(grad: torch.Tensor, atom_offsets: torch.Tensor, masses: torch.Tensor,
                       target_temperature: torch.Tensor, seeds: torch.Tensor, positions: torch.Tensor,
                       momenta: torch.Tensor, velocities: torch.Tensor, rnd_vel: torch.Tensor, forces: torch.Tensor,
                       kinetic_energy: torch.Tensor, temperature: torch.Tensor, status: torch.Tensor, *,
                       evaluation: int, steps: int, dt: float, kB: float, ensemble: int, friction: float = 0.0,
                       andersen_prob: float = 0.0, force_multiplier: float = 1.0) -> None:
    """Evaluation `evaluation` of an MD run of `steps` steps under ASE 3.22.1's `Langevin` (ensemble=MD_NVT_LANGEVIN)
    or `Andersen` (MD_NVT_ANDERSEN), fixcm=True, for every crystal, in place, one launch (csrc/md_device.cu,
    alignn_b200_md_thermostat_step): the forces, the second half of the previous step (evaluation >= 1), ekin and T of
    this evaluation, and unless evaluation == steps the first half of the next step with the noise of crystal c's seed.

    As `md_step`, plus: target_temperature [B] float64 (K); seeds [B] int64 or uint64 (the 64 bits of each crystal's
    seed); velocities / rnd_vel [N,3] float64, workspaces the launches of one run pass on (not read at evaluation 0);
    status MD_ONE_ATOM for a one-atom crystal under Langevin.  dt in ASE time units, friction in 1 / ASE time unit,
    andersen_prob per component and step.  sqrt(dt), dt ** 1.5 and 2 sqrt(3) are formed here, on the host, as numpy
    forms them.  Enqueue only: the statuses are the caller's to read back."""
    lib = _lib.load()
    _operands("md_thermostat_step",
              [(grad, torch.float32), (atom_offsets, torch.int64), (masses, torch.float64),
               (target_temperature, torch.float64), (seeds, (torch.int64, torch.uint64)), (positions, torch.float64),
               (momenta, torch.float64), (velocities, torch.float64), (rnd_vel, torch.float64),
               (forces, torch.float32), (kinetic_energy, torch.float64), (temperature, torch.float64),
               (status, torch.int32)], grad.device)
    B = atom_offsets.numel() - 1
    N = positions.numel() // 3
    if (B < 1 or positions.numel() != 3 * N or any(t.numel() != 3 * N for t in (momenta, velocities, rnd_vel, forces))
            or masses.numel() != N or any(t.numel() != B for t in (kinetic_energy, temperature, status,
                                                                     target_temperature, seeds))
            or grad.dim() != 2 or grad.shape[1] != 3 or grad.shape[0] > N):
        raise ValueError("md_thermostat_step: inconsistent operand shapes")
    _md_counts("md_thermostat_step", steps, evaluation)
    dt = float(dt)
    ok = math.isfinite(dt) and dt > 0                  # anything else the library rejects
    root_dt = math.sqrt(dt) if ok else float("nan")    # np.sqrt(dt): both correctly rounded
    dt_1_5 = dt ** 1.5 if ok else float("nan")         # Langevin.updatevars' dt**1.5, a Python float power
    p = _lib.MdThermostatParams(dt, float(kB), float(friction), float(andersen_prob), root_dt, dt_1_5,
                                2 * math.sqrt(3), int(evaluation), int(steps), int(ensemble), float(force_multiplier))
    _lib.check(lib.alignn_b200_md_thermostat_step(
        C.byref(p), atom_offsets.data_ptr(), B, grad.data_ptr(), grad.shape[0], masses.data_ptr(),
        target_temperature.data_ptr(), seeds.data_ptr(), positions.data_ptr(), momenta.data_ptr(), velocities.data_ptr(),
        rnd_vel.data_ptr(), forces.data_ptr(), kinetic_energy.data_ptr(), temperature.data_ptr(), status.data_ptr(),
        stream_ptr()), "alignn_b200_md_thermostat_step")


MD_NPT_BERENDSEN = 4              # run_md's code for NPT Berendsen (its own kernel, alignn_b200_md_npt_step)
MD_CELL_DEGENERATE = 4            # status of a crystal whose volume or barostat scale is not finite and > 0


@_on_tensor_device
def md_npt_step(grad: torch.Tensor, stress: torch.Tensor, atom_offsets: torch.Tensor, masses: torch.Tensor,
                target_temperature: torch.Tensor, target_pressure: torch.Tensor, compressibility: torch.Tensor,
                cells: torch.Tensor, positions: torch.Tensor, momenta: torch.Tensor, forces: torch.Tensor,
                stress_out: torch.Tensor, kinetic_energy: torch.Tensor, temperature: torch.Tensor,
                pressure: torch.Tensor, status: torch.Tensor, *, evaluation: int, steps: int, phase: int, dt: float,
                kB: float, taut: float, taup: float, force_multiplier: float = 1.0, stress_wt: float = 1.0) -> None:
    """One launch of an MD run of `steps` steps under ASE 3.22.1's `NPTBerendsen` (fixcm=True) for every crystal, in
    place (csrc/md_device.cu, alignn_b200_md_npt_step).  phase 0, after logged evaluation `evaluation`: the forces, the
    second half-kick (evaluation >= 1), the log rows, and unless evaluation == steps the velocity scaling and the
    barostat's rescaling of cells and positions.  phase 1, after evaluation A of the next step: the half-kick on its
    forces, the mean momentum removed, the drift.

    As `md_step`, plus: stress [B,3,3] fp32, the model's stress (phase 0; not read in phase 1); target_temperature (K),
    target_pressure (eV/A^3) and compressibility (A^3/eV) [B] float64; cells [B,3,3] float64 (rows are lattice vectors,
    scaled in place); stress_out [B,6] fp32 (written: the calculator's Voigt stress) and pressure [B] float64 (written:
    -trace/3 of that stress less the ideal-gas term, eV/A^3), the log rows of this evaluation; status
    MD_CELL_DEGENERATE for a cell whose volume or barostat scale is not finite and > 0 (nothing of the crystal is
    written).  dt, taut and taup in ASE time units.  Enqueue only: the statuses are the caller's to read back."""
    lib = _lib.load()
    _operands("md_npt_step",
              [(grad, torch.float32), (stress, torch.float32), (atom_offsets, torch.int64), (masses, torch.float64),
               (target_temperature, torch.float64), (target_pressure, torch.float64),
               (compressibility, torch.float64), (cells, torch.float64), (positions, torch.float64),
               (momenta, torch.float64), (forces, torch.float32), (stress_out, torch.float32),
               (kinetic_energy, torch.float64), (temperature, torch.float64), (pressure, torch.float64),
               (status, torch.int32)], grad.device)
    B = atom_offsets.numel() - 1
    N = positions.numel() // 3
    if (B < 1 or positions.numel() != 3 * N or momenta.numel() != 3 * N or forces.numel() != 3 * N
            or masses.numel() != N or stress.numel() != 9 * B or cells.numel() != 9 * B or stress_out.numel() != 6 * B
            or any(t.numel() != B for t in (target_temperature, target_pressure, compressibility, kinetic_energy,
                                             temperature, pressure, status))
            or grad.dim() != 2 or grad.shape[1] != 3 or grad.shape[0] > N):
        raise ValueError("md_npt_step: inconsistent operand shapes")
    _md_counts("md_npt_step", steps, evaluation)
    p = _lib.MdNptParams(float(dt), float(taut), float(taup), float(kB), int(evaluation), int(steps), int(phase),
                         float(force_multiplier), float(stress_wt))
    _lib.check(lib.alignn_b200_md_npt_step(
        C.byref(p), atom_offsets.data_ptr(), B, grad.data_ptr(), grad.shape[0], stress.data_ptr(), masses.data_ptr(),
        target_temperature.data_ptr(), target_pressure.data_ptr(), compressibility.data_ptr(), cells.data_ptr(),
        positions.data_ptr(), momenta.data_ptr(), forces.data_ptr(), stress_out.data_ptr(), kinetic_energy.data_ptr(),
        temperature.data_ptr(), pressure.data_ptr(), status.data_ptr(), stream_ptr()), "alignn_b200_md_npt_step")


MD_NPT_NOSE_HOOVER = 5            # run_md's code for ASE's NPT (its own kernel, alignn_b200_md_nose_hoover_step)
MD_NH_STATE = 29                  # ALIGNN_B200_MD_NH_STATE: h_past, eta, eta_past (3 x 3 each), zeta, zeta_past


@_on_tensor_device
def md_nose_hoover_step(grad: torch.Tensor, stress: torch.Tensor, atom_offsets: torch.Tensor, masses: torch.Tensor,
                        tfact: torch.Tensor, pfact: torch.Tensor, desired_ekin: torch.Tensor,
                        external_stress: torch.Tensor, cells: torch.Tensor, state: torch.Tensor,
                        positions: torch.Tensor, momenta: torch.Tensor, q: torch.Tensor, q_future: torch.Tensor,
                        forces: torch.Tensor, stress_out: torch.Tensor, kinetic_energy: torch.Tensor,
                        temperature: torch.Tensor, pressure: torch.Tensor, status: torch.Tensor, *, evaluation: int,
                        steps: int, dt: float, kB: float, force_multiplier: float = 1.0, stress_wt: float = 1.0) -> None:
    """Evaluation `evaluation` of an MD run of `steps` steps under ASE 3.22.1's `NPT` (Nose-Hoover thermostat and
    Parrinello-Rahman barostat) for every crystal, in place, one launch (csrc/md_device.cu,
    alignn_b200_md_nose_hoover_step): evaluation 0 initialises (centre-of-mass momentum removed, q from the positions,
    q_future by ASE's two passes), a later one finishes its step (q_future and the momenta from its forces); then the
    log rows, and unless evaluation == steps the start of the next step (cell, eta, zeta, the shift of q, the positions
    of the next evaluation).

    As `md_npt_step`, plus: tfact, pfact, desired_ekin [B] and external_stress [B,6] float64, the constants of ASE's
    `NPT._calculateconstants` / `set_stress` (pfact 0 means no barostat; the stress then drives nothing); cells [B,3,3]
    float64, upper triangular, advanced in place; state [B, MD_NH_STATE] float64 (zeroed before evaluation 0); q and
    q_future [N,3] float64 workspaces the kernel owns between launches.  Status MD_BAD_INPUT also for a cell that is
    not upper triangular at evaluation 0, MD_CELL_DEGENERATE for a singular or non-finite h, beta + I or next cell.
    dt in ASE time units.  Enqueue only: the statuses are the caller's to read back."""
    lib = _lib.load()
    f64 = torch.float64
    _operands("md_nose_hoover_step",
              [(grad, torch.float32), (stress, torch.float32), (atom_offsets, torch.int64), (masses, f64),
               (tfact, f64), (pfact, f64), (desired_ekin, f64), (external_stress, f64), (cells, f64), (state, f64),
               (positions, f64), (momenta, f64), (q, f64), (q_future, f64), (forces, torch.float32),
               (stress_out, torch.float32), (kinetic_energy, f64), (temperature, f64), (pressure, f64),
               (status, torch.int32)], grad.device)
    B = atom_offsets.numel() - 1
    N = positions.numel() // 3
    if (B < 1 or positions.numel() != 3 * N or any(t.numel() != 3 * N for t in (momenta, q, q_future, forces))
            or masses.numel() != N or stress.numel() != 9 * B or cells.numel() != 9 * B or stress_out.numel() != 6 * B
            or external_stress.numel() != 6 * B or state.numel() != MD_NH_STATE * B
            or any(t.numel() != B for t in (tfact, pfact, desired_ekin, kinetic_energy, temperature, pressure, status))
            or grad.dim() != 2 or grad.shape[1] != 3 or grad.shape[0] > N):
        raise ValueError("md_nose_hoover_step: inconsistent operand shapes")
    _md_counts("md_nose_hoover_step", steps, evaluation)
    p = _lib.MdNoseHooverParams(float(dt), float(kB), int(evaluation), int(steps), float(force_multiplier),
                                float(stress_wt))
    _lib.check(lib.alignn_b200_md_nose_hoover_step(
        C.byref(p), atom_offsets.data_ptr(), B, grad.data_ptr(), grad.shape[0], stress.data_ptr(), masses.data_ptr(),
        tfact.data_ptr(), pfact.data_ptr(), desired_ekin.data_ptr(), external_stress.data_ptr(), cells.data_ptr(),
        state.data_ptr(), positions.data_ptr(), momenta.data_ptr(), q.data_ptr(), q_future.data_ptr(),
        forces.data_ptr(), stress_out.data_ptr(), kinetic_energy.data_ptr(), temperature.data_ptr(),
        pressure.data_ptr(), status.data_ptr(), stream_ptr()), "alignn_b200_md_nose_hoover_step")


def md_noise(seed: int, step: int, count: int, *, tag: int = MD_NVT_LANGEVIN, atom0: int = 0, blocks: int = 1,
             device=None):
    """The thermostats' noise stream (csrc/md_noise.cuh) on the device, for tests: Philox block j of atom index
    atom0 + a (mod 2^32), a in [0, count), j in [0, blocks), at (seed, step, tag).  Returns (words [count, blocks, 4]
    int64 holding the uint32 words, uniforms [count, blocks, 2] float64, normals [count, blocks, 2] float64)."""
    lib = _lib.load()
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError(f"md_noise needs a CUDA device, got {dev}")
    if not 0 <= int(seed) < 2 ** 64 or not 0 <= int(atom0) < 2 ** 32:
        raise ValueError("md_noise: seed must be in [0, 2^64) and atom0 in [0, 2^32)")
    count, blocks = int(count), int(blocks)
    words = torch.empty(count, blocks, 4, dtype=torch.int32, device=dev)
    uniforms = torch.empty(count, blocks, 2, dtype=torch.float64, device=dev)
    normals = torch.empty(count, blocks, 2, dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.alignn_b200_md_noise(int(seed), int(step), int(tag), int(atom0), count, blocks, words.data_ptr(),
                                            uniforms.data_ptr(), normals.data_ptr(), stream_ptr()),
                   "alignn_b200_md_noise")
    return words.to(torch.int64) & 0xFFFFFFFF, uniforms, normals


PHONON_BAD_INPUT = 3              # status of a crystal whose slices do not lie inside the buffers
PHONON_NON_FINITE = 5             # status of a crystal with a non-finite force product
PHONON_MAX_CELLS = 3072           # ALIGNN_B200_PHONON_MAX_CELLS: cells of one supercell


def _supercell_arg(supercell):
    if supercell is None:
        return None
    s = tuple(int(v) for v in supercell)
    if len(s) != 3:
        raise ValueError(f"supercell must have 3 entries, got {supercell!r}")
    return C.cast((C.c_int32 * 3)(*s), C.c_void_p)


@_on_tensor_device
def phonon_force_constants(grad: torch.Tensor, atom_offsets: torch.Tensor, row_offsets: torch.Tensor,
                           fc_offsets: torch.Tensor, masses: torch.Tensor, force_constants: torch.Tensor,
                           dynamical_matrix: torch.Tensor, status: torch.Tensor, *, supercell, delta: float,
                           force_multiplier: float = 1.0) -> None:
    """ASE 3.22.1's `Phonons.read(acoustic=True)` for every crystal of a batch, one launch (csrc/phonon_device.cu,
    alignn_b200_phonon_force_constants): Frederiksen-corrected central differences, three rounds of symmetrize and
    acoustic, mass weighting.

    grad [rows,3] fp32: the model's forces of every displaced supercell (crystal c's 6n supercells of Nc n rows from
    row_offsets[c], displacement order atom, direction, sign -1 then +1); atom_offsets / row_offsets / fc_offsets [B+1]
    int64; masses [sum n] float64 (amu); force_constants / dynamical_matrix [fc_offsets[B]] float64 (written: crystal
    c's [Nc, 3n, 3n] C_N and D_N at fc_offsets[c]); status [B] int32 (0 ok, PHONON_BAD_INPUT: a slice is not inside its
    buffer, PHONON_NON_FINITE: a force product is not finite -- nothing else is read or written for it).  supercell is
    (N0, N1, N2); delta in A.  Enqueue only: the statuses are the caller's to read back."""
    lib = _lib.load()
    _operands("phonon_force_constants", [(grad, torch.float32), (atom_offsets, torch.int64),
                                         (row_offsets, torch.int64), (fc_offsets, torch.int64),
                                         (masses, torch.float64), (force_constants, torch.float64),
                                         (dynamical_matrix, torch.float64), (status, torch.int32)], grad.device)
    B = atom_offsets.numel() - 1
    if (B < 1 or row_offsets.numel() != B + 1 or fc_offsets.numel() != B + 1 or status.numel() != B
            or grad.dim() != 2 or grad.shape[1] != 3 or dynamical_matrix.numel() != force_constants.numel()):
        raise ValueError("phonon_force_constants: inconsistent operand shapes")
    _lib.check(lib.alignn_b200_phonon_force_constants(
        _supercell_arg(supercell), float(delta), float(force_multiplier), atom_offsets.data_ptr(), B,
        row_offsets.data_ptr(), grad.data_ptr(), grad.shape[0], masses.data_ptr(), fc_offsets.data_ptr(),
        force_constants.numel(), force_constants.data_ptr(), dynamical_matrix.data_ptr(), status.data_ptr(),
        stream_ptr()), "alignn_b200_phonon_force_constants")


@_on_tensor_device
def phonon_dynamical_matrix(dynamical_matrix: torch.Tensor, fc_offsets: torch.Tensor, crystals: torch.Tensor,
                            qpoints: torch.Tensor, out: torch.Tensor, status: torch.Tensor, *, supercell,
                            modes: int) -> None:
    """D(q) = sum_R exp(-2 pi i q.R) D_N[R] (ASE 3.22.1 `Phonons.band_structure`'s Fourier sum) for a block of
    (crystal, q) pairs whose crystals all have `modes` modes, one launch (alignn_b200_phonon_dynamical_matrix).

    dynamical_matrix [fc_offsets[B]] float64 (the D_N of `phonon_force_constants`); fc_offsets [B+1] int64; crystals
    [Q] int32; qpoints [Q,3] float64 (fractional); out [Q, modes, modes] complex128 (written: Hermitian, both
    triangles); status [B] int32 (PHONON_BAD_INPUT: crystal c's D_N slice is not [Nc, modes, modes] inside the buffer;
    its pairs are not written).  Enqueue only."""
    lib = _lib.load()
    _operands("phonon_dynamical_matrix", [(dynamical_matrix, torch.float64), (fc_offsets, torch.int64),
                                          (crystals, torch.int32), (qpoints, torch.float64),
                                          (out, torch.complex128), (status, torch.int32)], dynamical_matrix.device)
    B, Q = fc_offsets.numel() - 1, crystals.numel()
    if B < 1 or status.numel() != B or qpoints.numel() != 3 * Q or out.numel() != Q * int(modes) * int(modes):
        raise ValueError("phonon_dynamical_matrix: inconsistent operand shapes")
    _lib.check(lib.alignn_b200_phonon_dynamical_matrix(
        _supercell_arg(supercell), int(modes), dynamical_matrix.data_ptr(), fc_offsets.data_ptr(), B,
        dynamical_matrix.numel(), crystals.data_ptr(), qpoints.data_ptr(), Q, out.data_ptr(), status.data_ptr(),
        stream_ptr()), "alignn_b200_phonon_dynamical_matrix")


EOS_FORMS = {"murnaghan": 0, "birchmurnaghan": 1, "vinet": 2}    # ALIGNN_B200_EOS_*
EOS_OK, EOS_OUTSIDE, EOS_NO_FIT, EOS_BAD_INPUT = 0, 1, 2, 3       # per-row statuses of eos_fit
EOS_MAX_POINTS = 65536            # ALIGNN_B200_EOS_MAX_POINTS


@_on_tensor_device
def eos_fit(volumes: torch.Tensor, energies: torch.Tensor, params: torch.Tensor, status: torch.Tensor, *,
            form: int) -> None:
    """ASE 3.22.1's `EquationOfState(v, e, eos).fit()` for every row, one launch (csrc/eos_device.cu,
    alignn_b200_eos_fit): the parabola seed, then Levenberg-Marquardt to the least-squares optimum.

    volumes / energies [R, S] float64 (A^3, eV), S >= 4; params [R, 4] float64 (written: E0, B0 in eV/A^3, BP, V0);
    status [R] int32 (written: EOS_OK, EOS_OUTSIDE -- V0 not strictly inside the volumes, parameters kept --,
    EOS_NO_FIT or EOS_BAD_INPUT -- NaN parameters).  form is one of EOS_FORMS' values.  Enqueue only: the statuses are
    the caller's to read back."""
    lib = _lib.load()
    _operands("eos_fit", [(volumes, torch.float64), (energies, torch.float64), (params, torch.float64),
                          (status, torch.int32)], volumes.device)
    if (volumes.dim() != 2 or energies.shape != volumes.shape or params.shape != (volumes.shape[0], 4)
            or status.shape != (volumes.shape[0],)):
        raise ValueError("eos_fit: inconsistent operand shapes")
    if form not in EOS_FORMS.values() or not 4 <= volumes.shape[1] <= EOS_MAX_POINTS:
        raise ValueError(f"eos_fit: form must be one of {sorted(EOS_FORMS.values())} and the rows must have 4 to "
                         f"{EOS_MAX_POINTS} points, got form={form!r}, {volumes.shape[1]} points")
    _lib.check(lib.alignn_b200_eos_fit(int(form), volumes.data_ptr(), energies.data_ptr(), volumes.shape[0],
                                       volumes.shape[1], params.data_ptr(), status.data_ptr(), stream_ptr()),
               "alignn_b200_eos_fit")


class _SegmentMean(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gptr):
        lib = _lib.load()
        require_cuda(x, gptr)
        B, d = gptr.numel() - 1, x.shape[1]
        out = torch.empty(B, d, device=x.device, dtype=torch.float32)
        _lib.check(lib.alignn_b200_segment_mean(ptr(x), ptr(gptr), B, d, ptr(out), stream_ptr()), "alignn_b200_segment_mean")
        ctx.save_for_backward(gptr)
        ctx.n = x.shape[0]
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_out):
        lib = _lib.load()
        (gptr,) = ctx.saved_tensors
        g_out = g_out.contiguous()
        B, d = g_out.shape
        gx = torch.empty(ctx.n, d, device=g_out.device, dtype=torch.float32)
        _lib.check(lib.alignn_b200_segment_mean_backward(ptr(g_out), ptr(gptr), B, d, ptr(gx), stream_ptr()),
                   "alignn_b200_segment_mean_backward")
        return gx, None


@_on_tensor_device
def segment_mean(x: torch.Tensor, graph_ptr: torch.Tensor) -> torch.Tensor:
    """Per-graph mean over node rows (dgl.nn.AvgPooling, alignn.py:325)."""
    return _SegmentMean.apply(x.contiguous(), graph_ptr)


def segment_mean_any_order(x: torch.Tensor, graph_ptr: torch.Tensor, second_order: bool) -> torch.Tensor:
    """`segment_mean`, or (force training, which differentiates through the backward) the same pooling from torch operators."""
    if not second_order:
        return segment_mean(x, graph_ptr)
    counts = (graph_ptr[1:] - graph_ptr[:-1]).long()
    gid = torch.repeat_interleave(torch.arange(counts.numel(), device=x.device), counts, output_size=x.shape[0])
    sums = torch.zeros(counts.numel(), x.shape[1], device=x.device, dtype=x.dtype).index_add(0, gid, x)
    return sums / counts.clamp_min(1).to(x.dtype).unsqueeze(1)


# ---- tensor-core Linear (wgmma, bf16x3) ----------------------------------------------------------
class WeightImage:
    """bf16 hi/lo image of a weight matrix W[N,K] (or of W^T when transpose=True) in UMMA core-matrix
    order; valid until the weight changes (rebuilt every step in training)."""

    __slots__ = ("buf", "N", "K")

    def __init__(self, W: torch.Tensor, transpose: bool = False):
        require_cuda(W)
        if W.dim() != 2:
            raise RuntimeError("WeightImage needs a 2-D weight")
        self.N, self.K = (W.shape[1], W.shape[0]) if transpose else (W.shape[0], W.shape[1])
        tbl = ImageTable()
        tbl.add_image("w", self.N, self.K, [(W, transpose, 0, 0)], W.device)
        tbl.refresh()
        self.buf = tbl.images["w"].buf


class _Img:
    """An operand image owned by an ImageTable (same attributes as WeightImage)."""
    __slots__ = ("buf", "N", "K")

    def __init__(self, N: int, K: int, device):
        nbytes = int(_lib.load().alignn_b200_gemm_weight_image_bytes(N, K))
        if nbytes == 0:
            raise RuntimeError(f"alignn_b200 GEMM: unsupported weight shape N={N}, K={K} (need multiples of 32)")
        self.N, self.K = N, K
        self.buf = torch.zeros(nbytes, device=device, dtype=torch.uint8)     # zero: K padding stays zero forever


class ImageTable:
    """bf16 hi/lo operand images (and stacked / folded bias vectors) of a group of Linear layers, rebuilt by ONE
    table-driven launch (`alignn_b200_gemm_prepare_table`) when -- and only when -- a source tensor changed
    (storage pointer or autograd version).  Tables register their blocks once; a parent table (the model) absorbs
    the tables of its layers so that a training step refreshes every image of the model in a single launch.

    Inside a CUDA-graph capture the refresh of a table with trainable sources is always recorded: a captured training
    step must rebuild its images on every replay, whatever the version counters said at capture time."""

    def __init__(self, device=None):
        self.device = device
        self.images = {}
        self.vectors = {}
        self._blocks = []      # (image name, source tensor, transpose, n_off, k_off)
        self._biases = []      # (vector name, offset, n, a, b)
        self._children = []
        self._parent = None
        self._key = None
        self._dev = None       # (entries tensor, n_entries, max_units, bias tensor, n_bias, pointer key)

    # -- construction ---------------------------------------------------------------------------
    def add_image(self, name: str, N: int, K: int, blocks, device):
        """blocks: [(W, transpose, n_off, k_off)]; W is a 2-D fp32 tensor (a Linear weight)."""
        self.images[name] = _Img(N, K, device)
        for W, tr, n_off, k_off in blocks:
            if k_off % 8:
                raise RuntimeError("ImageTable: k_off must be a multiple of 8")
            self._blocks.append((name, W, bool(tr), int(n_off), int(k_off)))
        self._key = self._dev = None

    def add_vector(self, name: str, n: int, parts, device):
        """parts: [(offset, a, b_or_None)]: vector[offset : offset + len(a)] = a (+ b)."""
        self.vectors[name] = torch.zeros(n, device=device, dtype=torch.float32)
        for off, a, b in parts:
            self._biases.append((name, int(off), int(a.numel()), a, b))
        self._key = self._dev = None

    def absorb(self, child: "ImageTable"):
        self._children.append(child)
        child._parent = weakref.ref(self)
        self._key = self._dev = None

    # -- refresh ----------------------------------------------------------------------------------
    def _all(self):
        out = [self]
        for c in self._children:
            out.extend(c._all())
        return out

    def _sources(self):
        for t in self._all():
            for _, W, _, _, _ in t._blocks:
                yield W
            for _, _, _, a, b in t._biases:
                yield a
                if b is not None:
                    yield b

    def _build_device_table(self):
        ents, bias = [], []
        max_units = 1
        for t in self._all():
            for name, W, tr, n_off, k_off in t._blocks:
                if W.dim() != 2 or W.stride(1) != 1 or not W.is_cuda or W.dtype != torch.float32:
                    raise RuntimeError("ImageTable: sources must be 2-D fp32 CUDA tensors with unit column stride")
                img = t.images[name]
                rows, cols = W.shape
                n_img, k_img = (cols, rows) if tr else (rows, cols)
                if n_off + n_img > img.N or k_off + (k_img + 7) // 8 * 8 > img.K:
                    raise RuntimeError(f"ImageTable: block does not fit image {name}")
                ents.append(_lib.ImageEntry(W=W.data_ptr(), ldw=W.stride(0), rows=rows, cols=cols, transpose=int(tr), n_off=n_off,
                                            k_off=k_off, N=img.N, K=img.K, image=img.buf.data_ptr()))
                max_units = max(max_units, n_img * ((k_img + 7) // 8))
            for name, off, n, a, b in t._biases:
                dst = t.vectors[name]
                bias.append(_lib.BiasEntry(a=a.data_ptr(), b=None if b is None else b.data_ptr(),
                                           dst=dst.data_ptr() + 4 * off, n=n))
        dev = next(self._sources()).device

        def pack(items, cls):
            if not items:
                return None
            arr = (cls * len(items))(*items)
            host = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).pin_memory()
            self._host_keepalive.append(host)       # a captured copy reads this buffer again on every replay
            return host.to(dev, non_blocking=True)
        self._host_keepalive = []
        self._dev = (pack(ents, _lib.ImageEntry), len(ents), max_units, pack(bias, _lib.BiasEntry), len(bias),
                     tuple(s.data_ptr() for s in self._sources()))

    def refresh(self):
        """Rebuild the images if any source changed.  Returns True if a launch was issued."""
        srcs = list(self._sources())
        if not srcs:
            return False
        key = tuple((s.data_ptr(), s._version) for s in srcs)
        capturing = torch.cuda.is_current_stream_capturing() and any(s.requires_grad for s in srcs)
        if capturing and self._parent is not None and self._parent() is not None:
            capturing = False                       # the model-level table records the refresh of all its layers
        if key == self._key and not capturing:
            return False
        ptr_key = tuple(k[0] for k in key)
        if self._dev is None or self._dev[5] != ptr_key:
            self._build_device_table()
        ents, n_e, max_units, bias, n_b, _ = self._dev
        with torch.cuda.device(srcs[0].device):
            _lib.check(_lib.load().alignn_b200_gemm_prepare_table(ptr_any(ents), n_e, max_units, ptr_any(bias), n_b, stream_ptr()),
                       "alignn_b200_gemm_prepare_table")
        for t in self._all():
            t._key = tuple((s.data_ptr(), s._version) for s in t._sources())
        return True


def ptr_any(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


@_on_tensor_device
def gemm_nt(A: torch.Tensor, w: WeightImage, bias: Optional[torch.Tensor] = None,
            residual: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[M,N] = A[M,K] @ W^T (+ bias) (+ residual) on wgmma.  A may be a column slice (row stride >= K)."""
    lib = _lib.load()
    if A.dim() != 2 or A.stride(1) != 1 or A.shape[1] != w.K:
        raise RuntimeError(f"gemm_nt: A must be [M,{w.K}] with unit column stride, got {tuple(A.shape)}/{A.stride()}")
    for t in (A, bias, residual, out):
        if t is not None and (not t.is_cuda or t.dtype != torch.float32):
            raise RuntimeError("gemm_nt needs fp32 CUDA tensors")
    M = A.shape[0]
    if out is None:
        out = torch.empty(M, w.N, device=A.device, dtype=torch.float32)
    ldr = residual.stride(0) if residual is not None else 0
    if residual is not None and (residual.stride(1) != 1 or residual.shape != (M, w.N)):
        raise RuntimeError("gemm_nt: bad residual layout")
    with _span(f"gemm_nt<{min(w.N, 256)}>", 4 * M * (w.K + w.N * (1 + (residual is not None)))):
        _lib.check(lib.alignn_b200_gemm_nt(ptr_any(A), A.stride(0), ptr_any(w.buf), M, w.N, w.K, ptr_any(bias), ptr_any(residual),
                                            ldr, ptr_any(out), out.stride(0), stream_ptr()), "alignn_b200_gemm_nt")
    return out


@_on_tensor_device
def gemm_gather(A: torch.Tensor, w: WeightImage, bias: Optional[torch.Tensor] = None, *,
                add0: Optional[torch.Tensor] = None, idx0: Optional[torch.Tensor] = None,
                add1: Optional[torch.Tensor] = None, idx1: Optional[torch.Tensor] = None,
                stats: bool = False, out: Optional[torch.Tensor] = None, bn_bwd=None):
    """out[r] = A[r] @ W^T (+ bias) (+ add0[idx0[r]]) (+ add1[idx1[r]]) on wgmma.

    add0 / add1 are 2-D fp32 views with unit column stride and w.N columns (column slices of a wider matrix are fine);
    idx None = identity (a residual).  stats=True also returns the per-CTA partial column sums [rows, 2, N] of out and
    out^2 (alignn.py:123 batch statistics; feed `bn_finalize(partials, 0, M, ...)`).

    bn_bwd=(R, scale, shift, mean, rstd): out is the incoming gradient of a train-mode BatchNorm1d + SiLU with input
    R [M, N]; also returns partials [rows, 2, N] of sum gu and sum gu * xhat, gu = out * silu'(R * scale + shift),
    xhat = (R - mean) * rstd, i.e. what bn_backward_reduce reduces (c1, c2 = colsum(partials.view(rows, 2 * N), 1 / M)).
    out itself is bitwise what the call without bn_bwd writes.  Needs add1 = None and no stats request."""
    lib = _lib.load()
    if A.dim() != 2 or A.stride(1) != 1 or A.shape[1] != w.K:
        raise RuntimeError(f"gemm_gather: A must be [M,{w.K}] with unit column stride, got {tuple(A.shape)}/{A.stride()}")
    M = A.shape[0]
    for t in (A, bias, add0, add1, out):
        if t is not None and (not t.is_cuda or t.dtype != torch.float32):
            raise RuntimeError("gemm_gather needs fp32 CUDA tensors")
    for t, ix in ((add0, idx0), (add1, idx1)):
        if t is None:
            if ix is not None:
                raise RuntimeError("gemm_gather: index without addend")
            continue
        if t.dim() != 2 or t.stride(1) != 1 or t.shape[1] != w.N:
            raise RuntimeError("gemm_gather: addend must be [rows, N] with unit column stride")
        if ix is None and t.shape[0] != M:
            raise RuntimeError("gemm_gather: identity-indexed addend must have M rows")
        if ix is not None and (ix.dtype != torch.int32 or not ix.is_cuda or not ix.is_contiguous() or ix.numel() != M):
            raise RuntimeError("gemm_gather: index must be a contiguous int32 CUDA tensor with M entries")
    bn = (None,) * 5
    if bn_bwd is not None:
        if stats or add1 is not None:
            raise RuntimeError("gemm_gather: bn_bwd excludes stats and add1")
        bn = tuple(bn_bwd)
        R = bn[0]
        require_cuda(*bn[1:])
        if R.dim() != 2 or R.shape != (M, w.N) or R.stride(1) != 1 or not R.is_cuda or R.dtype != torch.float32 \
                or any(v.numel() != w.N for v in bn[1:]):
            raise RuntimeError("gemm_gather: bn_bwd needs R [M, N] with unit column stride and [N] vectors")
    if out is None:
        out = torch.empty(M, w.N, device=A.device, dtype=torch.float32)
    part = None
    if stats or bn_bwd is not None:
        rows = int(lib.alignn_b200_gemm_gather_stat_rows(M, w.N))
        part = torch.empty(max(rows, 1), 2, w.N, device=A.device, dtype=torch.float32)
    a = _lib.GemmGatherArgs(
        struct_size=C.sizeof(_lib.GemmGatherArgs), M=M, N=w.N, K=w.K, A=ptr_any(A), lda=A.stride(0),
        w_image=ptr_any(w.buf), bias=ptr_any(bias),
        add0=ptr_any(add0), ld0=add0.stride(0) if add0 is not None else 0, idx0=ptr_any(idx0),
        add1=ptr_any(add1), ld1=add1.stride(0) if add1 is not None else 0, idx1=ptr_any(idx1),
        C=ptr_any(out), ldc=out.stride(0), stats=ptr_any(part), stream=stream_ptr(),
        bn_R=ptr_any(bn[0]), ld_bn_R=bn[0].stride(0) if bn[0] is not None else 0,
        bn_scale=ptr_any(bn[1]), bn_shift=ptr_any(bn[2]), bn_mean=ptr_any(bn[3]), bn_rstd=ptr_any(bn[4]))
    nb = 4 * M * (w.K + w.N) + (8 * M if idx0 is not None else 0) + (4 * M * w.N if (add0 is not None and idx0 is None) else 0)
    nb += 4 * M * w.N if bn_bwd is not None else 0
    kind = "+gather" if idx0 is not None else ("+residual" if add0 is not None else "")
    kind += "+stats" if stats else ("+bn_bwd" if bn_bwd is not None else "")
    with _span(f"gemm_gather<{min(w.N, 256)}>" + kind, nb):
        _lib.check(lib.alignn_b200_gemm_gather(C.byref(a)), "alignn_b200_gemm_gather")
    return (out, part) if (stats or bn_bwd is not None) else out


def wgrad_supported(DA: int, DB: int) -> bool:
    return int(_lib.load().alignn_b200_wgrad_workspace_bytes(32, DA, DB, 1)) > 0


@_on_tensor_device
def wgrad(A: torch.Tensor, B: torch.Tensor, groups: int = 1) -> torch.Tensor:
    """out[g*DA + o, i] = sum_r A[r, g*DA + o] * B[r, i]  (dL/dW of a Linear: A = output grads, B = inputs)."""
    lib = _lib.load()
    require_cuda(A, B)
    K, DB = B.shape
    if A.dim() != 2 or A.shape[0] != K or A.shape[1] % groups:
        raise RuntimeError(f"wgrad: A must be [{K}, groups*DA], got {tuple(A.shape)}")
    DA = A.shape[1] // groups
    nbytes = int(lib.alignn_b200_wgrad_workspace_bytes(K, DA, DB, groups))
    if nbytes == 0 and K >= 0:
        raise RuntimeError(f"alignn_b200 wgrad: unsupported shape DA={DA}, DB={DB}")
    out = torch.empty(groups * DA, DB, device=A.device, dtype=torch.float32)
    ws = torch.empty(max(nbytes, 16), device=A.device, dtype=torch.uint8)
    with _span(f"wgrad<{DA},{DB}>", 4 * K * (groups * DA + DB)):
        _lib.check(lib.alignn_b200_wgrad(ptr(A), A.stride(0), ptr(B), B.stride(0), K, DA, DB, groups, ptr(out), DB, ptr_any(ws),
                                          nbytes, stream_ptr()), "alignn_b200_wgrad")
    return out


WGRAD_BATCH_MAX = 64      # problems per launch (kMaxProblems in csrc/wgrad_tc.cu)


@_on_tensor_device
def wgrad_batch(problems) -> None:
    """ONE launch for many square weight gradients: `problems` is a list of (A [K, >= d] view, B [K, >= d] view, out [d, d]
    view); out[o, i] = sum_r A[r, o] * B[r, i].  Views may be column slices of wider matrices (row stride = stride(0))."""
    lib = _lib.load()
    if not problems:
        return
    d = problems[0][2].shape[0]
    for i0 in range(0, len(problems), WGRAD_BATCH_MAX):
        chunk = problems[i0:i0 + WGRAD_BATCH_MAX]
        arr = (_lib.WgradProblem * len(chunk))()
        nbytes_in = 0
        for q, (A, B, out) in zip(arr, chunk):
            if not (A.is_cuda and B.is_cuda and out.is_cuda and A.dtype == B.dtype == out.dtype == torch.float32):
                raise RuntimeError("alignn_b200 kernels need fp32 CUDA tensors")
            if out.shape != (d, d) or A.shape[1] != d or B.shape[1] != d or A.shape[0] != B.shape[0] or A.stride(1) != 1 \
                    or B.stride(1) != 1 or out.stride(1) != 1:
                raise RuntimeError("wgrad_batch: every problem is A [K, d], B [K, d] -> out [d, d] with unit column stride")
            q.A, q.lda, q.B, q.ldb, q.K = ptr(A), A.stride(0), ptr(B), B.stride(0), A.shape[0]
            q.out, q.ld_out = ptr(out), out.stride(0)
            nbytes_in += 8 * A.shape[0] * d
        nbytes = int(lib.alignn_b200_wgrad_batch_workspace_bytes(arr, len(chunk), d))
        if nbytes == 0:
            raise RuntimeError(f"alignn_b200 wgrad_batch: unsupported batch (d={d}, n={len(chunk)})")
        # the non-cooperative fallback runs problem by problem and needs the single-problem workspace
        nbytes = max(nbytes, max(int(lib.alignn_b200_wgrad_workspace_bytes(A.shape[0], d, d, 1)) for A, _, _ in chunk))
        ws = torch.empty(nbytes, device=chunk[0][0].device, dtype=torch.uint8)
        with _span(f"wgrad_batch<{d}>", nbytes_in):
            _lib.check(lib.alignn_b200_wgrad_batch(arr, len(chunk), d, ptr_any(ws), nbytes, stream_ptr()), "alignn_b200_wgrad_batch")


class WgradQueue:
    """Deferred weight gradients.  While a queue is installed (`WgradQueue.current`), the conv Functions do not launch their
    weight-gradient GEMMs during backward; they register (A, B, destination) here and return None for those weights, and
    `flush()` computes all of them with one `wgrad_batch` launch, writing straight into the destinations -- slices of
    the flat gradient buffer of `alignn_b200.dp.FlatGradAllReducer`, which installs the queue.  A weight is only deferred
    if the queue knows a destination for it (`dest`: parameter data_ptr -> [d, d] view) and it has not been queued already
    in this backward (a layer applied twice falls back to the immediate path and autograd's accumulation)."""
    current: Optional["WgradQueue"] = None

    def __init__(self):
        self.dest = {}            # weight.data_ptr() -> destination view [d, d]
        self.vec_dest = {}        # bias / norm parameter data_ptr() -> destination view [d]
        self.items = []           # (A, B, out)
        self.vec_items = []       # (partial rows [rows, n*d], column offset, d, out)
        self._seen = set()

    def wants(self, *weights) -> bool:
        keys = [w.data_ptr() for w in weights]
        return all(k in self.dest and k not in self._seen for k in keys) and len(set(keys)) == len(keys)

    def wants_vecs(self, *params) -> bool:
        keys = [p.data_ptr() for p in params]
        return all(k in self.vec_dest and k not in self._seen for k in keys) and len(set(keys)) == len(keys)

    def add(self, A: torch.Tensor, B: torch.Tensor, weight: torch.Tensor) -> None:
        k = weight.data_ptr()
        self._seen.add(k)
        self.items.append((A, B, self.dest[k]))

    def add_vec(self, partials: torch.Tensor, block: int, d: int, param: torch.Tensor) -> None:
        """param.grad = column sums of partials[:, block*d:(block+1)*d] (per-block partial rows of egc_backward)."""
        k = param.data_ptr()
        self._seen.add(k)
        self.vec_items.append((partials, block * d, d, self.vec_dest[k]))

    def deferred_ptrs(self):
        return self._seen

    def flush(self) -> None:
        items, self.items = self.items, []
        vecs, self.vec_items = self.vec_items, []
        self._seen = set()
        wgrad_batch(items)
        colsum_batch(vecs)


@_on_tensor_device
def colsum_batch(problems) -> None:
    """ONE launch for many column sums: `problems` = list of (partials [rows, >= off + d], off, d, out [d])."""
    if not problems:
        return
    lib = _lib.load()
    arr = (_lib.ColsumProblem * len(problems))()
    for q, (part, off, d, out) in zip(arr, problems):
        if not (part.is_cuda and out.is_cuda and part.dtype == out.dtype == torch.float32) or part.stride(1) != 1 or out.numel() != d:
            raise RuntimeError("colsum_batch: fp32 CUDA partial rows with unit column stride and a [d] output")
        q.a, q.rows, q.stride, q.cols, q.alpha, q.out = part.data_ptr() + 4 * off, part.shape[0], part.stride(0), d, 1.0, ptr(out)
    _lib.check(lib.alignn_b200_colsum_batch(arr, len(problems), stream_ptr()), "alignn_b200_colsum_batch")


@_on_tensor_device
def colsum_rows(a: torch.Tensor) -> torch.Tensor:
    """Column sums of a tall contiguous [n, d] matrix, deterministic two-stage reduction."""
    lib = _lib.load()
    require_cuda(a)
    n, d = a.shape
    _check_d(d)
    rows = partial_rows(n, d)
    part = torch.empty(rows, d, device=a.device, dtype=torch.float32)
    _lib.check(lib.alignn_b200_colsum_partials(ptr(a), n, d, ptr(part), rows, stream_ptr()), "alignn_b200_colsum_partials")
    return colsum(part)


def linear_table(lin) -> ImageTable:
    """Images of one nn.Linear (weight zero-padded along K to a multiple of 32) and of its transpose, cached on the module."""
    dev = lin.weight.device
    tbl = getattr(lin, "_alignn_b200_images", None)
    if tbl is not None and tbl.device == dev:
        return tbl
    k_pad = (lin.in_features + 31) // 32 * 32
    tbl = ImageTable(dev)
    tbl.add_image("w", lin.out_features, k_pad, [(lin.weight, False, 0, 0)], dev)
    tbl.add_image("wT", k_pad, lin.out_features, [(lin.weight, True, 0, 0)], dev)
    object.__setattr__(lin, "_alignn_b200_images", tbl)
    return tbl


class input_grads_only:
    """Context manager for a backward pass whose PARAMETER gradients are thrown away -- `torch.autograd.grad(energy, r)`
    for forces (alignn/models/alignn_atomwise.py:530-539 outside force training): the library's autograd Functions then
    skip their weight-gradient GEMMs and bias / norm-parameter reductions and return None for them.  (autograd's own
    `needs_input_grad` cannot tell: it is fixed at forward time from `requires_grad`.)  A plain process-wide flag, because
    the autograd engine runs CUDA nodes on its own thread."""
    active = False

    def __enter__(self):
        self._prev = input_grads_only.active
        input_grads_only.active = True

    def __exit__(self, *exc):
        input_grads_only.active = self._prev


def _pad_cols(x: torch.Tensor, k_pad: int) -> torch.Tensor:
    x = x.contiguous()
    return x if x.shape[1] == k_pad else torch.nn.functional.pad(x, (0, k_pad - x.shape[1]))


class _TCLinearFn(torch.autograd.Function):
    """y = x W^T + b on the wgmma bf16x3 GEMMs (forward, data gradient, weight gradient)."""

    @staticmethod
    def forward(ctx, x, weight, bias, tbl):
        x = _pad_cols(x, tbl.images["w"].K)
        ctx.save_for_backward(x)
        ctx.tbl = tbl
        ctx.k_in = weight.shape[1]
        return gemm_gather(x, tbl.images["w"], bias.contiguous())

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, go):
        (x,) = ctx.saved_tensors
        go = go.contiguous()
        gx = None
        if ctx.needs_input_grad[0]:
            gx = gemm_gather(go, ctx.tbl.images["wT"])[:, :ctx.k_in]
        if input_grads_only.active:
            return gx, None, None, None
        gw = wgrad(go, x, 1)[:, :ctx.k_in]
        gb = colsum_rows(go)
        return gx, gw, gb, None


def tc_linear_supported(in_features: int, out_features: int) -> bool:
    k_pad = (in_features + 31) // 32 * 32
    return out_features in _lib.SUPPORTED_D and wgrad_supported(out_features, k_pad)


@_on_tensor_device
def tc_linear(x: torch.Tensor, lin) -> torch.Tensor:
    """nn.Linear forward/backward on the tensor-core kernels; the input width is zero-padded to a multiple of 32."""
    tbl = linear_table(lin)
    tbl.refresh()
    return _TCLinearFn.apply(x, lin.weight, lin.bias, tbl)


# ---- train-mode BatchNorm backward statistics taken by the consumer's data-gradient GEMM ----------------------------
# The first pass of a train-mode BatchNorm1d + SiLU backward reduces its input R and the incoming gradient g_out to
# c1 = mean(gu), c2 = mean(gu * xhat).  When g_out is the data gradient of the next layer's Linear, that GEMM's epilogue
# already holds g_out and can take the two sums on the way out (gemm_gather(..., bn_bwd=...)), saving the reduction pass.
# The hand-off between the two autograd Functions:
#   forward   the producer marks its output with a BNFold (R and the four vectors); a consumer that finds the mark on
#             its input keeps the BNFold on its ctx
#   backward  the consumer computes that input's gradient with the fold and attaches (fold, partials, _version) to the
#             tensor it returns; the producer uses the partials only if it receives that tensor at that version for its
#             own BNFold, and otherwise runs bn_backward_reduce -- autograd summed several contributions, a hook replaced
#             or changed the gradient, or no consumer GEMM produced it (the pool, user code).
# R must not outlive the backward that needs it (the producer's saved tensors are freed there, and a graph kept alive
# by the caller's `loss` would otherwise pin every R of the step): the consumer drops its reference after its data-
# gradient GEMM, and the producer's backward releases the fold's tensors.  A second backward through a retained graph
# therefore runs bn_backward_reduce.
_FOLD_ATTR, _PART_ATTR = "_alignn_b200_bn_fold", "_alignn_b200_bn_part"


class bn_fold:
    """Process-wide switch: with `bn_fold.enabled = False` consumers take no fold and every train-mode BatchNorm
    backward runs bn_backward_reduce."""
    enabled = True


class BNFold:
    __slots__ = ("vecs",)

    def __init__(self, R, scale, shift, mean, rstd):
        self.vecs = (R, scale, shift, mean, rstd)        # None once the producer's backward has run

    def release(self) -> None:
        self.vecs = None


def bn_fold_offer(out: torch.Tensor, R, scale, shift, mean, rstd) -> BNFold:
    """Producer forward: mark the BatchNorm + SiLU output `out` of input R."""
    fold = BNFold(R, scale, shift, mean, rstd)
    setattr(out, _FOLD_ATTR, fold)
    return fold


def bn_fold_take(x: torch.Tensor, n_cols: int) -> Optional[BNFold]:
    """Consumer forward: the mark of x's producer, if x's gradient will be a GEMM output of n_cols columns."""
    fold = getattr(x, _FOLD_ATTR, None)
    if fold is None or fold.vecs is None or not bn_fold.enabled or tuple(fold.vecs[0].shape) != (x.shape[0], n_cols):
        return None
    return fold


def dgrad_gemm(fold: Optional[BNFold], A: torch.Tensor, w: "WeightImage", **kw):
    """Consumer backward: gemm_gather(A, w, **kw) -> (C, partials of the fold or None)."""
    if fold is None or fold.vecs is None:
        return gemm_gather(A, w, **kw), None
    return gemm_gather(A, w, bn_bwd=fold.vecs, **kw)


def bn_fold_attach(g: torch.Tensor, fold: Optional[BNFold], part: Optional[torch.Tensor]) -> None:
    """Consumer backward: attach the partials to the gradient tensor g that is returned to autograd."""
    if fold is not None and part is not None:
        setattr(g, _PART_ATTR, (fold, part, g._version))


def bn_backward_stats(fold: Optional[BNFold], g_out: torch.Tensor, R, scale, shift, mean, rstd):
    """Producer backward: (c1, c2) from the consumer's partials if g_out is the tensor they were taken over, unchanged,
    for this producer's fold; bn_backward_reduce otherwise.  Releases the fold's tensors either way."""
    got = getattr(g_out, _PART_ATTR, None)
    if fold is not None:
        fold.release()
    if fold is not None and got is not None and got[0] is fold and got[2] == g_out._version:
        n, d = R.shape
        part = got[1]
        c = colsum(part.view(part.shape[0], 2 * d), 1.0 / n)
        return c[:d], c[d:]
    return bn_backward_reduce(R, g_out, scale, shift, mean, rstd)


# ---- Linear -> BatchNorm1d(train) -> SiLU (embedding MLP layers) ------------------------------------
class _MLPBNTrainFn(torch.autograd.Function):
    """One embedding layer in train mode, entirely on library kernels: tensor-core Linear, two-stage batch
    statistics (fp64 finalize + running-stat update), fused normalise+SiLU, and the matching backward."""

    @staticmethod
    def forward(ctx, x, weight, bias, gamma, beta, bn, tbl):
        ctx.fold_in = bn_fold_take(x, tbl.images["wT"].N)        # x is itself a train-mode BatchNorm output
        x = _pad_cols(x, tbl.images["w"].K)
        # Linear + per-channel batch statistics in one pass (column sums leave through the GEMM epilogue)
        R, part = gemm_gather(x, tbl.images["w"], bias.contiguous(), stats=True)
        n, d = R.shape
        track = bn.track_running_stats and bn.running_mean is not None
        scale, shift, mean, rstd = bn_finalize(part, 0, n, gamma.contiguous(), beta.contiguous(), bn.eps, float(bn.momentum),
                                               bn.running_mean if track else None, bn.running_var if track else None)
        if track and bn.num_batches_tracked is not None:
            bn.num_batches_tracked.add_(1)
        out = affine_silu_residual(R, None, scale, shift)
        ctx.fold_out = bn_fold_offer(out, R, scale, shift, mean, rstd)
        ctx.save_for_backward(x, R, scale, shift, mean, rstd)
        ctx.tbl = tbl
        ctx.k_in = weight.shape[1]
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, go):
        lib = _lib.load()
        x, R, scale, shift, mean, rstd = ctx.saved_tensors
        c1, c2 = bn_backward_stats(ctx.fold_out, go, R, scale, shift, mean, rstd)
        go = go.contiguous()
        n, d = R.shape
        gR = torch.empty_like(R)
        with _span("bn_backward_apply", 12 * n * d):
            _lib.check(lib.alignn_b200_bn_backward_apply(ptr(R), ptr(go), ptr(scale), ptr(shift), ptr(mean), ptr(rstd),
                                                         ptr(c1.contiguous()), ptr(c2.contiguous()), n, d, ptr(gR), stream_ptr()),
                       "alignn_b200_bn_backward_apply")
        gx = None
        fold_in, ctx.fold_in = ctx.fold_in, None         # used once: a retained graph's next backward falls back
        if ctx.needs_input_grad[0]:
            gx, part = dgrad_gemm(fold_in, gR, ctx.tbl.images["wT"])
            gx = gx[:, :ctx.k_in]
            bn_fold_attach(gx, fold_in, part)            # on the view autograd receives
        if input_grads_only.active:
            return gx, None, None, None, None, None, None
        gw = wgrad(gR, x, 1)[:, :ctx.k_in]
        # a bias that feeds a train-mode BatchNorm has an identically zero gradient (sum_rows gR == 0)
        return gx, gw, torch.zeros_like(c1), c2 * n, c1 * n, None, None


# ---- Linear -> LayerNorm -> SiLU (embedding layers of the LayerNorm model, alignn_atomwise.py:249-268) ---------------
class _MLPLNFn(torch.autograd.Function):
    """Tensor-core Linear, then ONE row kernel for LayerNorm + SiLU (forward) and one for their backward (which also
    leaves the per-block sums for d gamma / d beta); replaces 5 library passes over the [T, d] activations."""

    @staticmethod
    def forward(ctx, x, weight, bias, gamma, beta, eps, tbl):
        lib = _lib.load()
        x = _pad_cols(x, tbl.images["w"].K)
        h = gemm_gather(x, tbl.images["w"], bias.contiguous())
        n, d = h.shape
        gamma, beta = gamma.contiguous(), beta.contiguous()
        out = torch.empty_like(h)
        rowstat = torch.empty(n, 2, device=h.device, dtype=torch.float32)
        with _span("ln_silu_forward", 8 * n * d):
            _lib.check(lib.alignn_b200_ln_silu_forward(ptr(h), ptr(gamma), ptr(beta), float(eps), n, d, ptr(out), ptr(rowstat),
                                                        stream_ptr()), "alignn_b200_ln_silu_forward")
        ctx.save_for_backward(x, h, rowstat, gamma, beta)
        ctx.tbl = tbl
        ctx.k_in = weight.shape[1]
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, go):
        lib = _lib.load()
        x, h, rowstat, gamma, beta = ctx.saved_tensors
        go = go.contiguous()
        n, d = h.shape
        gh = torch.empty_like(h)
        rows = partial_rows(n, d)
        part = torch.empty(rows, 2 * d, device=h.device, dtype=torch.float32)
        with _span("ln_silu_backward", 12 * n * d):
            _lib.check(lib.alignn_b200_ln_silu_backward(ptr(h), ptr(go), ptr(rowstat), ptr(gamma), ptr(beta), n, d, ptr(gh),
                                                         ptr(part), rows, stream_ptr()), "alignn_b200_ln_silu_backward")
        gx = None
        if ctx.needs_input_grad[0]:
            gx = gemm_gather(gh, ctx.tbl.images["wT"])[:, :ctx.k_in]
        if input_grads_only.active:
            return gx, None, None, None, None, None, None
        gwb = colsum(part)
        gw = gb = None
        if ctx.needs_input_grad[1]:
            gw = wgrad(gh, x, 1)[:, :ctx.k_in]
        if ctx.needs_input_grad[2]:
            gb = colsum_rows(gh)
        return gx, gw, gb, gwb[:d], gwb[d:], None, None


@_on_tensor_device
def mlp_ln(x, lin, ln):
    tbl = linear_table(lin)
    tbl.refresh()
    return _MLPLNFn.apply(x, lin.weight, lin.bias, ln.weight, ln.bias, ln.eps, tbl)


@_on_tensor_device
def mlp_bn_train(x, lin, bn):
    tbl = linear_table(lin)
    tbl.refresh()
    return _MLPBNTrainFn.apply(x, lin.weight, lin.bias, bn.weight, bn.bias, bn, tbl)
