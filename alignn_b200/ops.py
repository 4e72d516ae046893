"""Tensor-level wrappers over the C ABI (include/alignn_b200.h).  Device memory, streams
and the autograd glue are PyTorch plumbing; all arithmetic of the edge-gated conv stage
runs in libalignn_b200.so.  Every function raises if the tensors are not fp32/int32 CUDA
tensors or if the library reports an error -- there is no fallback path.
"""
from __future__ import annotations

import ctypes as C
import functools
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


FIRE_DEFAULTS = dict(maxstep=0.2, dtmax=1.0, n_min=5, finc=1.1, fdec=0.5, astart=0.1, fa=0.99)   # ase FIRE defaults
FIRE_DT0, FIRE_A0 = 0.1, 0.1                                                                    # its initial dt and a
FIRE_BAD_INPUT = 3            # istate status of a crystal whose batch slice does not match its atom count
FIRE_MAX_STEPS = 2 ** 31 - 1  # steps travels as an int32


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
    par = dict(FIRE_DEFAULTS, **fire)
    want = ((grad, torch.float32), (active, torch.int32), (batch_offsets, torch.int32), (atom_offsets, torch.int64),
            (positions, torch.float64), (velocities, torch.float64), (forces, torch.float32), (fstate, torch.float64),
            (istate, torch.int32))
    for t, dt in want:
        if not t.is_cuda or t.device != grad.device:
            raise RuntimeError(f"fire_step needs all operands on one CUDA device; got {t.device} and {grad.device}")
        if t.dtype != dt or not t.is_contiguous():
            raise RuntimeError(f"fire_step: expected a contiguous {dt} tensor, got {t.dtype}")
    B, A = atom_offsets.numel() - 1, active.numel()
    N = positions.numel() // 3
    if (velocities.numel() != 3 * N or forces.numel() != 3 * N or fstate.numel() != 2 * B or istate.numel() != 4 * B
            or batch_offsets.numel() != A + 1 or grad.dim() != 2 or grad.shape[1] != 3):
        raise ValueError("fire_step: inconsistent operand shapes")
    if isinstance(steps, bool) or int(steps) != steps or not 1 <= int(steps) <= FIRE_MAX_STEPS:
        raise ValueError(f"fire_step: steps must be an integer in [1, {FIRE_MAX_STEPS}], got {steps!r}")
    if not 0 <= int(par["n_min"]) <= FIRE_MAX_STEPS:
        raise ValueError(f"fire_step: n_min must be in [0, {FIRE_MAX_STEPS}], got {par['n_min']!r}")
    p = _lib.FireParams(float(par["maxstep"]), float(par["dtmax"]), float(par["finc"]), float(par["fdec"]),
                        float(par["astart"]), float(par["fa"]), float(fmax), int(par["n_min"]), int(steps),
                        float(force_multiplier))
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
    par = dict(FIRE_DEFAULTS, **fire)
    want = ((grad, torch.float32), (stress, torch.float32), (active, torch.int32), (batch_offsets, torch.int32),
            (atom_offsets, torch.int64), (positions, torch.float64), (velocities, torch.float64), (forces, torch.float32),
            (cells0, torch.float64), (logdef, torch.float64), (defgrad, torch.float64), (cells, torch.float64),
            (cell_velocities, torch.float64), (cell_forces, torch.float64), (stress_out, torch.float32),
            (fstate, torch.float64), (istate, torch.int32))
    for t, dt in want:
        if not t.is_cuda or t.device != grad.device:
            raise RuntimeError(f"fire_cell_step needs all operands on one CUDA device; got {t.device} and {grad.device}")
        if t.dtype != dt or not t.is_contiguous():
            raise RuntimeError(f"fire_cell_step: expected a contiguous {dt} tensor, got {t.dtype}")
    B, A = atom_offsets.numel() - 1, active.numel()
    N = positions.numel() // 3
    if (velocities.numel() != 3 * N or forces.numel() != 3 * N or fstate.numel() != 2 * B or istate.numel() != 4 * B
            or batch_offsets.numel() != A + 1 or grad.dim() != 2 or grad.shape[1] != 3
            or stress.numel() != 9 * A or stress_out.numel() != 6 * B
            or any(t.numel() != 9 * B for t in (cells0, logdef, defgrad, cells, cell_velocities, cell_forces))):
        raise ValueError("fire_cell_step: inconsistent operand shapes")
    if isinstance(steps, bool) or int(steps) != steps or not 1 <= int(steps) <= FIRE_MAX_STEPS:
        raise ValueError(f"fire_cell_step: steps must be an integer in [1, {FIRE_MAX_STEPS}], got {steps!r}")
    if not 0 <= int(par["n_min"]) <= FIRE_MAX_STEPS:
        raise ValueError(f"fire_cell_step: n_min must be in [0, {FIRE_MAX_STEPS}], got {par['n_min']!r}")
    p = _lib.FireCellParams(_lib.FireParams(float(par["maxstep"]), float(par["dtmax"]), float(par["finc"]),
                                            float(par["fdec"]), float(par["astart"]), float(par["fa"]), float(fmax),
                                            int(par["n_min"]), int(steps), float(force_multiplier)), float(stress_wt))
    _lib.check(lib.alignn_b200_fire_cell_step(C.byref(p), active.data_ptr(), A, atom_offsets.data_ptr(), batch_offsets.data_ptr(),
                                              B, grad.data_ptr(), grad.shape[0], stress.data_ptr(), A, positions.data_ptr(),
                                              velocities.data_ptr(), forces.data_ptr(), cells0.data_ptr(), logdef.data_ptr(),
                                              defgrad.data_ptr(), cells.data_ptr(), cell_velocities.data_ptr(),
                                              cell_forces.data_ptr(), stress_out.data_ptr(), fstate.data_ptr(),
                                              istate.data_ptr(), stream_ptr()), "alignn_b200_fire_cell_step")


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
                stats: bool = False, out: Optional[torch.Tensor] = None):
    """out[r] = A[r] @ W^T (+ bias) (+ add0[idx0[r]]) (+ add1[idx1[r]]) on wgmma.

    add0 / add1 are 2-D fp32 views with unit column stride and w.N columns (column slices of a wider matrix are fine);
    idx None = identity (a residual).  stats=True also returns the per-CTA partial column sums [rows, 2, N] of out and
    out^2 (alignn.py:123 batch statistics; feed `bn_finalize(partials, 0, M, ...)`)."""
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
    if out is None:
        out = torch.empty(M, w.N, device=A.device, dtype=torch.float32)
    part = None
    if stats:
        rows = int(lib.alignn_b200_gemm_gather_stat_rows(M, w.N))
        part = torch.empty(max(rows, 1), 2, w.N, device=A.device, dtype=torch.float32)
    a = _lib.GemmGatherArgs(
        struct_size=C.sizeof(_lib.GemmGatherArgs), M=M, N=w.N, K=w.K, A=ptr_any(A), lda=A.stride(0),
        w_image=ptr_any(w.buf), bias=ptr_any(bias),
        add0=ptr_any(add0), ld0=add0.stride(0) if add0 is not None else 0, idx0=ptr_any(idx0),
        add1=ptr_any(add1), ld1=add1.stride(0) if add1 is not None else 0, idx1=ptr_any(idx1),
        C=ptr_any(out), ldc=out.stride(0), stats=ptr_any(part), stream=stream_ptr())
    nb = 4 * M * (w.K + w.N) + (8 * M if idx0 is not None else 0) + (4 * M * w.N if (add0 is not None and idx0 is None) else 0)
    kind = "+gather" if idx0 is not None else ("+residual" if add0 is not None else "")
    with _span(f"gemm_gather<{min(w.N, 256)}>" + kind + ("+stats" if stats else ""), nb):
        _lib.check(lib.alignn_b200_gemm_gather(C.byref(a)), "alignn_b200_gemm_gather")
    return (out, part) if stats else out


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


# ---- Linear -> BatchNorm1d(train) -> SiLU (embedding MLP layers) ------------------------------------
class _MLPBNTrainFn(torch.autograd.Function):
    """One embedding layer in train mode, entirely on library kernels: tensor-core Linear, two-stage batch
    statistics (fp64 finalize + running-stat update), fused normalise+SiLU, and the matching backward."""

    @staticmethod
    def forward(ctx, x, weight, bias, gamma, beta, bn, tbl):
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
        ctx.save_for_backward(x, R, scale, shift, mean, rstd)
        ctx.tbl = tbl
        ctx.k_in = weight.shape[1]
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, go):
        lib = _lib.load()
        x, R, scale, shift, mean, rstd = ctx.saved_tensors
        go = go.contiguous()
        n, d = R.shape
        c1, c2 = bn_backward_reduce(R, go, scale, shift, mean, rstd)
        gR = torch.empty_like(R)
        with _span("bn_backward_apply", 12 * n * d):
            _lib.check(lib.alignn_b200_bn_backward_apply(ptr(R), ptr(go), ptr(scale), ptr(shift), ptr(mean), ptr(rstd),
                                                         ptr(c1.contiguous()), ptr(c2.contiguous()), n, d, ptr(gR), stream_ptr()),
                       "alignn_b200_bn_backward_apply")
        gx = None
        if ctx.needs_input_grad[0]:
            gx = gemm_gather(gR, ctx.tbl.images["wT"])[:, :ctx.k_in]
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
