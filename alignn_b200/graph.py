"""Graph container for the edge-gated conv hot path.

The reference hands `dgl.DGLGraph` objects (`g`, `lg`) to `ALIGNN.forward`
(alignn/models/alignn.py:282-294); DGL is a third-party wheel that is not part of
this build.  `Graph` exposes the subset of the DGLGraph API the reference's model
and collate code touches (SURVEY.md App. C) and, in addition, carries the
**sorted-CSR edge index** the CUDA kernels consume:

    in_ptr [Nn+1], in_eid [Ne]   edge ids stably sorted by destination  (in-CSR)
    out_ptr[Nn+1], out_eid[Ne]   edge ids stably sorted by source       (out-CSR)

all int32.  The index is integer-exact, built once on the host when the graph is
made (the reference likewise builds graph structure on the CPU and caches it,
alignn/graphs.py:544,588; lmdb_dataset.py:220-224) and moves with `.to(device)`.
`line_graph()` emits L(g) with its edges already destination-sorted so that
`in_eid` is the identity for the graph that carries ~92 % of the bytes.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np
import torch

__all__ = ["Graph", "EdgeIndex", "batch", "unbatch", "reverse", "graph", "as_graph", "bond_cosines", "lightweight_graph"]


def _np(a):
    if isinstance(a, torch.Tensor):
        return a.detach().cpu().numpy()
    return np.asarray(a)


class EdgeIndex:
    """Sorted-CSR edge index of one graph (both orientations), int32 tensors.

    `parent`: set only by `Graph.line_graph()` on the L(g) it emits -- the parent g's (in_ptr, in_eid, out_ptr,
    out_eid).  It asserts that this graph is exactly the builders' L(g) of that parent, so the edges at each atom of g
    form one bipartite block (sources in(a), destinations out(a)); `ops.egc_backward` then runs the one-pass
    line-graph backward.  None everywhere else (atom graphs, `batch`, `unbatch`, `as_graph`, `reverse`)."""

    __slots__ = ("src", "dst", "in_ptr", "in_eid", "out_ptr", "out_eid", "dst_sorted",
                 "max_in_deg", "num_nodes", "parent")

    def __init__(self, src, dst, in_ptr, in_eid, out_ptr, out_eid, dst_sorted, max_in_deg, num_nodes, parent=None):
        self.src, self.dst = src, dst
        self.in_ptr, self.in_eid = in_ptr, in_eid
        self.out_ptr, self.out_eid = out_ptr, out_eid
        self.dst_sorted = bool(dst_sorted)
        self.max_in_deg = int(max_in_deg)
        self.num_nodes = int(num_nodes)
        self.parent = None if parent is None else tuple(parent)

    @staticmethod
    def build(src: np.ndarray, dst: np.ndarray, num_nodes: int) -> "EdgeIndex":
        """Stable counting sort by dst and by src (native: alignn_b200_csr_build_host).  Bit-exact vs
        oracle.csr_by_key."""
        from . import _lib
        lib = _lib.load()
        src = np.ascontiguousarray(src, dtype=np.int64).reshape(-1)
        dst = np.ascontiguousarray(dst, dtype=np.int64).reshape(-1)
        E = src.shape[0]
        if E >= 2 ** 31 or num_nodes >= 2 ** 31:
            raise ValueError("graph too large for int32 edge index")
        if dst.shape[0] != E:
            raise ValueError("src and dst differ in length")
        i32 = lambda k: np.empty(k, dtype=np.int32)  # noqa: E731
        s32, d32, in_ptr, in_eid, out_ptr, out_eid = i32(E), i32(E), i32(num_nodes + 1), i32(E), i32(num_nodes + 1), i32(E)
        flags = np.zeros(2, dtype=np.int32)
        p = lambda a: a.ctypes.data  # noqa: E731
        rc = lib.alignn_b200_csr_build_host(p(src), p(dst), num_nodes, E, p(s32), p(d32), p(in_ptr), p(in_eid),
                                            p(out_ptr), p(out_eid), p(flags[0:1]), p(flags[1:2]))
        if rc == -1:
            raise ValueError("edge endpoint out of range")
        _lib.check(rc, "alignn_b200_csr_build_host")
        t = torch.from_numpy
        return EdgeIndex(t(s32), t(d32), t(in_ptr), t(in_eid), t(out_ptr), t(out_eid),
                         bool(flags[0]), int(flags[1]), num_nodes)

    @staticmethod
    def build_device(src: torch.Tensor, dst: torch.Tensor, num_nodes: int) -> "EdgeIndex":
        """The same index built ON THE GPU from int32 CUDA tensors (alignn_b200_csr_build: integer histogram, scan,
        stable radix sort of edge ids; bit-identical to `build`).  One 8-byte read-back (dst_sorted, max in-degree)."""
        from . import _lib
        lib = _lib.load()
        if not (src.is_cuda and dst.is_cuda):
            raise RuntimeError("EdgeIndex.build_device needs CUDA tensors")
        src = src.to(torch.int32).contiguous()
        dst = dst.to(torch.int32).contiguous()
        E, dev = src.numel(), src.device
        i32 = lambda n: torch.empty(n, device=dev, dtype=torch.int32)  # noqa: E731
        in_ptr, out_ptr, in_eid, out_eid, flags = i32(num_nodes + 1), i32(num_nodes + 1), i32(E), i32(E), i32(2)
        nb = int(lib.alignn_b200_csr_build_workspace_bytes(num_nodes, E))
        if nb == 0:
            raise ValueError("graph too large for int32 edge index")
        ws = torch.empty(nb, device=dev, dtype=torch.uint8)
        with torch.cuda.device(dev):
            _lib.check(lib.alignn_b200_csr_build(src.data_ptr(), dst.data_ptr(), num_nodes, E, in_ptr.data_ptr(), in_eid.data_ptr(),
                                                 out_ptr.data_ptr(), out_eid.data_ptr(), flags.data_ptr(), ws.data_ptr(), nb,
                                                 _lib.stream_ptr()), "alignn_b200_csr_build")
        f = flags.tolist()
        return EdgeIndex(src, dst, in_ptr, in_eid, out_ptr, out_eid, bool(f[0]), int(f[1]), num_nodes)

    _FIELDS = ("src", "dst", "in_ptr", "in_eid", "out_ptr", "out_eid")

    def to(self, device, non_blocking=False) -> "EdgeIndex":
        moved = [getattr(self, f).to(device, non_blocking=non_blocking) for f in self._FIELDS]
        parent = None if self.parent is None else [t.to(device, non_blocking=non_blocking) for t in self.parent]
        return EdgeIndex(*moved, self.dst_sorted, self.max_in_deg, self.num_nodes, parent)

    def pin_memory(self) -> "EdgeIndex":
        moved = [getattr(self, f).pin_memory() for f in self._FIELDS]
        parent = None if self.parent is None else [t.pin_memory() for t in self.parent]
        return EdgeIndex(*moved, self.dst_sorted, self.max_in_deg, self.num_nodes, parent)

    def nbytes(self) -> int:
        n = sum(getattr(self, f).numel() * 4 for f in self._FIELDS)
        return n + (0 if self.parent is None else sum(t.numel() * 4 for t in self.parent))


class _EdgeBatch:
    """What a user function passed to `apply_edges` sees (edges.src / .dst / .data)."""

    def __init__(self, g: "Graph"):
        s, d = g.index.src.long(), g.index.dst.long()
        self.src = {k: v[s] for k, v in g.ndata.items()}
        self.dst = {k: v[d] for k, v in g.ndata.items()}
        self.data = dict(g.edata)


class Graph:
    """Batched directed multigraph with feature dicts and a sorted-CSR edge index."""

    def __init__(self, src=None, dst=None, num_nodes: Optional[int] = None,
                 batch_num_nodes=None, batch_num_edges=None, *, _index: Optional[EdgeIndex] = None):
        if _index is None:
            if isinstance(src, torch.Tensor) and src.is_cuda and num_nodes is not None:
                # edges already on the GPU (device-side neighbour list / line graph): build the index there
                _index = EdgeIndex.build_device(src.reshape(-1), torch.as_tensor(dst, device=src.device).reshape(-1),
                                                int(num_nodes))
            else:
                src, dst = _np(src).reshape(-1), _np(dst).reshape(-1)
                if num_nodes is None:
                    num_nodes = int(max(src.max(), dst.max())) + 1 if src.size else 0
                _index = EdgeIndex.build(src, dst, int(num_nodes))
        self.index = _index
        self._n = _index.num_nodes
        E = int(_index.src.numel())
        self._bnn = torch.tensor([self._n], dtype=torch.int64) if batch_num_nodes is None \
            else torch.as_tensor(batch_num_nodes, dtype=torch.int64).reshape(-1).cpu()
        self._bne = torch.tensor([E], dtype=torch.int64) if batch_num_edges is None \
            else torch.as_tensor(batch_num_edges, dtype=torch.int64).reshape(-1).cpu()
        if int(self._bnn.sum()) != self._n or int(self._bne.sum()) != E:
            raise ValueError("batch_num_nodes / batch_num_edges do not add up")
        self.ndata: dict = {}
        self.edata: dict = {}
        # per-graph node offsets [B+1] (int32) for pooling; part of the structure that moves with .to()
        seg = torch.zeros(self._bnn.numel() + 1, dtype=torch.int32)
        seg[1:] = torch.cumsum(self._bnn, 0).to(torch.int32)
        self._seg = seg

    # ---- DGLGraph API subset (SURVEY.md App. C) -----------------------------
    def edges(self):
        return self.index.src, self.index.dst

    def num_nodes(self) -> int:
        return self._n

    def num_edges(self) -> int:
        return int(self.index.src.numel())

    number_of_nodes = num_nodes
    number_of_edges = num_edges

    @property
    def batch_size(self) -> int:
        return int(self._bnn.numel())

    def batch_num_nodes(self):
        return self._bnn

    def batch_num_edges(self):
        return self._bne

    @property
    def device(self):
        return self.index.src.device

    def local_var(self) -> "Graph":
        """Shallow copy: same structure, fresh feature dicts (reference: alignn.py:88,159,295)."""
        g = Graph(batch_num_nodes=self._bnn, batch_num_edges=self._bne, _index=self.index)
        g.ndata.update(self.ndata)
        g.edata.update(self.edata)
        g._seg = self._seg
        return g

    def to(self, device, non_blocking: bool = False) -> "Graph":
        device = torch.device(device)
        if device == self.device:
            return self
        g = Graph(batch_num_nodes=self._bnn, batch_num_edges=self._bne,
                  _index=self.index.to(device, non_blocking))
        g._seg = self._seg.to(device, non_blocking=non_blocking)
        g.ndata = {k: v.to(device, non_blocking=non_blocking) for k, v in self.ndata.items()}
        g.edata = {k: v.to(device, non_blocking=non_blocking) for k, v in self.edata.items()}
        return g

    def pin_memory(self) -> "Graph":
        g = Graph(batch_num_nodes=self._bnn, batch_num_edges=self._bne, _index=self.index.pin_memory())
        g._seg = self._seg.pin_memory()
        g.ndata = {k: v.pin_memory() for k, v in self.ndata.items()}
        g.edata = {k: v.pin_memory() for k, v in self.edata.items()}
        return g

    def nbytes(self) -> int:
        """Bytes moved by `.to(device)` (structure + features)."""
        n = self.index.nbytes() + self._seg.numel() * 4
        for d in (self.ndata, self.edata):
            n += sum(v.numel() * v.element_size() for v in d.values())
        return n

    def apply_edges(self, func):
        """User-defined edge function (e.g. compute_bond_cosines, alignn/graphs.py:847)."""
        self.edata.update(func(_EdgeBatch(self)))

    def node_graph_offsets(self) -> torch.Tensor:
        """int32 [B+1] prefix of batch_num_nodes on this graph's device (per-graph pooling)."""
        if self._seg.device != self.device:       # graph assembled directly from device tensors
            self._seg = self._seg.to(self.device)
        return self._seg

    def line_graph(self, backtracking: bool = True, shared: bool = False) -> "Graph":
        """L(g): node i == edge i of g; edge (i -> j) iff dst(i) == src(j) and i != j.

        Same edge SET as `g.line_graph(shared=True)` at alignn/graphs.py:588 (backtracking
        pairs kept); emitted sorted by (j, i) -- destination-major -- instead of DGL's
        source-major order.  L(g)'s edge order is never observable (z is consumed, not
        returned), and within one destination the sources stay ascending, so segment sums
        add in the same order as the reference.
        """
        if not backtracking:
            raise NotImplementedError("backtracking=False is not used by the reference")
        from . import _lib
        lib = _lib.load()
        ix = self.index
        if self.device.type == "cuda":
            return self._line_graph_device(shared)
        src = np.ascontiguousarray(ix.src.cpu().numpy())
        in_ptr = np.ascontiguousarray(ix.in_ptr.cpu().numpy())
        in_eid = np.ascontiguousarray(ix.in_eid.cpu().numpy())
        E = src.shape[0]
        p = lambda a: a.ctypes.data  # noqa: E731
        T = int(lib.alignn_b200_line_graph_count_host(p(src), p(in_ptr), p(in_eid), E))
        if T < 0:
            raise RuntimeError("alignn_b200_line_graph_count_host failed")
        li, lj = np.empty(T, dtype=np.int64), np.empty(T, dtype=np.int64)
        bne = np.ascontiguousarray(self._bne.numpy(), dtype=np.int64)
        lbne = np.zeros(bne.shape[0], dtype=np.int64)
        _lib.check(lib.alignn_b200_line_graph_build_host(p(src), p(in_ptr), p(in_eid), E, p(bne), bne.shape[0], T,
                                                         p(li), p(lj), p(lbne)), "alignn_b200_line_graph_build_host")
        lg = Graph(li, lj, E, self._bne.clone(), lbne)
        lg.index.parent = (ix.in_ptr, ix.in_eid, ix.out_ptr, ix.out_eid)
        if self.device.type != "cpu":
            lg = lg.to(self.device)
        if shared:
            lg.ndata.update(self.edata)
        return lg


    def _line_graph_device(self, shared: bool) -> "Graph":
        """L(g) built on the GPU (alignn_b200_line_graph_offsets / _fill + alignn_b200_csr_build): same edge list as the
        host builder, bit for bit.  One small read-back (T and the per-crystal pair counts) sizes the outputs."""
        from . import _lib
        lib = _lib.load()
        ix, dev, E = self.index, self.device, self.num_edges()
        off = torch.empty(E + 1, device=dev, dtype=torch.int32)
        nb = int(lib.alignn_b200_line_graph_workspace_bytes(E))
        ws = torch.empty(max(nb, 1), device=dev, dtype=torch.uint8)
        with torch.cuda.device(dev):
            st = _lib.stream_ptr()
            _lib.check(lib.alignn_b200_line_graph_offsets(ix.src.data_ptr(), ix.dst.data_ptr(), ix.in_ptr.data_ptr(), E,
                                                          off.data_ptr(), ws.data_ptr(), nb, st), "alignn_b200_line_graph_offsets")
            eoff = torch.zeros(self._bne.numel() + 1, dtype=torch.int64)
            eoff[1:] = torch.cumsum(self._bne, 0)
            at = off[eoff.to(dev)].tolist()                      # pairs before each crystal's first bond; last = T
            T = int(at[-1])
            lsrc, ldst = (torch.empty(T, device=dev, dtype=torch.int32) for _ in range(2))
            _lib.check(lib.alignn_b200_line_graph_fill(ix.src.data_ptr(), ix.dst.data_ptr(), ix.in_ptr.data_ptr(),
                                                       ix.in_eid.data_ptr(), E, off.data_ptr(), lsrc.data_ptr(), ldst.data_ptr(), st),
                       "alignn_b200_line_graph_fill")
        lbne = torch.tensor([b - a for a, b in zip(at[:-1], at[1:])], dtype=torch.int64)
        lg = Graph(lsrc, ldst, E, self._bne.clone(), lbne)
        lg.index.parent = (ix.in_ptr, ix.in_eid, ix.out_ptr, ix.out_eid)
        if shared:
            lg.ndata.update(self.edata)
        return lg

    def batch_num_nodes_on_device(self) -> torch.Tensor:
        """batch_num_nodes as an int64 tensor on this graph's device (cached: no host copy inside a CUDA-graph capture)."""
        t = getattr(self, "_bnn_dev", None)
        if t is None or t.device != self.device:
            t = self._bnn.to(self.device)
            self._bnn_dev = t
        return t

    def edge_graph_offsets64(self) -> torch.Tensor:
        """int64 [B+1] prefix of batch_num_edges on this graph's device (per-crystal edge ranges, virial stress)."""
        t = getattr(self, "_eoff64", None)
        if t is None or t.device != self.device:
            t = torch.zeros(self._bne.numel() + 1, dtype=torch.int64)
            t[1:] = torch.cumsum(self._bne, 0)
            t = t.to(self.device)
            self._eoff64 = t
        return t


# ---- module-level helpers mirroring dgl.* ------------------------------------
def graph(data, num_nodes=None) -> Graph:
    """dgl.graph((src, dst), num_nodes=...) (alignn/graphs.py:544)."""
    return Graph(data[0], data[1], num_nodes)


def batch(graphs: Sequence[Graph]) -> Graph:
    """dgl.batch (alignn/lmdb_dataset.py:93-94): concatenate, offset ids, keep order."""
    noff, s, d = 0, [], []
    for g in graphs:
        s.append(g.index.src.cpu().numpy().astype(np.int64) + noff)
        d.append(g.index.dst.cpu().numpy().astype(np.int64) + noff)
        noff += g.num_nodes()
    bg = Graph(np.concatenate(s), np.concatenate(d), noff,
               torch.cat([g.batch_num_nodes() for g in graphs]),
               torch.cat([g.batch_num_edges() for g in graphs]))
    for k in graphs[0].ndata:
        bg.ndata[k] = torch.cat([g.ndata[k] for g in graphs], 0)
    for k in graphs[0].edata:
        bg.edata[k] = torch.cat([g.edata[k] for g in graphs], 0)
    return bg


def unbatch(g: Graph):
    """dgl.unbatch (alignn_atomwise.py:492)."""
    out, no, eo = [], 0, 0
    src, dst = g.index.src.cpu().numpy(), g.index.dst.cpu().numpy()
    for n, e in zip(g.batch_num_nodes().tolist(), g.batch_num_edges().tolist()):
        h = Graph(src[eo:eo + e] - no, dst[eo:eo + e] - no, n)
        h.ndata = {k: v[no:no + n] for k, v in g.ndata.items()}
        h.edata = {k: v[eo:eo + e] for k, v in g.edata.items()}
        out.append(h)
        no, eo = no + n, eo + e
    return out


def reverse(g: Graph, copy_ndata: bool = True, copy_edata: bool = False) -> Graph:
    """dgl.reverse (alignn_atomwise.py:555): swap src/dst, keep edge ids."""
    ix = g.index
    r = Graph(batch_num_nodes=g.batch_num_nodes(), batch_num_edges=g.batch_num_edges(),
              _index=EdgeIndex(ix.dst, ix.src, ix.out_ptr, ix.out_eid, ix.in_ptr, ix.in_eid,
                               False, 0, ix.num_nodes))
    if copy_ndata:
        r.ndata.update(g.ndata)
    if copy_edata:
        r.edata.update(g.edata)
    return r


def as_graph(g) -> Graph:
    """Accept our Graph, or anything DGLGraph-like (edges/num_nodes/batch_num_* /ndata/edata)."""
    if isinstance(g, Graph):
        return g
    if not (hasattr(g, "edges") and hasattr(g, "num_nodes")):
        raise TypeError(f"expected alignn_b200.Graph or a DGLGraph-like object, got {type(g)!r}")
    # only the STRUCTURE (sorted-CSR index) is cached on the foreign object; features are taken from the live object
    # on every call, so updated edata / ndata (MD, relaxation, augmentation) are never stale
    cached = getattr(g, "_alignn_b200_graph", None)
    if cached is None:
        s, d = g.edges()
        cached = Graph(s, d, g.num_nodes(), g.batch_num_nodes(), g.batch_num_edges())
        dev = s.device if isinstance(s, torch.Tensor) else torch.device("cpu")
        if dev.type != "cpu" and cached.device != dev:
            cached = cached.to(dev)
        try:
            g._alignn_b200_graph = cached
        except Exception:
            pass
    out = cached.local_var()
    out.ndata.clear()
    out.edata.clear()
    out.ndata.update(dict(g.ndata))
    out.edata.update(dict(g.edata))
    return out


def lightweight_graph(g: Graph, cart: torch.Tensor, inner_cutoff: float):
    """The bonds of a CUDA graph `g` no longer than `inner_cutoff`, as eALIGNN builds them inside forward
    (`lightweight_line_graph` with `compute_pair_vector_and_distance`, alignn/models/utils.py:47-55, 129-222):
    r = (cart[dst] + edata["images"]) - cart[src] in fp32, bonds with |r| > inner_cutoff dropped, order kept.
    Returns (filtered Graph, r' [E',3]).  The filtered graph shares `ndata`, holds `edata` filtered to the kept bonds plus
    `edge_ids` (crystal-local ids when the batch has several crystals, global ids otherwise, as the reference numbers
    them) and the kept bonds per crystal in batch_num_edges.  Its index is built on the device, so its
    `line_graph()` also runs there and carries the parent descriptor."""
    from . import ops
    if g.device.type != "cuda":
        raise RuntimeError("lightweight_graph needs a CUDA graph (the filter is a device kernel)")
    eoff = g.edge_graph_offsets64()
    src, dst, r, _, eids, kept = ops.bond_cutoff_filter(cart, g.index, g.edata["images"], eoff, inner_cutoff)
    glob = eids
    if g.batch_size > 1:                                    # crystal-local ids -> positions in g
        gid = torch.repeat_interleave(torch.arange(g.batch_size, device=g.device), kept.to(g.device), output_size=eids.numel())
        glob = eids + eoff[gid]
    out = Graph(src, dst, g.num_nodes(), g.batch_num_nodes(), kept)
    out.ndata.update(g.ndata)
    out.edata = {k: v[glob] for k, v in g.edata.items()}
    out.edata["edge_ids"] = eids
    return out, r


def bond_cosines(r: torch.Tensor, lg: Graph) -> torch.Tensor:
    """Bond-angle cosines for every L(g) edge (compute_bond_cosines, alignn/graphs.py:847-864)."""
    r1 = -r[lg.index.src.long()]
    r2 = r[lg.index.dst.long()]
    c = torch.sum(r1 * r2, dim=1) / (torch.norm(r1, dim=1) * torch.norm(r2, dim=1))
    return torch.clamp(c, -1, 1)
