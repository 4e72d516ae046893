"""Shape-bucketed CUDA-graph replay for variable-size batches.

Real loaders hand the model batches whose atom / bond / bond-pair counts (N, E, T) change every step
(alignn/lmdb_dataset.py:87-108), while a CUDA graph is captured for fixed shapes.  This module pads a collated batch
`(g, lg)` to the next bucket `(N_b, E_b, T_b)` by appending ONE padding crystal whose bonds are arranged so that its
line graph has exactly the missing number of bond pairs, and replays one captured graph per bucket.

Why results do not change (LayerNorm models -- the ones the reference actually trains, alignn/train.py:238 -- and
eval-mode BatchNorm): every kernel of the conv path works row by row; a row's output depends on its own inputs and on
the rows of its own crystal (segment sums never cross crystals, SURVEY.md section 8e), so the rows of the real
crystals are bit-identical with and without the padding crystal, whose own prediction is simply dropped.  Its
contribution to a loss must be masked by the caller (`PaddedBatch.num_real`); with zero loss it contributes exactly zero
to every parameter gradient.  Train-mode BatchNorm is the exception -- batch statistics would see the padding rows --
and is refused.
"""
from __future__ import annotations

import math
from typing import Callable, Dict, Tuple

import numpy as np
import torch

from .graph import Graph, batch as batch_graphs, bond_cosines, unbatch


def _star(dT: int) -> Tuple[int, int, int]:
    """(a, b, r) with a*b + r == dT, r < a: a bonds s->h and b bonds h->t give a*b pairs, one bond s2->h2 and r bonds
    h2->t2 give r more."""
    if dT <= 0:
        return 0, 0, 0
    a = max(1, int(math.isqrt(dT)))
    b = dT // a
    return a, b, dT - a * b


def padding_needs(dE: int, dT: int) -> Tuple[int, int]:
    """Minimum (atoms, bonds) a padding crystal needs to realise dT bond pairs (dE only matters as an upper bound)."""
    a, b, r = _star(dT)
    bonds = a + b + ((1 + r) if r else 0)
    return 8, bonds


def make_padding_crystal(dN: int, dE: int, dT: int, atom_features: int) -> Graph:
    """A crystal with exactly dN atoms, dE bonds and dT line-graph pairs (dN >= 8, dE >= padding_needs(...)[1])."""
    need_n, need_e = padding_needs(dE, dT)
    if dN < need_n or dE < need_e:
        raise ValueError(f"padding crystal needs >= {need_n} atoms and >= {need_e} bonds for {dT} pairs, got {dN}, {dE}")
    a, b, r = _star(dT)
    src, dst = [], []
    # atoms: 0 = s, 1 = h, 2 = t, 3 = s2, 4 = h2, 5 = t2, 6 -> 7 carries the bonds that must not pair with anything
    src += [0] * a + [1] * b
    dst += [1] * a + [2] * b
    if r:
        src += [3] + [4] * r
        dst += [4] + [5] * r
    free = dE - len(src)
    src += [6] * free
    dst += [7] * free
    g = Graph(np.asarray(src, dtype=np.int64), np.asarray(dst, dtype=np.int64), dN)
    g.ndata["atom_features"] = torch.zeros(dN, atom_features)
    rvec = torch.zeros(dE, 3)
    rvec[:, 0] = 2.0                                   # a harmless 2 A bond along x
    g.edata["r"] = rvec
    return g


def bucket_of(n: int, edges: Tuple[int, ...]) -> int:
    for e in edges:
        if n <= e:
            return e
    raise ValueError(f"size {n} exceeds the largest bucket {edges[-1]}")


def geometric_buckets(lo: int, hi: int, ratio: float = 1.25) -> Tuple[int, ...]:
    out, v = [], float(lo)
    while v < hi:
        out.append(int(math.ceil(v / 64) * 64))
        v *= ratio
    out.append(int(math.ceil(hi / 64) * 64))
    return tuple(sorted(set(out)))


class PaddedBatch:
    def __init__(self, g: Graph, lg: Graph, lat: torch.Tensor, num_real: int):
        self.g, self.lg, self.lat, self.num_real = g, lg, lat, num_real


def pad_batch(g: Graph, lg: Graph, lat: torch.Tensor, N_b: int, E_b: int, T_b: int) -> PaddedBatch:
    """Append one padding crystal so that the batch has exactly (N_b, E_b, T_b) atoms / bonds / bond pairs.  Host
    graphs in, host graphs out (the line graph of the padded batch is rebuilt: its edge list is the old one followed by
    the padding pairs, both destination-major)."""
    N, E, T = g.num_nodes(), g.num_edges(), lg.num_edges()
    dN, dE, dT = N_b - N, E_b - E, T_b - T
    nf = g.ndata["atom_features"].shape[1]
    pad = make_padding_crystal(dN, dE, dT, nf)
    parts = unbatch(g) + [pad]
    for p in parts:
        for k in list(p.ndata):
            if k not in ("atom_features",):
                del p.ndata[k]
    gp = batch_graphs(parts)
    lgp = gp.line_graph(shared=True)
    if lgp.num_edges() != T_b:
        raise RuntimeError(f"padding produced {lgp.num_edges()} bond pairs, wanted {T_b}")
    lgp.edata["h"] = bond_cosines(gp.edata["r"], lgp)
    latp = torch.cat([lat, torch.eye(3, dtype=lat.dtype).unsqueeze(0)], 0)
    return PaddedBatch(gp, lgp, latp, g.batch_size)


class BucketedForward:
    """`out = runner(g, lg, lat)`: pads the host batch to its bucket, copies it into the bucket's static device buffers
    and replays the CUDA graph captured for that bucket (capturing it on first use).  `fn(g, lg, lat)` is the captured
    callable -- e.g. `lambda g, lg, lat: model((g, lg, lat))` for inference, or a closure doing forward + loss + backward
    for training.  Outputs are returned as captured (static tensors): row i < num_real belongs to real crystal i."""

    def __init__(self, fn: Callable, device, n_edges, e_edges, t_edges, warmup: int = 2):
        self.fn, self.device = fn, torch.device(device)
        self.n_edges, self.e_edges, self.t_edges = tuple(n_edges), tuple(e_edges), tuple(t_edges)
        self.warmup = warmup
        self._graphs: Dict[tuple, tuple] = {}
        self._stream = torch.cuda.Stream(self.device)

    def bucket(self, g: Graph, lg: Graph) -> tuple:
        # room for the padding crystal itself: 8 atoms, and enough bonds to realise the missing pairs
        N_b = bucket_of(g.num_nodes() + 8, self.n_edges)
        T_b = bucket_of(lg.num_edges(), self.t_edges)
        need_e = padding_needs(0, T_b - lg.num_edges())[1]
        E_b = bucket_of(g.num_edges() + need_e, self.e_edges)
        return N_b, E_b, T_b

    @staticmethod
    def _copy_graph(dst: Graph, src: Graph):
        for f in dst.index._FIELDS:
            getattr(dst.index, f).copy_(getattr(src.index, f), non_blocking=True)
        # the captured launches baked in whether `in_eid` is passed: the static atom graph always passes it, the static
        # line graph never does (Graph.line_graph emits destination-sorted edges)
        if dst.index.dst_sorted and not src.index.dst_sorted:
            raise RuntimeError("BucketedForward: line graph of the batch is not destination-sorted")
        # the line-graph descriptor (parent CSR of the padded batch) has the bucket's shapes too
        if (dst.index.parent is None) != (src.index.parent is None):
            raise RuntimeError("BucketedForward: line-graph descriptor present in only one of the batches")
        for t, u in zip(dst.index.parent or (), src.index.parent or ()):
            t.copy_(u, non_blocking=True)
        dst.index.max_in_deg = src.index.max_in_deg
        dst._seg.copy_(src._seg, non_blocking=True)
        dst._bnn, dst._bne = src._bnn, src._bne
        for name, fresh in (("_bnn_dev", src._bnn), ("_eoff64", None)):
            cached = getattr(dst, name, None)
            if cached is not None:
                if fresh is None:
                    fresh = torch.zeros(src._bne.numel() + 1, dtype=torch.int64)
                    fresh[1:] = torch.cumsum(src._bne, 0)
                cached.copy_(fresh, non_blocking=True)
        for k, v in src.ndata.items():
            dst.ndata[k].copy_(v, non_blocking=True)
        for k, v in src.edata.items():
            dst.edata[k].copy_(v, non_blocking=True)

    def __call__(self, g: Graph, lg: Graph, lat: torch.Tensor):
        key = self.bucket(g, lg)
        pb = pad_batch(g, lg, lat, *key)
        full_key = key + (pb.g.batch_size,)
        entry = self._graphs.get(full_key)
        if entry is None:
            sg, slg, slat = pb.g.to(self.device), pb.lg.to(self.device), pb.lat.to(self.device)
            sg.index.dst_sorted = False            # always hand the kernels the permutation (see _copy_graph)
            self._stream.wait_stream(torch.cuda.current_stream(self.device))
            with torch.cuda.stream(self._stream):
                for _ in range(self.warmup):
                    self.fn(sg, slg, slat)
            torch.cuda.current_stream(self.device).wait_stream(self._stream)
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr, stream=self._stream):
                out = self.fn(sg, slg, slat)
            entry = (gr, sg, slg, slat, out)
            self._graphs[full_key] = entry
        gr, sg, slg, slat, out = entry
        self._copy_graph(sg, pb.g)
        self._copy_graph(slg, pb.lg)
        slat.copy_(pb.lat, non_blocking=True)
        gr.replay()
        return out, pb.num_real
