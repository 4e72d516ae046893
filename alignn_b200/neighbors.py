"""Periodic radius-graph construction on the host (crystal -> bond list with displacement vectors).

This is the input side of the hot path for real structures and for BASELINE config 4 (ALIGNN-FF on a
~1000-atom periodic supercell); the in-tree ALIGNN-FF configs use `neighbor_strategy="radius_graph"`
(`alignn/examples/sample_data_ff/config_example_atomwise.json`).  It restates the algorithm of
`alignn/graphs.py:267-364` without jarvis-tools / DGL:

  1. enumerate the periodic images needed for `cutoff (+ bond_tol)` from the reciprocal lattice lengths,
  2. distances from every atom of the home cell to every image of every atom (native scan in the library,
     `alignn_b200_radius_graph_*_host`: 1000 atoms x 27 images in tens of milliseconds),
  3. a bond u -> v for every pair with 0 < |r| <= cutoff (`atol` guards the self distance), bonds ordered by
     (u, image index, v) exactly like `torch.where` on the [N, images*N] mask,
  4. if the highest-numbered atom ended up without any bond the cutoff is increased by `cutoff_extra` and the
     search repeated (the reference tests `dgl.graph((u, v)).num_nodes() == len(atoms)`).

Both directions of a bond appear (as two separate rows, NOT adjacent: this builder emits source-major order),
multi-edges to different images and self-image bonds occur.  `radius_graph_device` / `crystal_graph_device` run the
same scan (and the index / line-graph construction) on the GPU with bit-identical results (SURVEY.md section 8f rows 2, 4).
"""
from __future__ import annotations

import math
from typing import Tuple

import numpy as np
import torch

from .graph import Graph, bond_cosines


# ---- image tables and growth rules (pure functions, shared by the host and device builders) ------------------------
def knn_image_cells(lat, cutoff: float) -> np.ndarray:
    """Cell offsets the k-NN candidate search visits (`get_all_neighbors`): meshgrid "ij" over [-m_i, m_i] with
    m_i = ceil(cutoff * |recip_i| / 2 pi) + 1, as float64 [I, 3].  The table is symmetric: cells[I-1-c] == -cells[c]."""
    recp_len = np.sqrt(((2 * math.pi * np.linalg.inv(lat).T) ** 2).sum(1))
    maxr = np.ceil(cutoff * recp_len / (2 * math.pi)) + 1
    ranges = [np.arange(-m, m + 1, dtype=np.float64) for m in maxr]
    return np.stack(np.meshgrid(*ranges, indexing="ij"), -1).reshape(-1, 3)


def radius_image_cells(lat, frac, cutoff: float, bond_tol: float = 0.5) -> np.ndarray:
    """Cell offsets the radius search visits (graphs.py:267-364): from floor(min frac) - m to ceil(max frac) + m - 1
    per axis, m = ceil((cutoff + bond_tol) |recip_i| / 2 pi), meshgrid "ij" (torch.cartesian_prod) order."""
    recp = 2 * math.pi * np.linalg.inv(lat).T
    recp_len = np.sqrt((recp ** 2).sum(1))
    maxr = np.ceil((cutoff + bond_tol) * recp_len / (2 * math.pi))
    nmin = np.floor(frac.min(0)) - maxr
    nmax = np.ceil(frac.max(0)) + maxr
    ranges = [np.arange(a, b, dtype=np.float64) for a, b in zip(nmin, nmax)]
    return np.stack(np.meshgrid(*ranges, indexing="ij"), -1).reshape(-1, 3)


def grow_knn_cutoff(cutoff: float, lat) -> float:
    """graphs.py:170-186: a crystal with an atom short of k candidates retries at max(|a|, |b|, |c|), or at twice the
    cutoff once it is already that long."""
    abc = np.linalg.norm(np.asarray(lat, dtype=np.float64), axis=1)
    return float(abc.max()) if cutoff < abc.max() else 2 * cutoff


def grow_radius_cutoff(cutoff: float, cutoff_extra: float) -> float:
    """graphs.py:347-350: a crystal whose last atom has no bond retries at cutoff + cutoff_extra."""
    return cutoff + cutoff_extra


def ragged_offsets(sizes) -> np.ndarray:
    """int64 [B+1] exclusive prefix of per-crystal sizes (atoms or image-table rows)."""
    out = np.zeros(len(sizes) + 1, dtype=np.int64)
    out[1:] = np.cumsum(np.asarray(sizes, dtype=np.int64))
    return out


def _checked_structures(structures, neighbor_strategy: str, max_neighbors: int):
    if neighbor_strategy not in ("k-nearest", "radius_graph"):
        raise ValueError(f"Not implemented yet: neighbor_strategy={neighbor_strategy!r}")
    if neighbor_strategy == "k-nearest" and int(max_neighbors) < 1:
        raise ValueError(f"max_neighbors must be >= 1, got {max_neighbors}")
    lats, Xs = [], []
    for lat, X in structures:
        lat = np.asarray(lat, dtype=np.float64)
        X = np.asarray(X, dtype=np.float64)
        if lat.shape != (3, 3) or not np.isfinite(lat).all() or np.linalg.matrix_rank(lat) < 3:
            raise ValueError("every lattice must be a finite, invertible 3x3 matrix")
        if X.ndim != 2 or X.shape[1] != 3 or X.shape[0] == 0 or not np.isfinite(X).all():
            raise ValueError("every structure needs at least one atom with finite [n, 3] Cartesian coordinates")
        lats.append(lat)
        Xs.append(X)
    if not lats:
        raise ValueError("no structures")
    return lats, Xs


def knn_cut_is_tied(lattice_mat, cart_coords, max_neighbors: int = 12, rtol: float = 1e-6, reach: int = 3) -> bool:
    """True when some atom's max_neighbors-th and next nearest neighbour distances (over the periodic images within
    `reach` cells) are equal to `rtol` relative.  The images x + R and x - R of an atom are always equally far, so such
    ties are common.  The k-nearest graph keeps every candidate at the k-th distance, compared exactly, so at a tie
    rounding-level changes of the cell or positions decide which images the graph keeps."""
    lat = np.asarray(lattice_mat, dtype=np.float64)
    X = np.asarray(cart_coords, dtype=np.float64)
    k = int(max_neighbors)
    r = np.arange(-reach, reach + 1)
    shifts = np.stack(np.meshgrid(r, r, r, indexing="ij"), -1).reshape(-1, 3).astype(np.float64) @ lat
    cand = (X[None, :, :] + shifts[:, None, :]).reshape(-1, 3)
    for x in X:
        d = np.linalg.norm(cand - x, axis=1)
        d = np.sort(d[d > 1e-8])
        if d.size > k and d[k] - d[k - 1] <= rtol * d[k - 1]:
            return True
    return False


def _neighbors_device(structures, neighbor_strategy: str, cutoff: float, max_neighbors: int, cutoff_extra: float,
                      device):
    """The batched device builder behind `knn_graph_device` and `crystal_graphs_device` (csrc/crystal_graph_device.cu).

    Host side: per-crystal image tables and the growth loop -- one read-back per round (per-crystal status and the
    candidate offsets at the crystal boundaries); a crystal that needs a larger cutoff gets a new table, the others keep
    theirs, and the scan reruns over the batch.  k-NN then reads back the kept count and the per-crystal bond offsets.
    Returns (u, v int32, r, images float32 [E,3] on the device, batch_num_edges, lattices, frac coords, atoms/crystal)."""
    from . import _lib
    lib = _lib.load()
    knn = neighbor_strategy == "k-nearest"
    lats, Xs = _checked_structures(structures, neighbor_strategy, max_neighbors)
    dev = torch.device(device)
    B = len(lats)
    sizes = [x.shape[0] for x in Xs]
    aoff = ragged_offsets(sizes)
    N = int(aoff[-1])
    fracs = [x @ np.linalg.inv(lat) for lat, x in zip(lats, Xs)]
    lat_host = np.ascontiguousarray(np.stack(lats))
    k = int(max_neighbors)
    atoms = torch.from_numpy(np.concatenate([np.concatenate(Xs).ravel(), np.concatenate(fracs).ravel()])).to(dev)
    X_d, frac_d = atoms[:3 * N], atoms[3 * N:]
    aoff_d = torch.from_numpy(aoff).to(dev)
    crys_d = torch.from_numpy(np.repeat(np.arange(B, dtype=np.int32), sizes)).to(dev)
    cut = [float(cutoff)] * B
    cells = [None] * B
    todo = range(B)
    offsets = torch.empty(N + 1, device=dev, dtype=torch.int32)
    status = torch.empty(B, device=dev, dtype=torch.int32)
    nb = int(lib.alignn_b200_crystal_scan_workspace_bytes(N))
    ws = torch.empty(nb, device=dev, dtype=torch.uint8)
    with torch.cuda.device(dev):
        st = _lib.stream_ptr()
        while True:
            for b in todo:
                cells[b] = knn_image_cells(lats[b], cut[b]) if knn else radius_image_cells(lats[b], fracs[b], cut[b])
            soff = ragged_offsets([c.shape[0] for c in cells])
            I = int(soff[-1])
            tables = torch.from_numpy(np.concatenate([np.concatenate([c @ lat for c, lat in zip(cells, lats)]).ravel(),
                                                      np.concatenate(cells).ravel(), np.asarray(cut)])).to(dev)
            soff_d = torch.from_numpy(soff).to(dev)
            batch = _lib.CrystalBatch(X_d.data_ptr(), tables.data_ptr(), tables[3 * I:].data_ptr(), lat_host.ctypes.data,
                                      aoff_d.data_ptr(), soff_d.data_ptr(), crys_d.data_ptr(), tables[6 * I:].data_ptr(),
                                      B, N, I, max(c.shape[0] for c in cells), 1e-8 if knn else 1e-5)
            _lib.check(lib.alignn_b200_crystal_scan_count(batch, 1 if knn else 0, offsets.data_ptr(), status.data_ptr(),
                                                          ws.data_ptr(), nb, st), "alignn_b200_crystal_scan_count")
            back = torch.cat([status, offsets[aoff_d]]).tolist()
            stat, at = back[:B], back[B:]
            todo = [b for b in range(B) if (stat[b] < k if knn else stat[b] == 0)]
            if not todo:
                break
            for b in todo:
                cut[b] = grow_knn_cutoff(cut[b], lats[b]) if knn else grow_radius_cutoff(cut[b], cutoff_extra)
        C = int(at[-1])
        if not knn:
            u, v = (torch.empty(C, device=dev, dtype=torch.int32) for _ in range(2))
            r, img = (torch.empty(C, 3, device=dev, dtype=torch.float32) for _ in range(2))
            _lib.check(lib.alignn_b200_crystal_radius_fill(batch, offsets.data_ptr(), u.data_ptr(), v.data_ptr(), r.data_ptr(),
                                                           img.data_ptr(), st), "alignn_b200_crystal_radius_fill")
            bne = [b - a for a, b in zip(at[:-1], at[1:])]
        else:
            nk = int(lib.alignn_b200_knn_graph_workspace_bytes(N, B, C))
            if nk == 0:
                raise ValueError("batch too large for int32 candidate indices")
            kws = torch.empty(nk, device=dev, dtype=torch.uint8)
            kept = torch.empty(N + 1, device=dev, dtype=torch.int32)
            _lib.check(lib.alignn_b200_knn_graph_select(batch, offsets.data_ptr(), C, k, kept.data_ptr(), kws.data_ptr(), nk, st),
                       "alignn_b200_knn_graph_select")
            R = int(kept[-1].item())
            bond_off = torch.empty(B + 1, device=dev, dtype=torch.int64)
            _lib.check(lib.alignn_b200_knn_graph_order(batch, offsets.data_ptr(), kept.data_ptr(), C, R, bond_off.data_ptr(),
                                                       kws.data_ptr(), nk, st), "alignn_b200_knn_graph_order")
            bo = bond_off.tolist()
            E = int(bo[-1])
            u, v = (torch.empty(E, device=dev, dtype=torch.int32) for _ in range(2))
            r, img = (torch.empty(E, 3, device=dev, dtype=torch.float32) for _ in range(2))
            _lib.check(lib.alignn_b200_knn_graph_emit(batch, frac_d.data_ptr(), C, R, u.data_ptr(), v.data_ptr(), r.data_ptr(),
                                                      img.data_ptr(), kws.data_ptr(), nk, st), "alignn_b200_knn_graph_emit")
            bne = [b - a for a, b in zip(bo[:-1], bo[1:])]
    return u, v, r, img, bne, lats, fracs, sizes


def knn_graph_device(lattice_mat, cart_coords, max_neighbors: int = 12, cutoff: float = 8.0, device="cuda"):
    """`knn_graph` built on the GPU: the candidate scan, shell selection, canonicalisation and bond order run as CUDA
    kernels (csrc/crystal_graph_device.cu).  Returns (u, v, r, images) as CUDA tensors with `knn_graph`'s contents and
    dtypes (int64, int64, float32 [E,3], int64 [E,3])."""
    u, v, r, img, _, _, _, _ = _neighbors_device([(lattice_mat, cart_coords)], "k-nearest", cutoff, max_neighbors, 0.0, device)
    return u.long(), v.long(), r, img.long()


def crystal_graphs_device(structures, atom_features: torch.Tensor, neighbor_strategy: str = "k-nearest",
                          cutoff: float = 8.0, max_neighbors: int = 12, cutoff_extra: float = 3.5, device="cuda"):
    """(g, lg, lat) of a batch of periodic structures, built on the GPU: what `dgl.batch` of `atom_dgl_multigraph`
    outputs (graphs.py:472-589) plus the stacked lattices give the models (`ALIGNN`, `ALIGNNAtomWise`,
    `eALIGNNAtomWise`).

    `structures`: sequence of (lattice_mat [3,3], cart_coords [n,3]); `atom_features`: [sum n, F] tensor in the same atom
    order (the caller's embedding table).  `neighbor_strategy` "k-nearest" (the reference default: `knn_graph` per
    crystal) or "radius_graph" (`radius_graph` per crystal with this `cutoff_extra`; atom_dgl_multigraph's 3.5).
    g.ndata: atom_features, V (the cell volume |a . (b x c)| on every atom), frac_coords (fp32); g.edata: r, images
    (fp32); lg = L(g) with lg.edata["h"] = bond cosines; lat [B,3,3] fp32."""
    dev = torch.device(device)
    u, v, r, img, bne, lats, fracs, sizes = _neighbors_device(structures, neighbor_strategy, cutoff, max_neighbors,
                                                              cutoff_extra, dev)
    N = sum(sizes)
    if atom_features.shape[0] != N:
        raise ValueError(f"atom_features has {atom_features.shape[0]} rows for {N} atoms")
    vol = [abs(float(np.dot(np.cross(lat[0], lat[1]), lat[2]))) for lat in lats]
    host = np.concatenate([np.repeat(np.asarray(vol), sizes), np.concatenate(fracs).ravel(), np.stack(lats).ravel()])
    host = torch.from_numpy(host.astype(np.float32)).to(dev)
    g = Graph(u, v, N, torch.tensor(sizes, dtype=torch.int64), torch.tensor(bne, dtype=torch.int64))
    g.ndata["atom_features"] = atom_features.to(dev)
    g.ndata["V"] = host[:N]
    g.ndata["frac_coords"] = host[N:4 * N].view(N, 3)
    g.edata["r"] = r
    g.edata["images"] = img
    lg = g.line_graph(shared=True)
    lg.edata["h"] = bond_cosines(r, lg)
    return g, lg, host[4 * N:].view(len(lats), 3, 3)


def radius_graph_device(lattice_mat, cart_coords, cutoff: float = 5.0, bond_tol: float = 0.5, atol: float = 1e-5,
                        cutoff_extra: float = 0.5, device="cuda"):
    """`radius_graph` with the distance scan ON THE GPU (alignn_b200_radius_graph_offsets / _fill: one warp per atom,
    double precision with the host builder's operation order): identical bonds in identical order and identical fp32
    displacement vectors, returned as CUDA tensors (u int32, v int32, r float32 [E,3], image_index int32) plus the
    [I,3] cell table -- what an MD loop needs to rebuild g and L(g) every step without leaving the device
    (alignn/ff/calculators.py:284-291 rebuilds them on the CPU)."""
    from . import _lib
    lib = _lib.load()
    dev = torch.device(device)
    lat = np.asarray(lattice_mat, dtype=np.float64)
    X = np.asarray(cart_coords, dtype=np.float64)
    n = X.shape[0]
    frac = X @ np.linalg.inv(lat)
    Xd = torch.from_numpy(np.ascontiguousarray(X)).to(dev)
    while True:
        recp = 2 * math.pi * np.linalg.inv(lat).T
        recp_len = np.sqrt((recp ** 2).sum(1))
        maxr = np.ceil((cutoff + bond_tol) * recp_len / (2 * math.pi))
        nmin = np.floor(frac.min(0)) - maxr
        nmax = np.ceil(frac.max(0)) + maxr
        ranges = [np.arange(a, b, dtype=np.float64) for a, b in zip(nmin, nmax)]
        cells = np.stack(np.meshgrid(*ranges, indexing="ij"), -1).reshape(-1, 3)
        sh = torch.from_numpy(np.ascontiguousarray(cells @ lat)).to(dev)
        off = torch.empty(n + 1, device=dev, dtype=torch.int32)
        nb = int(lib.alignn_b200_radius_graph_workspace_bytes(n))
        ws = torch.empty(max(nb, 1), device=dev, dtype=torch.uint8)
        with torch.cuda.device(dev):
            st = _lib.stream_ptr()
            _lib.check(lib.alignn_b200_radius_graph_offsets(Xd.data_ptr(), sh.data_ptr(), n, sh.shape[0], float(cutoff), float(atol),
                                                            off.data_ptr(), ws.data_ptr(), nb, st), "alignn_b200_radius_graph_offsets")
            E = int(off[-1].item())
            u, v, ci = (torch.empty(E, device=dev, dtype=torch.int32) for _ in range(3))
            r = torch.empty(E, 3, device=dev, dtype=torch.float32)
            _lib.check(lib.alignn_b200_radius_graph_fill(Xd.data_ptr(), sh.data_ptr(), n, sh.shape[0], float(cutoff), float(atol),
                                                         off.data_ptr(), u.data_ptr(), v.data_ptr(), ci.data_ptr(), r.data_ptr(), st),
                       "alignn_b200_radius_graph_fill")
        # graphs.py:347-350: the highest-numbered atom must have a bond.  Bonds are (u, c, v)-ordered, so the last bond's
        # source is the largest source; v covers the rest.
        if E and max(int(u[-1].item()), int(v.max().item())) + 1 == n:
            return u, v, r, ci, cells
        cutoff += cutoff_extra


def crystal_graph_device(lattice_mat, cart_coords, atom_features: torch.Tensor, cutoff: float = 4.0, device="cuda",
                         neighbor_strategy: str = "radius_graph", max_neighbors: int = 12):
    """(g, lg) of one periodic structure built entirely on the GPU: neighbour list, sorted-CSR index, line graph and bond
    cosines (alignn/graphs.py:267-364 or 155-264, 544, 588-589).  Same graphs, bit for bit, as
    `crystal_graph(..., neighbor_strategy, max_neighbors)` followed by `.to(device)`."""
    if neighbor_strategy == "k-nearest":
        u, v, r, _ = knn_graph_device(lattice_mat, cart_coords, max_neighbors=max_neighbors, cutoff=cutoff, device=device)
    elif neighbor_strategy == "radius_graph":
        u, v, r, _, _ = radius_graph_device(lattice_mat, cart_coords, cutoff=cutoff, device=device)
    else:
        raise ValueError(f"Not implemented yet: neighbor_strategy={neighbor_strategy!r}")
    n = int(np.asarray(cart_coords).shape[0])
    g = Graph(u, v, n)
    g.ndata["atom_features"] = atom_features.to(r.device)
    g.edata["r"] = r
    lg = g.line_graph(shared=True)
    lg.edata["h"] = bond_cosines(r, lg)
    return g, lg


def radius_graph(lattice_mat, cart_coords, cutoff: float = 5.0, bond_tol: float = 0.5, atol: float = 1e-5,
                 cutoff_extra: float = 0.5) -> Tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
    """Returns (u, v, r, images): int64 [E], int64 [E], float32 [E,3] (dst image position - src position),
    float64 [E,3] (integer cell offsets of the destination image)."""
    from . import _lib
    lib = _lib.load()
    lat = np.asarray(lattice_mat, dtype=np.float64)
    X = np.asarray(cart_coords, dtype=np.float64)
    n = X.shape[0]
    frac = X @ np.linalg.inv(lat)
    while True:
        cells = radius_image_cells(lat, frac, cutoff, bond_tol)                          # cartesian_prod order
        shifts = cells @ lat                                                             # [I, 3]
        # native scan (csrc/graph_host.cu), same double-precision arithmetic and bond order as the restatement
        Xc = np.ascontiguousarray(X)
        sh = np.ascontiguousarray(shifts)
        p = lambda a: a.ctypes.data  # noqa: E731
        cnt = int(lib.alignn_b200_radius_graph_count_host(p(Xc), p(sh), n, sh.shape[0], float(cutoff), float(atol)))
        if cnt < 0:
            raise RuntimeError("alignn_b200_radius_graph_count_host failed")
        u, v, ci = (np.empty(cnt, dtype=np.int64) for _ in range(3))
        r = np.empty((cnt, 3), dtype=np.float32)
        _lib.check(lib.alignn_b200_radius_graph_build_host(p(Xc), p(sh), n, sh.shape[0], float(cutoff), float(atol), cnt,
                                                           p(u), p(v), p(ci), p(r)), "alignn_b200_radius_graph_build_host")
        if cnt and max(int(u.max()), int(v.max())) + 1 == n:
            return u, v, r, cells[ci]
        cutoff = grow_radius_cutoff(cutoff, cutoff_extra)


def crystal_graph(lattice_mat, cart_coords, atom_features: torch.Tensor, cutoff: float = 4.0,
                  neighbor_strategy: str = "radius_graph", max_neighbors: int = 12):
    """(g, lg) for one periodic structure, laid out like `Graph.atom_dgl_multigraph` output (graphs.py:472-592):
    g.ndata['atom_features'], g.edata['r'], lg = L(g) with lg.edata['h'] = bond cosines.
    `neighbor_strategy` is the reference's switch (graphs.py:497-536): "radius_graph" or "k-nearest"."""
    if neighbor_strategy == "k-nearest":
        u, v, r, _ = knn_graph(lattice_mat, cart_coords, max_neighbors=max_neighbors, cutoff=cutoff)
    elif neighbor_strategy == "radius_graph":
        u, v, r, _ = radius_graph(lattice_mat, cart_coords, cutoff=cutoff)
    else:
        raise ValueError(f"Not implemented yet: neighbor_strategy={neighbor_strategy!r}")
    g = Graph(u, v, int(np.asarray(cart_coords).shape[0]))
    g.ndata["atom_features"] = atom_features
    g.edata["r"] = torch.from_numpy(r)
    lg = g.line_graph(shared=True)
    lg.edata["h"] = bond_cosines(g.edata["r"], lg)
    return g, lg


def diamond_supercell(reps: int = 5, a: float = 5.431, jitter: float = 0.0, seed: int = 0):
    """Diamond-cubic silicon supercell, 8 * reps^3 atoms (reps = 5 -> 1000 atoms: BASELINE config 4 shape).
    Returns (lattice_mat [3,3], cart_coords [N,3])."""
    basis = np.array([[0, 0, 0], [0, .5, .5], [.5, 0, .5], [.5, .5, 0],
                      [.25, .25, .25], [.25, .75, .75], [.75, .25, .75], [.75, .75, .25]])
    cells = np.stack(np.meshgrid(*[np.arange(reps)] * 3, indexing="ij"), -1).reshape(-1, 3)
    frac = (cells[:, None, :] + basis[None, :, :]).reshape(-1, 3) / reps
    lat = np.eye(3) * a * reps
    X = frac @ lat
    if jitter:
        X = X + np.random.default_rng(seed).normal(scale=jitter, size=X.shape)
    return lat, X


def _all_neighbors(lat, X, cutoff, atol=1e-8):
    """Every (u, v, image, distance) with 0 < |x_v + image@lat - x_u| <= cutoff (what jarvis'
    `Atoms.get_all_neighbors(r=cutoff)` lists per site), from the native scan."""
    from . import _lib
    lib = _lib.load()
    n = X.shape[0]
    cells = knn_image_cells(lat, cutoff)
    sh = np.ascontiguousarray(cells @ lat)
    Xc = np.ascontiguousarray(X)
    p = lambda a: a.ctypes.data  # noqa: E731
    cnt = int(lib.alignn_b200_radius_graph_count_host(p(Xc), p(sh), n, sh.shape[0], float(cutoff), float(atol)))
    u, v, ci = (np.empty(cnt, dtype=np.int64) for _ in range(3))
    r = np.empty((cnt, 3), dtype=np.float32)
    _lib.check(lib.alignn_b200_radius_graph_build_host(p(Xc), p(sh), n, sh.shape[0], float(cutoff), float(atol), cnt,
                                                       p(u), p(v), p(ci), p(r)), "alignn_b200_radius_graph_build_host")
    img = cells[ci].astype(np.int64)
    d = (X[v] + img @ lat) - X[u]
    return u, v, img, np.sqrt((d ** 2).sum(1))


def knn_graph(lattice_mat, cart_coords, max_neighbors: int = 12, cutoff: float = 8.0):
    """k-nearest-neighbour crystal graph with shell completion, made undirected the reference's way
    (`nearest_neighbor_edges` + `build_undirected_edgedata`, alignn/graphs.py:155-264, `use_canonize=True`).

    Per atom: neighbours within `cutoff` sorted by distance; everything out to the distance of the k-th one is kept
    (whole shells, so the degree is >= k); if some atom has fewer than k neighbours the cutoff grows to max(a, b, c)
    or doubles (:170-186).  Each kept pair is canonised to (min id, max id, image of the second atom relative to the
    first) and every canonical bond emits BOTH directions adjacently, (u, v, d) then (v, u, -d) (:253-257).
    Self-image bonds appear with +image and -image as two canonical bonds, as in the reference.
    Bond order: canonical pairs in order of first encounter (atoms ascending, neighbours by (distance, v, image)),
    images of one pair in lexicographic order -- the reference's order inside a pair is Python-set iteration order
    and not reproducible; no model output depends on it.
    Returns (u, v, r[float32], images[int64]).
    """
    lat = np.asarray(lattice_mat, dtype=np.float64)
    X = np.asarray(cart_coords, dtype=np.float64)
    n = X.shape[0]
    while True:
        u, v, img, dist = _all_neighbors(lat, X, cutoff)
        counts = np.bincount(u, minlength=n)
        if counts.min() >= max_neighbors:
            break
        cutoff = grow_knn_cutoff(cutoff, lat)
    order = np.lexsort((img[:, 2], img[:, 1], img[:, 0], v, dist, u))     # by u, then distance, then (v, image)
    u, v, img, dist = u[order], v[order], img[order], dist[order]
    start = np.concatenate([[0], np.cumsum(counts)])
    kth = dist[start[:-1] + max_neighbors - 1]                             # distance of the k-th neighbour per atom
    keep = dist <= kth[u]
    u, v, img = u[keep], v[keep], img[keep]
    swap = v < u                                                           # canonize_edge (:127-152)
    cu, cv = np.where(swap, v, u), np.where(swap, u, v)
    cimg = np.where(swap[:, None], -img, img)
    pairs = {}
    for a, b, im in zip(cu.tolist(), cv.tolist(), map(tuple, cimg.tolist())):
        pairs.setdefault((a, b), set()).add(im)
    uu, vv, rr, ii = [], [], [], []
    frac = X @ np.linalg.inv(lat)
    for (a, b), ims in pairs.items():
        for im in sorted(ims):
            d = (frac[b] + np.asarray(im, dtype=np.float64) - frac[a]) @ lat   # :245-249
            uu += [a, b]
            vv += [b, a]
            rr += [d, -d]
            ii += [im, im]
    return (np.asarray(uu, dtype=np.int64), np.asarray(vv, dtype=np.int64), np.asarray(rr, dtype=np.float32),
            np.asarray(ii, dtype=np.int64).reshape(-1, 3))
