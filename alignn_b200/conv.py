"""EdgeGatedGraphConv / ALIGNNConv on the H100 kernels.

Mirrors the reference operator interface for this path:
    EdgeGatedGraphConv(input_features, output_features, residual=True).forward(g, node_feats, edge_feats) -> (x, y)
    ALIGNNConv(in_features, out_features).forward(g, lg, x, y, z) -> (x, y, z)
(alignn/models/alignn.py:48-167; LayerNorm twins alignn/models/alignn_atomwise.py:127-246),
with identical attribute / state_dict names (SURVEY.md App. A) so reference checkpoints load
with `load_state_dict`.

The four node Linear layers run as ONE [Nn,d]x[d,4d] GEMM and the edge gate as one [Ne,d]x[d,d]
GEMM, both on the wgmma bf16x3 tensor-core kernel (csrc/gemm_tc.cu); everything else of the layer --
u_add_v, sigmoid, both update_all reductions, the division, both norms, SiLU, residuals -- is a single
fused CUDA kernel forward and two backward (csrc/egc_kernels.cu); data gradients reuse the GEMM kernel with
transposed weight images, weight gradients run on the split-K tensor-core kernel (csrc/wgrad_tc.cu).  All of
it is reached through the C ABI (include/alignn_b200.h).
"""
from __future__ import annotations

import torch
from torch import nn
from torch.autograd.function import once_differentiable

from . import ops
from .graph import as_graph
from .ops import NORM_AFFINE, NORM_LAYER, NORM_STATS

GATE_EPS = 1e-6   # alignn.py:109


class second_order:
    """Context manager for code that differentiates through its own backward -- force / stress training,
    `torch.autograd.grad(..., create_graph=True)` at alignn/models/alignn_atomwise.py:530-539 (SURVEY.md section 8b
    "autograd contract").  BatchNorm convs (and the embedding MLPs, alignn.mlp_forward) then run as compositions of
    differentiable torch operators; LayerNorm convs keep the CUDA Function, whose backward is differentiable once more
    (_EdgeGatedConvBackwardFn)."""
    active = False

    def __enter__(self):
        self._prev = second_order.active
        second_order.active = True

    def __exit__(self, *exc):
        second_order.active = self._prev


def _torch_ops_forward(mod, ix, x, y, need_edge_out: bool):
    """alignn/models/alignn.py:98-127 with plain torch operators (same summation structure as the reference's DGL
    path: gather, multiply, index_add); differentiable to any order."""
    F = torch.nn.functional
    src, dst = ix.src.long(), ix.dst.long()
    e_src, e_dst = mod.src_gate(x), mod.dst_gate(x)
    m = e_src[src] + e_dst[dst] + mod.edge_gate(y)
    sigma = torch.sigmoid(m)
    Bh = mod.dst_update(x)
    zeros = torch.zeros_like(Bh)
    sum_sigma_h = zeros.index_add(0, dst, Bh[src] * sigma)
    sum_sigma = zeros.index_add(0, dst, sigma)
    h = sum_sigma_h / (sum_sigma + GATE_EPS)
    xn = F.silu(mod.bn_nodes(mod.src_update(x) + h))
    x_out = x + xn if mod.residual else xn
    y_out = None
    if need_edge_out or isinstance(mod.bn_edges, nn.BatchNorm1d):
        yn = F.silu(mod.bn_edges(m))            # (BatchNorm: evaluated even when dead, for the running statistics)
        y_out = (y + yn if mod.residual else yn) if need_edge_out else None
    return x_out, y_out


class _Cfg:
    """Per-call, non-tensor configuration of the fused stage."""
    __slots__ = ("index", "norm_nodes", "norm_edges", "residual", "need_edge_out", "ln_eps",
                 "bn_nodes", "bn_edges", "n_aux", "e_aux", "images")


def _bn_eval_vectors(bn: nn.BatchNorm1d):
    """scale/shift/mean/rstd of an eval-mode BatchNorm1d, cached on the module by tensor versions."""
    key = tuple((t._version, t.data_ptr()) for t in (bn.weight, bn.bias, bn.running_mean, bn.running_var))
    cache = getattr(bn, "_alignn_b200_eval", None)
    if cache is not None and cache[0] == key:
        return cache[1]
    with torch.no_grad():
        rstd = torch.rsqrt(bn.running_var + bn.eps)
        scale = bn.weight * rstd
        shift = bn.bias - bn.running_mean * scale
        vecs = (scale.contiguous(), shift.contiguous(), bn.running_mean.detach().clone(), rstd.contiguous())
    bn._alignn_b200_eval = (key, vecs)
    return vecs


class _EdgeGatedConvFn(torch.autograd.Function):
    """x, y, 5 Linear (weight, bias) pairs, 2 norm (weight, bias) pairs -> (x_out, y_out)."""

    @staticmethod
    def forward(ctx, cfg: _Cfg, x, y, W_sg, b_sg, W_dg, b_dg, W_eg, b_eg, W_su, b_su, W_du, b_du, nw, nb, ew, eb):
        ix = cfg.index
        d = x.shape[1]
        # inputs that are train-mode BatchNorm outputs: their gradients (gx, gy below) also leave those BatchNorms'
        # backward statistics (ops.bn_fold_take)
        ctx.fold_in = (None, None)
        if cfg.norm_nodes != NORM_LAYER:
            ctx.fold_in = (ops.bn_fold_take(x, d), ops.bn_fold_take(y, d))
        x = x.contiguous()
        y = y.contiguous()
        ops.require_cuda(x, y)
        Nn, d = x.shape
        Ne = y.shape[0]
        needs_grad = any(ctx.needs_input_grad)
        stats = cfg.norm_nodes == NORM_STATS
        n_aux = e_aux = None
        if cfg.norm_nodes == NORM_AFFINE:
            n_aux = _bn_eval_vectors(cfg.bn_nodes)
            e_aux = _bn_eval_vectors(cfg.bn_edges)
            n_w, n_b, e_w, e_b = n_aux[0], n_aux[1], e_aux[0], e_aux[1]
        elif stats:
            n_w = n_b = e_w = e_b = None
        else:
            n_w, n_b, e_w, e_b = nw.contiguous(), nb.contiguous(), ew.contiguous(), eb.contiguous()
        bnn, bne = cfg.bn_nodes, cfg.bn_edges

        # node projections P = [e_src | Bh | e_dst | src_update] (include/alignn_b200.h); the edge-gate bias rides in
        # the e_dst block, so the gate needs no bias of its own
        img = cfg.images            # operand images, refreshed by one table-driven launch per step (ops.ImageTable)
        P = ops.gemm_gather(x, img.images["cat"], img.vectors["bcat"])
        # pass 1 over the edge rows (csrc/gemm_tc.cu): m = e_src[src] + e_dst[dst] + edge_gate(y) on wgmma,
        # the P rows gathered in the epilogue, BatchNorm batch statistics of m on the way out
        e_part = None
        if Ne > 0:
            res = ops.gemm_gather(y, img.images["eg"], None, add0=P[:, 0:d], idx0=ix.src,
                                  add1=P[:, 2 * d:3 * d], idx1=ix.dst, stats=stats)
            M, e_part = res if stats else (res, None)
        else:
            M = y.new_empty((0, d))
        norm_e = cfg.norm_edges
        if stats and Ne > 0:
            # statistics (and running buffers) are updated even when the edge output is dead
            # (SURVEY.md App. D-11): the reference always evaluates bn_edges(m).
            track_e = bne.track_running_stats and bne.running_mean is not None
            e_aux = ops.bn_finalize(e_part, 0, Ne, ew, eb, bne.eps, _momentum(bne),
                                    bne.running_mean if track_e else None, bne.running_var if track_e else None)
            e_w, e_b = e_aux[0], e_aux[1]
        if stats:
            norm_e = NORM_AFFINE
        # pass 2 (csrc/egc_kernels.cu): sigmoid, both segment reductions by sorted-CSR index, y_out = y + silu(norm(m))
        out = ops.egc_forward(ix, x, y, M, P, n_w, n_b, e_w, e_b, norm_nodes=cfg.norm_nodes, norm_edges=norm_e,
                              residual=cfg.residual, save=needs_grad, need_edge_out=cfg.need_edge_out and Ne > 0,
                              gate_eps=GATE_EPS, ln_eps=cfg.ln_eps, gate_is_m=True)
        x_out, y_out = out["x_out"], out["y_out"]
        if stats:
            track_n = bnn.track_running_stats and bnn.running_mean is not None
            n_aux = ops.bn_finalize(out["partials"], 1, Nn, nw, nb, bnn.eps, _momentum(bnn),
                                    bnn.running_mean if track_n else None, bnn.running_var if track_n else None)
            x_out = ops.affine_silu_residual(out["XP"], x if cfg.residual else None, n_aux[0], n_aux[1])
            ctx.fold_out = (ops.bn_fold_offer(x_out, out["XP"], *n_aux),
                            ops.bn_fold_offer(y_out, out["M"], *e_aux) if y_out is not None else None)
            for bn in (bnn, bne):
                if bn.track_running_stats and bn.num_batches_tracked is not None:
                    bn.num_batches_tracked.add_(1)
        if needs_grad:
            ctx.cfg = cfg
            cfg.n_aux, cfg.e_aux = n_aux, e_aux
            ctx.save_for_backward(x, y, P, out["M"], out["XP"], out["S"], out["H"], nw, nb, ew, eb)
            ctx.weights = (W_sg, W_dg, W_eg, W_su, W_du)          # identities only: ops.WgradQueue maps them to destinations
            ctx.biases = (b_sg, b_dg, b_eg, b_su, b_du)
        ctx.y_dead = y_out is None
        if y_out is None:       # dead edge output (or an edgeless graph): hand autograd an empty placeholder
            y_out = x.new_empty((0, d))
            ctx.mark_non_differentiable(y_out)
        return x_out, y_out

    @staticmethod
    def backward(ctx, gx_out, gy_out):
        if torch.is_grad_enabled() and ctx.cfg.norm_nodes == NORM_LAYER:
            # create_graph=True (force training): the first backward becomes a differentiable function of x, y, the
            # incoming gradients and the parameters, whose own backward runs on the library kernels
            x, y, P, M, XP, S, H, nw, nb, ew, eb = ctx.saved_tensors
            W_sg, W_dg, W_eg, W_su, W_du = ctx.weights
            b_sg, b_dg, b_eg, b_su, b_du = ctx.biases
            gy_live = None if (ctx.y_dead or gy_out is None) else gy_out
            grads = _EdgeGatedConvBackwardFn.apply(ctx, (P, M, XP, S, H), x, y, gx_out, gy_live, W_sg, b_sg, W_dg, b_dg,
                                                   W_eg, b_eg, W_su, b_su, W_du, b_du, nw, nb, ew, eb)
            return (None,) + tuple(grads)
        return _first_backward_once(ctx, gx_out, gy_out)


def _first_backward(ctx, gx_out, gy_out, saved=None, create_graph=False):
    """The conv's backward on the library kernels.  Returns the 17 gradients of _EdgeGatedConvFn.forward's inputs;
    with create_graph=True also (GP, GM, GSh) for the double backward, and weight gradients are never deferred."""
    cfg = ctx.cfg
    x, y, P, M, XP, S, H, nw, nb, ew, eb = saved if saved is not None else ctx.saved_tensors
    img_catT, img_egT = cfg.images.images["catT"], cfg.images.images["egT"]
    d = x.shape[1]
    gx_out = gx_out.contiguous()
    gy_out = None if (ctx.y_dead or gy_out is None) else gy_out.contiguous()
    if cfg.norm_nodes == NORM_LAYER:
        n = dict(w=nw.contiguous(), b=nb.contiguous())
        e = dict(w=ew.contiguous(), b=eb.contiguous())
    else:
        sc, sh, mu, rs = cfg.n_aux
        n = dict(w=sc, b=sh, mean=mu, rstd=rs)
        e = {}
        if cfg.e_aux is not None:
            sc, sh, mu, rs = cfg.e_aux
            e = dict(w=sc, b=sh, mean=mu, rstd=rs)
        if cfg.norm_nodes == NORM_STATS:
            # from the partials the consumer's data-gradient GEMM attached to gx_out / gy_out, else a reduction pass
            fn, fe = ctx.fold_out
            n["c1"], n["c2"] = ops.bn_backward_stats(fn, gx_out, XP, n["w"], n["b"], n["mean"], n["rstd"])
            if gy_out is not None:
                e["c1"], e["c2"] = ops.bn_backward_stats(fe, gy_out, M, e["w"], e["b"], e["mean"], e["rstd"])
            elif fe is not None:
                fe.release()
    # Parameter gradients are off the critical path of backward.  With a queue installed (FlatGradAllReducer.deferring())
    # the five weight-gradient GEMMs and the nine bias / norm-parameter reductions of this conv are only registered
    # here and computed by two batched launches at the end of backward, straight into the flat gradient buffer.
    params = not ops.input_grads_only.active                # a forces-only backward discards every parameter gradient
    queue = None if create_graph else ops.WgradQueue.current
    W_sg, W_dg, W_eg, W_su, W_du = ctx.weights
    b_sg, b_dg, b_eg, b_su, b_du = ctx.biases
    vec_needed = [b_sg, b_dg, b_eg, b_su, b_du, nw, nb] + ([ew, eb] if gy_out is not None else [])
    deferred = params and queue is not None and ops.wgrad_supported(d, d) and queue.wants(W_sg, W_du, W_dg, W_su, W_eg) \
        and queue.wants_vecs(*vec_needed)
    res = ops.egc_backward(cfg.index, P, M, XP, S, H, gx_out, gy_out, n, e, reduce=params and not deferred,
                           norm_nodes=cfg.norm_nodes, norm_edges=cfg.norm_edges,
                           gate_eps=GATE_EPS, ln_eps=cfg.ln_eps, keep_gsh=create_graph)
    GM, GP, vd, vs = res[:4]
    # GEMM halves of the backward on the tensor cores: data gradients (gemm_tc.cu, transposed weight images,
    # residual added in the epilogue) and weight gradients (wgrad_tc.cu, split-K over rows)
    need = ctx.needs_input_grad
    gx = gy = None
    fold_x, fold_y = (None, None) if create_graph else ctx.fold_in
    ctx.fold_in = (None, None)          # used once: a retained graph's next backward falls back (ops.BNFold)
    if need[1]:
        gx, part = ops.dgrad_gemm(fold_x, GP, img_catT, add0=gx_out if cfg.residual else None)
        ops.bn_fold_attach(gx, fold_x, part)
    if deferred:
        for j, W in enumerate((W_sg, W_du, W_dg, W_su)):           # column blocks of GP: e_src | Bh | e_dst | src_update
            queue.add(GP[:, j * d:(j + 1) * d], x, W)
        queue.add(GM, y, W_eg)
        # partial rows of the destination pass: {g_ew, g_eb, g_nw, g_nb, gb_su, gb_dg}; of the source pass: {gb_sg, gb_du}
        if gy_out is not None:
            queue.add_vec(vd, 0, d, ew)
            queue.add_vec(vd, 1, d, eb)
        queue.add_vec(vd, 2, d, nw)
        queue.add_vec(vd, 3, d, nb)
        queue.add_vec(vd, 4, d, b_su)
        queue.add_vec(vd, 5, d, b_dg)
        queue.add_vec(vd, 5, d, b_eg)                            # sum_e gm_e == sum_v sum_{e->v} gm_e
        queue.add_vec(vs, 0, d, b_sg)
        queue.add_vec(vs, 1, d, b_du)
    elif params:
        gWcat = ops.wgrad(GP, x, groups=4)      # [4d, d] rows: src_gate | dst_update | dst_gate | src_update
        gW_eg = ops.wgrad(GM, y, groups=1)
    if need[2]:
        res_y = gy_out if (gy_out is not None and cfg.residual) else None
        gy, part = ops.dgrad_gemm(fold_y, GM, img_egT, add0=res_y)
        ops.bn_fold_attach(gy, fold_y, part)
    if not params or deferred:
        grads = (None, gx, gy) + (None,) * 14
        return (grads, GP, GM, res[4]) if create_graph else grads
    gW_sg, gW_du, gW_dg, gW_su = gWcat[0:d], gWcat[d:2 * d], gWcat[2 * d:3 * d], gWcat[3 * d:4 * d]
    gb_sg, gb_du = vs[0], vs[1]
    gb_su, gb_dg = vd[4], vd[5]
    gb_eg = gb_dg                           # sum_e gm_e == sum_v sum_{e->v} gm_e
    g_nw, g_nb = vd[2], vd[3]
    g_ew, g_eb = (vd[0], vd[1]) if gy_out is not None else (None, None)
    grads = (None, gx, gy, gW_sg, gb_sg, gW_dg, gb_dg, gW_eg, gb_eg, gW_su, gb_su, gW_du, gb_du, g_nw, g_nb, g_ew, g_eb)
    return (grads, GP, GM, res[4]) if create_graph else grads


# today's first-order backward: no grad mode inside, and a create_graph backward through it (BatchNorm convs) fails
# loudly when differentiated again
_first_backward_once = once_differentiable(_first_backward)


class _EdgeGatedConvBackwardFn(torch.autograd.Function):
    """The first backward of a LayerNorm conv as a function of (x, y, gx_out, gy_out, parameters) -> (gx, gy, parameter
    gradients).  Its forward is the first backward on the library kernels; its backward (the double backward) projects
    the cotangents of gx, gy through the weight images, runs alignn_b200_egc_backward_vjp, and finishes through the
    forward GEMMs.  The parameter gradients it returns are values only: differentiating through them raises."""

    @staticmethod
    def forward(ctx, fctx, saved, x, y, gx_out, gy_out, W_sg, b_sg, W_dg, b_dg, W_eg, b_eg, W_su, b_su, W_du, b_du,
                nw, nb, ew, eb):
        ctx.set_materialize_grads(False)
        P, M, XP, S, H = saved
        grads, GP, GM, GSh = _first_backward(fctx, gx_out, gy_out, (x, y) + saved + (nw, nb, ew, eb), create_graph=True)
        ctx.cfg, ctx.residual = fctx.cfg, fctx.cfg.residual
        ctx.save_for_backward(x, y, P, M, XP, S, H, nw, nb, ew, eb, gx_out.contiguous(),
                              None if gy_out is None else gy_out.contiguous(), GP, GM, GSh)
        return grads[1:]

    @staticmethod
    @once_differentiable
    def backward(ctx, gx_bar, gy_bar, *gparam_bar):
        if any(g is not None for g in gparam_bar):
            raise NotImplementedError(
                "alignn_b200.EdgeGatedGraphConv: the parameter gradients of a create_graph=True backward cannot be "
                "differentiated again (the double backward covers the input gradients gx, gy); wrap the first "
                "autograd.grad in alignn_b200.ops.input_grads_only() if only input gradients are needed")
        cfg = ctx.cfg
        x, y, P, M, XP, S, H, nw, nb, ew, eb, gx_out, gy_out, GP, GM, GSh = ctx.saved_tensors
        img = cfg.images.images
        d = x.shape[1]
        Ne = y.shape[0]
        gx_bar = torch.zeros_like(x) if gx_bar is None else gx_bar.contiguous()
        gy_bar = None if (gy_bar is None or Ne == 0) else gy_bar.contiguous()
        # through the GEMMs of the first backward: gx = GP Wcat (+ gx_out), gy = GM W_eg (+ gy_out)
        GPbar = ops.gemm_gather(gx_bar, img["cat"])
        GMbar = ops.gemm_gather(gy_bar, img["eg"]) if gy_bar is not None else None
        Pbar, Mbar, gxo_bar, gyo_bar, vd, vs = ops.egc_backward_vjp(
            cfg.index, P, M, XP, S, H, gx_out, gy_out, GSh, GPbar, GMbar,
            gx_bar if ctx.residual else None, gy_bar if (ctx.residual and gy_out is not None) else None,
            nw.contiguous(), nb.contiguous(), ew.contiguous(), eb.contiguous(), gate_eps=GATE_EPS, ln_eps=cfg.ln_eps)
        # through the forward GEMMs: P = x Wcat^T + bcat, M = y W_eg^T + e_src[src] + e_dst[dst]
        need = ctx.needs_input_grad
        x_bar = ops.gemm_gather(Pbar, img["catT"]) if need[2] else None
        y_bar = ops.gemm_gather(Mbar, img["egT"]) if need[3] else None
        if ops.input_grads_only.active:
            return (None, None, x_bar, y_bar, gxo_bar, gyo_bar) + (None,) * 14
        gWcat = ops.wgrad(Pbar, x, groups=4)
        gWcat.add_(ops.wgrad(GP, gx_bar, groups=4))
        gW_eg = ops.wgrad(Mbar, y, groups=1)
        if gy_bar is not None:
            gW_eg.add_(ops.wgrad(GM, gy_bar, groups=1))
        gW_sg, gW_du, gW_dg, gW_su = gWcat[0:d], gWcat[d:2 * d], gWcat[2 * d:3 * d], gWcat[3 * d:4 * d]
        gb_sg, gb_du = vs[0], vs[1]
        gb_su, gb_dg = vd[4], vd[5]
        gb_eg = gb_dg                           # sum_e Mbar_e == sum_v sum_{e->v} Mbar_e
        g_nw, g_nb = vd[2], vd[3]
        g_ew, g_eb = (vd[0], vd[1]) if gy_out is not None else (None, None)
        return (None, None, x_bar, y_bar, gxo_bar, gyo_bar, gW_sg, gb_sg, gW_dg, gb_dg, gW_eg, gb_eg, gW_su, gb_su,
                gW_du, gb_du, g_nw, g_nb, g_ew, g_eb)


def _momentum(bn: nn.BatchNorm1d) -> float:
    if bn.momentum is None:
        raise NotImplementedError("BatchNorm1d(momentum=None) (cumulative average) is not supported")
    return float(bn.momentum)


class EdgeGatedGraphConvBase(nn.Module):
    """Edge-gated graph convolution (arXiv:1711.07553) -- shared implementation.

    Parameter names follow alignn/models/alignn.py:68-76.  `norm` selects BatchNorm1d
    (alignn.py) or LayerNorm (alignn_atomwise.py) for bn_nodes / bn_edges.
    """

    def __init__(self, input_features: int, output_features: int, residual: bool = True, norm: str = "batchnorm"):
        super().__init__()
        if input_features != output_features:
            raise NotImplementedError(
                "alignn_b200 kernels need input_features == output_features (the reference only ever "
                "instantiates square layers; its residual path requires it, alignn.py:125-127)")
        self.residual = residual
        self.norm_kind = norm
        mk = (lambda: nn.BatchNorm1d(output_features)) if norm == "batchnorm" else (lambda: nn.LayerNorm(output_features))
        self.src_gate = nn.Linear(input_features, output_features)
        self.dst_gate = nn.Linear(input_features, output_features)
        self.edge_gate = nn.Linear(input_features, output_features)
        self.bn_edges = mk()
        self.src_update = nn.Linear(input_features, output_features)
        self.dst_update = nn.Linear(input_features, output_features)
        self.bn_nodes = mk()

    def image_table(self) -> "ops.ImageTable":
        """Operand images of the five Linear layers: node projections stacked [src_gate; dst_update; dst_gate;
        src_update] (P column order of include/alignn_b200.h), their transposes for the data gradient, the edge gate and
        its transpose, and the stacked bias with the edge-gate bias folded into the dst_gate block."""
        dev = self.src_gate.weight.device
        tbl = getattr(self, "_alignn_b200_images", None)
        if tbl is not None and tbl.device == dev:
            return tbl
        d = self.src_gate.out_features
        order = (self.src_gate, self.dst_update, self.dst_gate, self.src_update)
        tbl = ops.ImageTable()
        tbl.device = dev
        tbl.add_image("cat", 4 * d, d, [(m.weight, False, i * d, 0) for i, m in enumerate(order)], dev)
        tbl.add_image("catT", d, 4 * d, [(m.weight, True, 0, i * d) for i, m in enumerate(order)], dev)
        tbl.add_image("eg", d, d, [(self.edge_gate.weight, False, 0, 0)], dev)
        tbl.add_image("egT", d, d, [(self.edge_gate.weight, True, 0, 0)], dev)
        tbl.add_vector("bcat", 4 * d, [(0, self.src_gate.bias, None), (d, self.dst_update.bias, None),
                                       (2 * d, self.dst_gate.bias, self.edge_gate.bias), (3 * d, self.src_update.bias, None)], dev)
        object.__setattr__(self, "_alignn_b200_images", tbl)
        return tbl

    def forward(self, g, node_feats: torch.Tensor, edge_feats: torch.Tensor, _need_edge_out: bool = True):
        g = as_graph(g)
        if node_feats.dtype != torch.float32 or edge_feats.dtype != torch.float32:
            raise RuntimeError("alignn_b200.EdgeGatedGraphConv is fp32-only (the reference default dtype, "
                               f"alignn/config.py:163); got {node_feats.dtype}")
        if not node_feats.is_cuda:
            raise RuntimeError("alignn_b200.EdgeGatedGraphConv has no CPU path: move the model, features and graphs "
                               "to a CUDA device.")
        if g.device != node_feats.device:
            raise RuntimeError(f"graph is on {g.device} but features are on {node_feats.device}; call g.to(device)")
        if node_feats.shape[0] != g.num_nodes() or edge_feats.shape[0] != g.num_edges():
            raise RuntimeError("feature rows do not match the graph: "
                               f"{tuple(node_feats.shape)} nodes vs {g.num_nodes()}, "
                               f"{tuple(edge_feats.shape)} edges vs {g.num_edges()}")
        if second_order.active and self.norm_kind != "layernorm":
            # BatchNorm convs have no double backward on the kernels: differentiable torch operators instead
            return _torch_ops_forward(self, g.index, node_feats, edge_feats, _need_edge_out)
        cfg = _Cfg()
        cfg.index = g.index
        cfg.residual = bool(self.residual)
        cfg.need_edge_out = bool(_need_edge_out)
        cfg.bn_nodes, cfg.bn_edges = self.bn_nodes, self.bn_edges
        cfg.n_aux = cfg.e_aux = None
        cfg.images = self.image_table()
        cfg.images.refresh()          # no launch if the model-level table already refreshed this step
        if self.norm_kind == "layernorm":
            cfg.norm_nodes = cfg.norm_edges = NORM_LAYER
            cfg.ln_eps = float(self.bn_nodes.eps)
        else:
            use_batch_stats = self.training or not self.bn_nodes.track_running_stats
            cfg.norm_nodes = cfg.norm_edges = NORM_STATS if use_batch_stats else NORM_AFFINE
            cfg.ln_eps = 1e-5
        with torch.cuda.device(node_feats.device):     # kernels launch on the tensors' device, whatever the current one is
            x, y = self._run_kernels(cfg, node_feats, edge_feats)
        return x, (y if _need_edge_out else None)

    def _run_kernels(self, cfg, node_feats, edge_feats):
        # contiguous HERE, outside the Function: its saved x, y must be the autograd inputs themselves, or the double
        # backward would see a detached copy and drop the x / y terms
        return _EdgeGatedConvFn.apply(
            cfg, node_feats.contiguous(), edge_feats.contiguous(),
            self.src_gate.weight, self.src_gate.bias, self.dst_gate.weight, self.dst_gate.bias,
            self.edge_gate.weight, self.edge_gate.bias, self.src_update.weight, self.src_update.bias,
            self.dst_update.weight, self.dst_update.bias,
            self.bn_nodes.weight, self.bn_nodes.bias, self.bn_edges.weight, self.bn_edges.bias)


class ALIGNNConvBase(nn.Module):
    """Line graph update (alignn/models/alignn.py:132-167): node_update on g, edge_update on L(g)."""

    conv_cls = None  # set by subclasses

    def __init__(self, in_features: int, out_features: int):
        super().__init__()
        self.node_update = self.conv_cls(in_features, out_features)
        self.edge_update = self.conv_cls(out_features, out_features)

    def forward(self, g, lg, x, y, z, _need_z_out: bool = True):
        g, lg = as_graph(g), as_graph(lg)
        x, m = self.node_update(g, x, y)
        # L(g) node i == g edge i: bond features m are the node features of the line graph
        y, z = self.edge_update(lg, m, z, _need_edge_out=_need_z_out)
        return x, y, z
