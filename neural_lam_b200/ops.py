"""Thin PyTorch-side wrappers over the C ABI (include/nlam_b200.h): tensor checks, strides,
stream plumbing and the autograd glue.  PyTorch is used for device memory, streams and
autograd bookkeeping only; all compute on the forward path is in libnlam_b200.so.
"""
import ctypes

import torch

from . import _lib
from ._lib import NlamMlp, NlamRowSrc


class profile_launches:
    """``with profile_launches() as prof: ...`` — collects (kernel name, µs, algorithmic bytes) of every kernel the
    library launches inside the block (``nlam_profile_*``: CUDA events around each launch; eager mode only, not inside
    a CUDA-graph capture).  ``prof.rows`` is filled on exit."""

    def __enter__(self):
        self.rows = []
        _lib.lib().nlam_profile_enable(1)
        return self

    def __exit__(self, *exc):
        L = _lib.lib()
        torch.cuda.synchronize()
        name = ctypes.create_string_buffer(96)
        ms, nb = ctypes.c_float(), ctypes.c_double()
        for i in range(L.nlam_profile_count()):
            _lib.check(L.nlam_profile_get(i, name, 96, ctypes.byref(ms), ctypes.byref(nb)))
            self.rows.append((name.value.decode(), ms.value * 1e3, nb.value))
        L.nlam_profile_enable(0)
        return False

    def names(self):
        return [r[0] for r in self.rows]


def _require_cuda(*tensors):
    for t in tensors:
        if t is None:
            continue
        if not t.is_cuda:
            raise RuntimeError(
                "neural_lam_b200: tensors must live on a CUDA device — there is no CPU fallback "
                "(got a tensor on %s)" % (t.device,)
            )
        if t.dtype != torch.float32:
            raise TypeError(f"neural_lam_b200: float32 tensors expected, got {t.dtype}")


def _stream_ptr(device):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def as_rows(x):
    """View ``x`` of shape (N,H) or (B,N,H) as (ptr-compatible tensor, B, batch stride in
    elements) with dense rows; keeps stride-0 batch expansions (reference expand_to_batch,
    models/step_predictors/base.py:122-139) without materialising them."""
    if x.dim() == 2:
        if x.stride(1) != 1 or x.stride(0) != x.shape[1]:
            x = x.contiguous()
        return x, 1, 0
    if x.dim() != 3:
        raise ValueError(f"expected (N,H) or (B,N,H) tensor, got shape {tuple(x.shape)}")
    B, N, H = x.shape
    ok = (H == 1 or x.stride(2) == 1) and (N == 1 or x.stride(1) == H)
    if not ok or (B > 1 and x.stride(0) != 0 and x.stride(0) < N * H):
        x = x.contiguous()
    bs = x.stride(0) if B > 1 else 0
    return x, B, bs


def mlp_struct(seq):
    """NlamMlp view of a make_mlp ``nn.Sequential`` (Linear, SiLU, ..., Linear[, LayerNorm])."""
    linears = [m for m in seq if isinstance(m, torch.nn.Linear)]
    lns = [m for m in seq if isinstance(m, torch.nn.LayerNorm)]
    if not linears or len(linears) > _lib.NLAM_MAX_LINEAR:
        raise _lib.NlamError(f"unsupported MLP depth ({len(linears)} Linear layers)")
    s = NlamMlp()
    s.n_linear = len(linears)
    s.in_dim = linears[0].in_features
    for i, lin in enumerate(linears):
        _require_cuda(lin.weight, lin.bias)
        s.out_dim[i] = lin.out_features
        s.w[i] = lin.weight.data_ptr()
        s.b[i] = lin.bias.data_ptr()
    if lns:
        ln = lns[-1]
        s.ln_gamma = ln.weight.data_ptr()
        s.ln_beta = ln.bias.data_ptr()
        s.ln_eps = ln.eps
    else:
        s.ln_gamma = None
        s.ln_beta = None
        s.ln_eps = 1e-5
    return s


def _iptr(t, offset_rows=0):
    """Device address of an int32 index tensor (offset by whole entries)."""
    if t is None:
        return None
    assert t.dtype == torch.int32 and t.is_cuda and t.is_contiguous()
    return t.data_ptr() + 4 * offset_rows


def _row_srcs(prepared, idx=None, r0=0):
    """NlamRowSrc array of ``as_rows`` views ``(t, B, batch stride)``: row r of source i reads row r0 + r of it, or the row
    ``idx[i][r0 + r]`` where ``idx[i]`` (an int32 device tensor) is given."""
    arr = (NlamRowSrc * len(prepared))()
    for r, (t, _, bs), ix in zip(arr, prepared, idx or [None] * len(prepared)):
        d = t.shape[-1]
        r.ptr, r.idx = (t.data_ptr() + 4 * r0 * d, None) if ix is None else (t.data_ptr(), _iptr(ix, r0))
        r.bstride, r.dim = bs, d
    return arr


def _step_io(prev, boundary, bmask, out):
    """The forecast-step epilogue's tensors: ``prev`` (B, G, D), ``boundary`` of prev's shape with its (G) mask ``bmask`` (or
    both None), ``out`` of prev's shape, not prev itself (allocated when None) -> the four, contiguous."""
    prev = prev.contiguous()
    if boundary is not None:
        assert bmask is not None, "a boundary state needs its mask"
        boundary, bmask = boundary.contiguous(), bmask.contiguous()
        assert boundary.shape == prev.shape and bmask.numel() == prev.shape[1]
    if out is None:
        out = torch.empty_like(prev)
    assert out.is_contiguous() and out.shape == prev.shape and out.data_ptr() != prev.data_ptr()
    return prev, boundary, bmask, out


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _std_io(std_out, prev, n_out):
    """The predicted-std form of a fused step: ``std_out`` (a dense float32 device tensor of prev's shape (B, G, d)) and
    the MLP's output count ``n_out`` (2·d) -> whether the fused kernels can take the call (False: the widths disagree)."""
    if tuple(std_out.shape) != tuple(prev.shape) or not std_out.is_contiguous():
        raise ValueError(f"std_out: expected a contiguous tensor of shape {tuple(prev.shape)}, got {tuple(std_out.shape)}")
    _require_cuda(std_out)
    return n_out == 2 * prev.shape[-1]


def rowmlp(seq, sources, res=None, flags=0, idx=None, res_idx=None, row_range=None):
    """``out[r] = (res[res_idx[r]] or 0) + seq(cat_s sources_s[idx_s[r]])`` for rows r in
    ``row_range`` (default all) with the row-MLP kernels (``nlam_rowmlp_fwd``).

    sources: tensors (N_s,d_s)/(B,N_s,d_s); idx: per-source int32 device tensors (or None
    for identity).  The number of output rows is the length of the index tensors, or N for
    identity sources."""
    L = _lib.lib()
    prepared = [as_rows(s) for s in sources]
    _require_cuda(*[p[0] for p in prepared])
    idx = idx or [None] * len(sources)
    B = max(p[1] for p in prepared)
    n_total = None
    for (t, _, _), ix in zip(prepared, idx):
        n = ix.numel() if ix is not None else t.shape[-2]
        if n_total is None:
            n_total = n
        elif n != n_total:
            raise ValueError("rowmlp: sources disagree on the number of rows")
    r0, r1 = (0, n_total) if row_range is None else row_range
    n_rows = r1 - r0
    dev = prepared[0][0].device
    if any(b not in (1, B) for _, b, _ in prepared):
        raise ValueError("rowmlp: sources disagree on batch size")
    arr = _row_srcs(prepared, idx, r0)
    mlp = mlp_struct(seq)
    nf = mlp.out_dim[mlp.n_linear - 1]
    three_d = any(s.dim() == 3 for s in sources) or (res is not None and res.dim() == 3)
    resp = None
    if res is not None:
        keep, rb, rbs = as_rows(res)
        _require_cuda(keep)
        if rb not in (1, B) and B != 1:
            raise ValueError("rowmlp: residual batch mismatch")
        B = max(B, rb)
        resp = _row_srcs([(keep, rb, rbs)], [res_idx], r0)
    out = torch.empty((B, n_rows, nf), device=dev, dtype=torch.float32)
    with torch.cuda.device(dev):
        _lib.check(L.nlam_rowmlp_fwd(ctypes.byref(mlp), arr, len(prepared), resp, None, out.data_ptr(), None,
                                     n_rows, B, flags, _stream_ptr(dev)))
    return out if three_d else out[0]


class Graph:
    """Owner of one ``NlamGraph`` handle (receiver-sorted CSR + tile tables on one device)."""

    def __init__(self, edge_index_cpu, device, n_rec_hint=0):
        L = _lib.lib()
        ei = edge_index_cpu.detach().to("cpu", torch.int64).contiguous()
        if ei.dim() != 2 or ei.shape[0] != 2 or ei.shape[1] < 1:
            raise ValueError(f"edge_index must have shape (2, E>=1), got {tuple(ei.shape)}")
        dev = torch.device(device)
        if dev.type != "cuda":
            raise RuntimeError("neural_lam_b200: graphs live on CUDA devices only (no CPU fallback)")
        idx = dev.index if dev.index is not None else torch.cuda.current_device()
        self.device = torch.device("cuda", idx)
        torch.cuda.init()
        with torch.cuda.device(idx):
            torch.cuda.current_stream().synchronize()  # make sure the primary context exists
            h = ctypes.c_void_p()
            _lib.check(L.nlam_graph_create(ctypes.byref(h), ei.data_ptr(), ei.shape[1], n_rec_hint, idx))
        self._h = h
        self._L = L
        self.n_edges = L.nlam_graph_num_edges(h)
        self.n_rec = L.nlam_graph_num_rec(h)
        self.n_send = L.nlam_graph_num_send(h)
        self.max_in_degree = L.nlam_graph_max_in_degree(h)
        self.is_sorted = bool(L.nlam_graph_is_sorted(h))
        self.uniform_degree = L.nlam_graph_uniform_degree(h)
        self.perm = L.nlam_graph_perm(h)
        self.inv_perm = L.nlam_graph_inv_perm(h)

    @property
    def handle(self):
        return self._h

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                self._L.nlam_graph_destroy(self._h)
                self._h = None
        except Exception:
            pass


def gather_rows(x, idx, n_rows=None, deg_ptr=None):
    """out[..., r, :] = x[..., idx[r], :] (optionally scaled by 1/max(deg(idx[r]),1) with
    deg taken from the CSR offsets ``deg_ptr``).  ``idx``: int32 device tensor or raw address."""
    L = _lib.lib()
    xr, B, bs = as_rows(x)
    _require_cuda(xr)
    H = xr.shape[-1]
    if isinstance(idx, torch.Tensor):
        n_rows = idx.numel()
        idx = _iptr(idx)
    if isinstance(deg_ptr, torch.Tensor):
        deg_ptr = _iptr(deg_ptr)
    out = torch.empty((B, n_rows, H), device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        _lib.check(L.nlam_gather_rows(xr.data_ptr(), bs, idx, n_rows, out.data_ptr(), n_rows * H, B, H,
                                      deg_ptr, _stream_ptr(x.device)))
    return out if x.dim() == 3 else out[0]


def segment_sum(x, ptr, order, mean=False, out_rows=None):
    """out[..., n, :] = scale * sum_{k in [ptr[n], ptr[n+1])} x[..., order[k], :] with
    ``ptr`` (n_seg+1) / ``order`` int32 device tensors (order None = identity); rows
    n_seg..out_rows-1 (if any) are zero.  Sequential CSR order: deterministic."""
    L = _lib.lib()
    xr, B, bs = as_rows(x)
    _require_cuda(xr)
    H = xr.shape[-1]
    n_seg = ptr.numel() - 1
    rows = n_seg if out_rows is None else out_rows
    if rows > n_seg:
        out = torch.zeros((B, rows, H), device=x.device, dtype=torch.float32)
    else:
        out = torch.empty((B, rows, H), device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        _lib.check(L.nlam_segment_sum(_iptr(ptr), _iptr(order), n_seg, xr.data_ptr(), bs, out.data_ptr(), rows * H,
                                      B, H, 1 if mean else 0, _stream_ptr(x.device)))
    return out if x.dim() == 3 else out[0]


class GatherRowsFn(torch.autograd.Function):
    """y = x[idx]; backward is the deterministic CSR segment sum over the rows that read
    each source row (no atomics): gx[n] = sum_{k in [bwd_ptr[n], bwd_ptr[n+1])} g[bwd_order[k]]."""

    @staticmethod
    def forward(ctx, x, idx, bwd_ptr, bwd_order):
        ctx.save_for_backward(bwd_ptr, bwd_order)
        ctx.x_rows = x.shape[-2]
        return gather_rows(x, idx)

    @staticmethod
    def backward(ctx, g):
        bwd_ptr, bwd_order = ctx.saved_tensors
        return segment_sum(g.contiguous(), bwd_ptr, bwd_order, out_rows=ctx.x_rows), None, None, None


class SegmentSumFn(torch.autograd.Function):
    """aggr[n] = (sum|mean)_{k in segment n} msg[order[k]]; backward gathers (and rescales):
    gmsg[i] = g[seg_of[i]] / max(deg,1)."""

    @staticmethod
    def forward(ctx, msg, ptr, order, seg_of, mean):
        ctx.save_for_backward(ptr, seg_of)
        ctx.mean = mean
        return segment_sum(msg, ptr, order, mean=mean)

    @staticmethod
    def backward(ctx, g):
        ptr, seg_of = ctx.saved_tensors
        gm = gather_rows(g.contiguous(), seg_of, deg_ptr=ptr if ctx.mean else None)
        return gm, None, None, None, None


def inet_fwd(graph, edge_seq, aggr_seq, send, rec, edge_csr, update_edges, flags, want_aggr=False, edge_inplace=False,
             edge_only=False, proj_in=None, next_edge_seq=None):
    """One fused InteractionNet/PropagationNet forward through ``nlam_inet_fwd``.
    ``edge_csr`` must be in CSR edge order.  ``edge_inplace``: write e' = e + m over ``edge_csr`` itself (a dense
    batched tensor the caller owns).  ``edge_only``: stop after the aggregation (``NLAM_EDGE_ONLY``; the node update runs in a
    later call, see ``node_update_step``); rec_out is None then.  ``proj_in`` / ``next_edge_seq``: chained stack over one node
    set (``nlam_inet_fwd_chain``; check ``inet_chain_supported`` first): take this layer's node projections from the previous
    call, and let the node kernel compute those of the next layer's edge MLP — a 4th return value ``proj_out`` then.
    Returns (rec_out, edge_out|None, aggr|None), 3-D."""
    L = _lib.lib()
    s, Bs, sbs = as_rows(send)
    r, Br, rbs = as_rows(rec)
    e, Be, ebs = as_rows(edge_csr)
    _require_cuda(s, r, e)
    B = max(Bs, Br, Be)
    for b in (Bs, Br, Be):
        if b not in (1, B):
            raise ValueError("inet_fwd: inconsistent batch sizes")
    H = r.shape[-1]
    if r.shape[-2] != graph.n_rec:
        raise ValueError(f"rec_rep has {r.shape[-2]} rows, graph has {graph.n_rec} receivers")
    if s.shape[-2] < graph.n_send:
        raise ValueError(f"send_rep has {s.shape[-2]} rows, edge_index references sender {graph.n_send - 1}")
    if e.shape[-2] != graph.n_edges:
        raise ValueError(f"edge_rep has {e.shape[-2]} rows, graph has {graph.n_edges} edges")
    dev = r.device
    if dev != graph.device:
        raise RuntimeError(f"graph handle lives on {graph.device}, tensors on {dev}")
    em = mlp_struct(edge_seq)
    am = mlp_struct(aggr_seq)
    want_aggr = want_aggr or edge_only
    rec_out = None if edge_only else torch.empty((B, graph.n_rec, H), device=dev, dtype=torch.float32)
    if (update_edges and edge_inplace and Be == B and (B == 1 or ebs == graph.n_edges * H)
            and L.nlam_inet_inplace_supported(graph.handle, ctypes.byref(em), s.data_ptr(), sbs, r.data_ptr(), rbs,
                                              e.data_ptr(), ebs, B, flags)):
        edge_out = e
    else:
        edge_out = torch.empty((B, graph.n_edges, H), device=dev, dtype=torch.float32) if update_edges else None
    aggr = torch.empty((B, graph.n_rec, H), device=dev, dtype=torch.float32) if want_aggr else None
    hint = _lib.HINT_ONE_HIDDEN if (em.n_linear == 2 and am.n_linear == 2 and em.ln_gamma and am.ln_gamma) else 0
    ws_bytes = L.nlam_inet_workspace_bytes(graph.handle, B, H, flags | hint)
    ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
    if proj_in is not None or next_edge_seq is not None:
        nm = mlp_struct(next_edge_seq) if next_edge_seq is not None else None
        proj_out = torch.empty((2, B, graph.n_rec, H), device=dev, dtype=torch.float32) if nm is not None else None
        with torch.cuda.device(dev):
            _lib.check(L.nlam_inet_fwd_chain(
                graph.handle, ctypes.byref(em), ctypes.byref(am), ctypes.byref(nm) if nm is not None else None,
                s.data_ptr(), sbs, r.data_ptr(), rbs, e.data_ptr(), ebs,
                rec_out.data_ptr(), edge_out.data_ptr() if update_edges else None,
                aggr.data_ptr() if want_aggr else None, proj_in.data_ptr() if proj_in is not None else None,
                proj_out.data_ptr() if proj_out is not None else None, B, flags, ws.data_ptr(), ws_bytes, _stream_ptr(dev)))
        return rec_out, edge_out, aggr, proj_out
    with torch.cuda.device(dev):
        _lib.check(L.nlam_inet_fwd(
            graph.handle, ctypes.byref(em), ctypes.byref(am),
            s.data_ptr(), sbs, r.data_ptr(), rbs, e.data_ptr(), ebs,
            rec_out.data_ptr() if rec_out is not None else None, edge_out.data_ptr() if update_edges else None,
            aggr.data_ptr() if want_aggr else None, B, flags | (_lib.EDGE_ONLY if edge_only else 0),
            ws.data_ptr(), ws_bytes, _stream_ptr(dev)))
    return rec_out, edge_out, aggr


def inet_chain_supported(graph, edge_seq, aggr_seq, next_edge_seq, node_rep, flags):
    """Can ``inet_fwd`` on this layer of a stack over one node set consume projections of the previous call and (with
    ``next_edge_seq``) produce the next layer's (``nlam_inet_chain_supported``)?"""
    L = _lib.lib()
    x, B, bs = as_rows(node_rep)
    if not x.is_cuda:
        return False
    em, am = mlp_struct(edge_seq), mlp_struct(aggr_seq)
    nm = mlp_struct(next_edge_seq) if next_edge_seq is not None else None
    return bool(L.nlam_inet_chain_supported(graph.handle, ctypes.byref(em), ctypes.byref(am),
                                            ctypes.byref(nm) if nm is not None else None, x.data_ptr(), bs, x.data_ptr(), bs, B,
                                            flags))


def step_epilogue(net_out, prev, boundary, bmask, diff_std, diff_mean, out=None, clamp=None):
    """new = bmask*boundary + (1-bmask)*(prev + net_out*diff_std + diff_mean) (no-grad path); ``clamp`` =
    (kind int32 (D), lo (D), up (D)): the clamped update of models/step_predictors/base.py:366-396 instead of the plain
    residual for the variables with limits."""
    L = _lib.lib()
    net_out = net_out.contiguous()
    _require_cuda(net_out, prev, diff_std, diff_mean, boundary, bmask)
    B, G, D = net_out.shape
    if prev.shape != net_out.shape or diff_std.numel() != D or diff_mean.numel() != D:
        raise ValueError(f"step_epilogue: net_out {tuple(net_out.shape)}, prev {tuple(prev.shape)}, diff statistics "
                         f"{diff_std.numel()}/{diff_mean.numel()} disagree")
    prev, boundary, bmask, out = _step_io(prev, boundary, bmask, out)
    with torch.cuda.device(net_out.device):
        if clamp is not None:
            kind, lo, up = clamp
            assert kind.dtype == torch.int32 and kind.numel() == D and lo.numel() == D and up.numel() == D
            _lib.check(L.nlam_step_epilogue_clamped(net_out.data_ptr(), prev.data_ptr(), _ptr(boundary), _ptr(bmask),
                                                    diff_std.data_ptr(), diff_mean.data_ptr(), kind.data_ptr(), lo.data_ptr(),
                                                    up.data_ptr(), out.data_ptr(), B, G, D, _stream_ptr(net_out.device)))
        else:
            _lib.check(L.nlam_step_epilogue(net_out.data_ptr(), prev.data_ptr(), _ptr(boundary), _ptr(bmask), diff_std.data_ptr(),
                                            diff_mean.data_ptr(), out.data_ptr(), B, G, D, _stream_ptr(net_out.device)))
    return out


def rowmlp_step(seq, x, prev, boundary, bmask, diff_std, diff_mean, flags=0, out=None, std_out=None):
    """``bmask*boundary + (1-bmask)*(prev + (seq(x)*diff_std + diff_mean))`` in ONE launch
    (``nlam_rowmlp_step_fwd``: output_map + the forecast-step epilogue); returns None when the
    library does not fuse this shape / math mode (the caller then runs the two kernels).
    ``std_out`` (prev's shape (B, G, d)): ``seq`` has 2·d outputs, the first d take the epilogue and
    ``std_out = softplus(the last d)`` (``nlam_rowmlp_step_std_fwd``)."""
    L = _lib.lib()
    if flags & _lib.MATH_FP32:
        return None
    xr, B, bs = as_rows(x)
    _require_cuda(xr, prev, diff_std, diff_mean, boundary, bmask)
    mlp = mlp_struct(seq)
    G = xr.shape[-2]
    n_out = mlp.out_dim[mlp.n_linear - 1]
    if std_out is not None:
        if prev.shape[:2] != (B, G) or not _std_io(std_out, prev, n_out):
            return None
    elif prev.shape != (B, G, n_out):
        return None
    prev, boundary, bmask, out = _step_io(prev, boundary, bmask, out)
    with torch.cuda.device(xr.device):
        args = (ctypes.byref(mlp), _row_srcs([(xr, B, bs)]), 1, prev.data_ptr(), _ptr(boundary), _ptr(bmask), diff_std.data_ptr(),
                diff_mean.data_ptr(), out.data_ptr())
        tail = (G, B, flags, _stream_ptr(xr.device))
        rc = (L.nlam_rowmlp_step_fwd(*args, *tail) if std_out is None
              else L.nlam_rowmlp_step_std_fwd(*args, std_out.data_ptr(), *tail))
    if rc == _lib.E_UNSUPPORTED:
        return None
    _lib.check(rc)
    return out


def node_update_step(node_seq, out_seq, rec, aggr, prev, boundary, bmask, diff_std, diff_mean, flags=0, out=None, std_out=None):
    """``bmask*boundary + (1-bmask)*(prev + out_seq(rec + node_seq([rec | aggr]))*diff_std + diff_mean)`` in ONE launch
    (``nlam_node_update_step_fwd``: node update of the mesh->grid layer + output_map + forecast-step epilogue; the updated
    grid representation never goes to HBM).  Returns None when the library does not fuse this shape / math mode.
    ``std_out``: the predicted-std form as in ``rowmlp_step`` (``nlam_node_update_step_std_fwd``)."""
    L = _lib.lib()
    if flags & _lib.MATH_FP32:
        return None
    rr, B, rbs = as_rows(rec)
    ar, Ba, abs_ = as_rows(aggr)
    _require_cuda(rr, ar, prev, diff_std, diff_mean, boundary, bmask)
    nm, om = mlp_struct(node_seq), mlp_struct(out_seq)
    D = om.out_dim[om.n_linear - 1]
    G = rr.shape[-2]
    Bt = max(B, Ba)
    if std_out is not None:
        if not _std_io(std_out, prev, D):
            return None
        D //= 2
    if (rr.shape[-1] != 64 or ar.shape[-1] != 64 or ar.shape[-2] != G or prev.shape != (Bt, G, D) or Ba != Bt
            or (Bt > 1 and abs_ != G * 64) or B not in (1, Bt)):
        return None
    prev, boundary, bmask, out = _step_io(prev, boundary, bmask, out)
    with torch.cuda.device(rr.device):
        args = (ctypes.byref(nm), ctypes.byref(om), rr.data_ptr(), rbs if B > 1 else 0, ar.data_ptr(), prev.data_ptr(),
                _ptr(boundary), _ptr(bmask), diff_std.data_ptr(), diff_mean.data_ptr(), out.data_ptr())
        tail = (G, Bt, flags, _stream_ptr(rr.device))
        rc = (L.nlam_node_update_step_fwd(*args, *tail) if std_out is None
              else L.nlam_node_update_step_std_fwd(*args, std_out.data_ptr(), *tail))
    if rc == _lib.E_UNSUPPORTED:
        return None
    _lib.check(rc)
    return out


def decode_step(graph, edge_seq, node_seq, out_seq, send, rec, edge_csr, prev, boundary, bmask, diff_std, diff_mean, flags=0,
                out=None, std_out=None):
    """The whole mesh->grid decoder of a forecast step in two launches (``nlam_decode_step_fwd``): the edge projections,
    then one kernel for the messages, the per-receiver aggregation, the node update ``rec + node_seq([rec | aggr])``,
    ``out_seq`` and the forecast-step epilogue ``bmask*boundary + (1-bmask)*(prev + y*diff_std + diff_mean)``.
    ``edge_csr``: edge features in CSR edge order, shared by the batch.  Returns None when the library does not fuse this
    graph / shape / math mode (the caller then runs ``inet_fwd(edge_only=True)`` + ``node_update_step``).  ``std_out``: the
    predicted-std form as in ``rowmlp_step`` (``nlam_decode_step_std_fwd``)."""
    L = _lib.lib()
    if flags & _lib.MATH_FP32:
        return None
    s, Bs, sbs = as_rows(send)
    r, Br, rbs = as_rows(rec)
    e, Be, ebs = as_rows(edge_csr)
    _require_cuda(s, r, e, prev, diff_std, diff_mean, boundary, bmask)
    B = max(Bs, Br, Be)
    em, nm, om = mlp_struct(edge_seq), mlp_struct(node_seq), mlp_struct(out_seq)
    D = om.out_dim[om.n_linear - 1]
    G = r.shape[-2]
    if std_out is not None:
        if not _std_io(std_out, prev, D):
            return None
        D //= 2
    if (any(b not in (1, B) for b in (Bs, Br, Be)) or (Be > 1 and ebs != 0) or r.shape[-1] != 64 or s.shape[-1] != 64
            or e.shape[-1] != 64 or G != graph.n_rec or s.shape[-2] < graph.n_send or e.shape[-2] != graph.n_edges
            or prev.shape != (B, G, D) or r.device != graph.device):
        return None
    prev, boundary, bmask, out = _step_io(prev, boundary, bmask, out)
    dev = r.device
    ws_bytes = L.nlam_decode_workspace_bytes(graph.handle, B)
    ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
    with torch.cuda.device(dev):
        args = (graph.handle, ctypes.byref(em), ctypes.byref(nm), ctypes.byref(om), s.data_ptr(), sbs if Bs > 1 else 0,
                r.data_ptr(), rbs if Br > 1 else 0, e.data_ptr(), ebs if Be > 1 else 0, prev.data_ptr(), _ptr(boundary),
                _ptr(bmask), diff_std.data_ptr(), diff_mean.data_ptr(), out.data_ptr())
        tail = (B, flags, ws.data_ptr(), ws_bytes, _stream_ptr(dev))
        rc = (L.nlam_decode_step_fwd(*args, *tail) if std_out is None
              else L.nlam_decode_step_std_fwd(*args, std_out.data_ptr(), *tail))
    if rc == _lib.E_UNSUPPORTED:
        return None
    _lib.check(rc)
    return out


def encode(graph, embed_seq, sources, grid_seq, edge_seq, mesh, edge_csr, flags=0, want_emb=False, edge_seq_b=None):
    """The grid side of a forecast step's encoder in ONE launch (``nlam_encode_fwd``): ``grid_emb = embed_seq(cat sources)``
    and ``grid_rep = grid_emb + grid_seq(grid_emb)`` (B, G, 64), and for the grid -> mesh layer on ``graph`` whose edge MLP is
    ``edge_seq`` (and for a second one, ``edge_seq_b``, on the same graph; both with grid_emb as senders, ``mesh`` as
    receivers and ``edge_csr`` as edge features, shared by the batch) ``proj = [P_s | P_r]`` flat, ``P_s = grid_emb·W1sᵀ``
    (B, G, 64) and ``P_r = mesh·W1rᵀ + b1`` (n_mesh, 64) — the ``proj_in`` of that layer's ``inet_fwd`` with send = P_s.
    Returns ``(grid_rep, [proj per layer], grid_emb | None)``; grid_emb is stored where ``want_emb`` (not with
    ``edge_seq_b``), else it stays on chip.  Returns None when the library does not fuse these shapes / this math mode (the
    caller then runs the embedder, the g2m layer(s) and ``grid_seq`` as separate calls)."""
    L = _lib.lib()
    if flags & _lib.MATH_FP32:
        return None
    prepared = [as_rows(t) for t in sources]
    m, Bm, mbs = as_rows(mesh)
    e, Be, ebs = as_rows(edge_csr)
    _require_cuda(m, e, *[t for t, _, _ in prepared])
    B = max(b for _, b, _ in prepared)
    G = prepared[0][0].shape[-2]
    if (any(b not in (1, B) for _, b, _ in prepared) or any(t.shape[-2] != G for t, _, _ in prepared)
            or Bm not in (1, B) or Be not in (1, B) or m.shape[-1] != 64 or e.shape[-1] != 64
            or m.shape[-2] != graph.n_rec or e.shape[-2] != graph.n_edges or m.device != graph.device):
        return None
    edge_seqs = [edge_seq] if edge_seq_b is None else [edge_seq, edge_seq_b]
    second = edge_seq_b is not None
    em, gm = mlp_struct(embed_seq), mlp_struct(grid_seq)
    sm = [mlp_struct(s) for s in edge_seqs]
    grid_rep = torch.empty((B, G, 64), device=m.device, dtype=torch.float32)
    projs = [torch.empty((B * G + graph.n_rec) * 64, device=m.device, dtype=torch.float32) for _ in edge_seqs]
    grid_emb = torch.empty((B, G, 64), device=m.device, dtype=torch.float32) if want_emb else None
    with torch.cuda.device(m.device):
        rc = L.nlam_encode_fwd(graph.handle, ctypes.byref(em), _row_srcs(prepared), len(prepared), ctypes.byref(gm),
                               ctypes.byref(sm[0]), ctypes.byref(sm[1]) if second else None, m.data_ptr(), mbs if Bm > 1 else 0,
                               e.data_ptr(), ebs if Be > 1 else 0, grid_rep.data_ptr(), projs[0].data_ptr(),
                               projs[1].data_ptr() if second else None, _ptr(grid_emb), G, B, flags, _stream_ptr(m.device))
    if rc == _lib.E_UNSUPPORTED:
        return None
    _lib.check(rc)
    return grid_rep, projs, grid_emb


def latent_sample(param_seq, embed_seq, x, eps, flags=0):
    """Graph-EFM's latent step in ONE launch (``nlam_latent_sample_fwd``): ``p = param_seq(x)``, ``mean, std`` from p
    (64 outputs: std = 1; 128 outputs: std = 1e-4 + softplus(p[..., 64:])), ``z = mean + eps * std`` and
    ``embed_seq(z)`` -> (B, N, 64); p and z stay on chip.  ``x``, ``eps``: (B, N, 64).  Returns None when the library does not
    fuse these shapes / this math mode (the caller then composes the three steps)."""
    L = _lib.lib()
    if flags & _lib.MATH_FP32:
        return None
    xr, Bx, xbs = as_rows(x)
    er, Be, ebs = as_rows(eps)
    _require_cuda(xr, er)
    B = max(Bx, Be)
    if (Bx not in (1, B) or Be not in (1, B) or xr.shape[-1] != 64 or er.shape[-1] != 64 or er.shape[-2] != xr.shape[-2]
            or xr.device != er.device):
        return None
    pm, em = mlp_struct(param_seq), mlp_struct(embed_seq)
    N = xr.shape[-2]
    out = torch.empty((B, N, 64), device=xr.device, dtype=torch.float32)
    args = (ctypes.byref(pm), ctypes.byref(em), xr.data_ptr(), xbs if Bx > 1 else 0, er.data_ptr(), ebs if Be > 1 else 0,
            out.data_ptr(), N, B, flags)
    if not L.nlam_latent_sample_supported(*args):
        return None
    with torch.cuda.device(xr.device):
        _lib.check(L.nlam_latent_sample_fwd(*args, _stream_ptr(xr.device)))
    return out


class RecomputeFn(torch.autograd.Function):
    """Forward = hand-written kernels (``kernel_fn``, run without autograd); backward =
    re-evaluate the same math as a differentiable graph (``torch_fn``: custom gather /
    segment-sum Functions for the index work, ATen/cuBLAS for the dense GEMMs) and pull
    gradients out of it.  Nothing but the inputs is saved (recompute-in-backward)."""

    @staticmethod
    def forward(ctx, kernel_fn, torch_fn, *tensors):
        ctx.torch_fn = torch_fn
        ctx.save_for_backward(*tensors)
        outs = kernel_fn(*tensors)
        if isinstance(outs, torch.Tensor):
            ctx.single = True
            return outs
        ctx.single = False
        return tuple(outs)

    @staticmethod
    def backward(ctx, *gouts):
        tensors = ctx.saved_tensors
        needs = ctx.needs_input_grad[2:]
        with torch.enable_grad():
            ins = [t.detach().requires_grad_(bool(n)) for t, n in zip(tensors, needs)]
            outs = ctx.torch_fn(*ins)
            if isinstance(outs, torch.Tensor):
                outs = (outs,)
            pairs = [(o, g) for o, g in zip(outs, gouts) if g is not None and o.requires_grad]
            wanted = [t for t, n in zip(ins, needs) if n]
            grads = torch.autograd.grad([o for o, _ in pairs], wanted, [g for _, g in pairs], allow_unused=True)
        it = iter(grads)
        res = [next(it) if n else None for n in needs]
        return (None, None, *res)


class KernelBackwardFn(torch.autograd.Function):
    """Forward = hand-written kernels; backward = hand-written kernels too (``bwd_fn(saved inputs, output grads) ->
    input grads``, see backward.py).  Nothing but the inputs is saved (recompute-in-backward)."""

    @staticmethod
    def forward(ctx, kernel_fn, bwd_fn, *tensors):
        ctx.bwd_fn = bwd_fn
        ctx.save_for_backward(*tensors)
        outs = kernel_fn(*tensors)
        if isinstance(outs, torch.Tensor):
            return outs
        return tuple(outs)

    @staticmethod
    def backward(ctx, *gouts):
        needs = ctx.needs_input_grad[2:]
        with torch.no_grad():
            grads = ctx.bwd_fn(ctx.saved_tensors, gouts, needs)
        return (None, None, *[g if n else None for g, n in zip(grads, needs)])


def run_with_recompute(kernel_fn, torch_fn, tensors, bwd_fn=None):
    """Kernel forward; if autograd is recording, attach the backward: the hand-written one (``bwd_fn``) where the shape
    is covered, else the recompute through a differentiable restatement (``torch_fn``)."""
    if torch.is_grad_enabled() and any(t.requires_grad for t in tensors):
        if bwd_fn is not None:
            return KernelBackwardFn.apply(kernel_fn, bwd_fn, *tensors)
        return RecomputeFn.apply(kernel_fn, torch_fn, *tensors)
    with torch.no_grad():
        return kernel_fn(*tensors)
