"""Hand-written backward of the path: gradients of the make_mlp networks (reference utils/networks.py:27-40) and of
InteractionNet / PropagationNet (reference gnn_layers.py:110-157, :231-249; exercised by the reference's
tests/test_gnn_layers.py section F and by training, models/module.py:303) composed from libnlam_b200 launches only —
no ATen / cuBLAS math:

  * dense products on the generic wgmma Linear kernel (``nlam_linear``, csrc/tc7.cu): ``dX = dY · W`` is a Linear with
    the transposed weight, ``dW = dYᵀ · X`` a split-K product over zero-padded transposes of dY and X whose partial
    products are reduced in a fixed order;
  * SiLU / LayerNorm forward + backward, bias column sums, transposes, the gather-add of the message gradient and the
    CSR segment sums (sender-CSR for the sender gather's backward) from csrc/bwd.cu / simt.cu.

Recompute-in-backward: nothing but the layer inputs is kept from the forward; the pre-activations the backward needs
(z = pre-SiLU, y = pre-LayerNorm) are re-evaluated here with the same kernels.  TF32 operands, fp32 accumulation — the
reference's own GPU configuration for forward AND backward (train_model.py:484-488).  PyTorch supplies device memory
(``torch.empty``) and the autograd bookkeeping only.
"""
import ctypes

import torch

from . import _lib


def _sp(t):
    return ctypes.c_void_p(torch.cuda.current_stream(t.device).cuda_stream)


def _ptr(t, offset_elems=0):
    return None if t is None else t.data_ptr() + 4 * offset_elems


def _dense3(x):
    """(B, n, k) float32 contiguous (stride-0 batch expansions are materialised: gradients are per batch element)"""
    if x.dim() == 2:
        x = x.unsqueeze(0)
    return x.contiguous()


def linear(x0, w, n_out, *, w_off=0, ldw=None, w_cols=0, w_bs=0, x1=None, bias=None, act=False, ln=None, add=(), post=None,
           res=None, out2=False, x0_pitch=0, k0=None, shape=None, x0_bs=None):
    """``epi([x0 | x1] · W[:, cols]ᵀ + bias + gathered addends)`` on the generic wgmma Linear kernel.
    x0 / x1: dense (B, n, k) tensors (or, with ``shape=(B, n)``, ``k0`` and ``x0_pitch`` / ``x0_bs``: a raw strided
    view); ``w``: parameter / buffer holding the weight, ``w_off`` its column offset, ``ldw`` its row pitch;
    ``add`` / ``post``: (tensor (B|1, rows, n_out), int32 index pointer, batch stride) gathered addends before / after the
    epilogue; ``ln``: (gamma, beta, eps); ``res``: dense (B, n, n_out) residual.  Returns out or (out, out2)."""
    L = _lib.lib()
    if shape is None:
        B, n, k0 = x0.shape
        x0_bs = n * k0
    else:
        B, n = shape
    k1 = 0
    x1_bs = 0
    if x1 is not None:
        k1 = x1.shape[-1]
        x1_bs = x1.shape[1] * k1
    ldw = ldw if ldw is not None else (k0 + k1)
    out = torch.empty((B, n, n_out), device=x0.device, dtype=torch.float32)
    o2 = torch.empty((B, n, n_out), device=x0.device, dtype=torch.float32) if out2 else None
    adds = list(add) + [(None, None, 0)] * (2 - len(add))
    pt, pi, pbs = post if post is not None else (None, None, 0)
    g, bt, eps = ln if ln is not None else (None, None, 0.0)
    with torch.cuda.device(x0.device):
        _lib.check(L.nlam_linear(
            _ptr(x0), x0_bs, k0, x0_pitch, _ptr(x1), x1_bs, k1, _ptr(w, w_off), ldw, w_cols, w_bs, _ptr(bias), n_out,
            1 if act else 0, _ptr(g), _ptr(bt), eps,
            _ptr(adds[0][0]), adds[0][1], adds[0][2], _ptr(adds[1][0]), adds[1][1], adds[1][2],
            _ptr(pt), pi, pbs, _ptr(res), (res.shape[1] * n_out if res is not None else 0), n, B, _ptr(out), _ptr(o2), _sp(x0)))
    return (out, o2) if out2 else out


def silu(z, gh=None):
    out = torch.empty_like(z)
    with torch.cuda.device(z.device):
        _lib.check(_lib.lib().nlam_silu(_ptr(z), _ptr(gh), _ptr(out), z.numel(), _sp(z)))
    return out


def layernorm_fwd(y, gamma, beta, eps):
    out = torch.empty_like(y)
    H = y.shape[-1]
    with torch.cuda.device(y.device):
        _lib.check(_lib.lib().nlam_layernorm_fwd(_ptr(y), _ptr(gamma), _ptr(beta), eps, _ptr(out), y.numel() // H, H, _sp(y)))
    return out


def _scratch(device, C):
    return torch.empty(_lib.lib().nlam_bwd_scratch_floats(C), device=device, dtype=torch.float32)


def layernorm_bwd(g, y, gamma, eps):
    """-> (g_y, dgamma, dbeta)"""
    H = y.shape[-1]
    gy = torch.empty_like(y)
    dg = torch.empty(H, device=y.device, dtype=torch.float32)
    db = torch.empty(H, device=y.device, dtype=torch.float32)
    sc = _scratch(y.device, H)
    with torch.cuda.device(y.device):
        _lib.check(_lib.lib().nlam_layernorm_bwd(_ptr(g), _ptr(y), _ptr(gamma), eps, _ptr(gy), _ptr(dg), _ptr(db),
                                                 y.numel() // H, H, _ptr(sc), _sp(y)))
    return gy, dg, db


def colsum(g):
    C = g.shape[-1]
    out = torch.empty(C, device=g.device, dtype=torch.float32)
    sc = _scratch(g.device, C)
    with torch.cuda.device(g.device):
        _lib.check(_lib.lib().nlam_colsum(_ptr(g), g.numel() // C, C, _ptr(out), _ptr(sc), _sp(g)))
    return out


def transpose_pad(x, rows, C, pitch, rows_pad, x_off=0):
    xt = torch.empty((C, rows_pad), device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        _lib.check(_lib.lib().nlam_transpose_pad(_ptr(x, x_off), rows, C, pitch, _ptr(xt), rows_pad, _sp(x)))
    return xt


def pack(sources, kp):
    """zero-padded concatenation of up to four dense (B, n, d) tensors -> (B, n, kp)"""
    B, n = sources[0].shape[0], sources[0].shape[1]
    out = torch.empty((B, n, kp), device=sources[0].device, dtype=torch.float32)
    s = list(sources) + [None] * (4 - len(sources))
    d = [t.shape[-1] if t is not None else 0 for t in s]
    bs = [t.shape[1] * t.shape[2] if t is not None else 0 for t in s]
    with torch.cuda.device(out.device):
        _lib.check(_lib.lib().nlam_pack_rows(_ptr(s[0]), _ptr(s[1]), _ptr(s[2]), _ptr(s[3]), *d, *bs, _ptr(out), kp, n, B, _sp(out)))
    return out


def grad_weight(gy, x, out, out_off=0, out_pitch=None, x_off=0, x_cols=None, x_pitch=None):
    """``out[:, off : off + K] = gyᵀ · x``: gy (R, N) dense rows, x (R, K) rows (column slice ``x_off``/``x_cols`` of a
    tensor with row pitch ``x_pitch``).  Split-K on the tensor cores: the R rows are cut into S ranges, each CTA
    multiplies its range of the zero-padded transposes, the S partial (N, K) products are summed in order."""
    L = _lib.lib()
    R = gy.numel() // gy.shape[-1]
    N = gy.shape[-1]
    K = x_cols if x_cols is not None else x.shape[-1]
    x_pitch = x_pitch if x_pitch is not None else x.shape[-1]
    out_pitch = out_pitch if out_pitch is not None else out.shape[-1]
    n_tiles = (N + 127) // 128
    S = max(1, min(296 // n_tiles, (R + 511) // 512))
    k_per = ((R + S - 1) // S + 31) // 32 * 32
    rows_pad = S * k_per
    gyT = transpose_pad(gy, R, N, N, rows_pad)
    for c0 in range(0, K, 256):                       # the Linear kernel's output width is <= 256
        kc = min(256, K - c0)
        xT = transpose_pad(x, R, kc, x_pitch, rows_pad, x_off=x_off + c0)
        part = linear(gyT, xT, kc, ldw=rows_pad, w_cols=k_per, w_bs=k_per, shape=(S, N), k0=k_per, x0_pitch=rows_pad, x0_bs=k_per)
        with torch.cuda.device(gy.device):
            _lib.check(L.nlam_reduce_partials(_ptr(part), S, N, kc, _ptr(out, out_off + c0), out_pitch, 0, _sp(gy)))


def grad_input(gy, w, n_in, w_off=0, ldw=None, res=None):
    """``gy · W[:, w_off : w_off + n_in]`` (+ res): gy (B, n, N) dense (N any width: zero-padded to a multiple of 32),
    W (N, ldw) row-major.  n_in > 256 (wider than the Linear kernel's output): one Linear per 256-column block of W,
    each written into its column slice of the result; ``res`` only with n_in <= 256."""
    B, n, N = gy.shape
    ldw = ldw if ldw is not None else w.shape[-1]
    Np = (N + 31) // 32 * 32
    if res is not None and n_in > 256:
        raise _lib.NlamError(f"grad_input: a residual needs n_in <= 256 (got {n_in})")
    x0 = gy if Np == N else pack([gy], Np)
    out = None if n_in <= 256 else torch.empty((B, n, n_in), device=gy.device, dtype=torch.float32)
    for c0 in range(0, n_in, 256):
        kc = min(256, n_in - c0)
        wT = transpose_pad(w, N, kc, ldw, (N + 3) // 4 * 4, x_off=w_off + c0)   # (kc, N padded to a multiple of 4)
        part = linear(x0, wT, kc, ldw=wT.shape[1], w_cols=N, res=res)
        if out is None:
            return part
        out[..., c0:c0 + kc] = part
    return out


def segment_sum(x, ptr, order, n_seg, mean=False):
    """CSR segment sum over raw index pointers (``ptr`` n_seg+1 entries, ``order`` nullable), x (B, n, H) dense"""
    B, n, H = x.shape
    out = torch.empty((B, n_seg, H), device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        _lib.check(_lib.lib().nlam_segment_sum(ptr, order, n_seg, _ptr(x), n * H, _ptr(out), n_seg * H, B, H, 1 if mean else 0, _sp(x)))
    return out


def add_gather(a, v, idx, deg_ptr, n_e):
    """a (B, n_e, H) | None, v (B, n_v, H), idx raw pointer -> a + v[idx] (/ deg)"""
    B, n_v, H = v.shape
    out = torch.empty((B, n_e, H), device=v.device, dtype=torch.float32)
    with torch.cuda.device(v.device):
        _lib.check(_lib.lib().nlam_add_gather(_ptr(a), _ptr(v), idx, deg_ptr, n_e, n_v, H, B, _ptr(out), _sp(v)))
    return out


# ------------------------------------------------------------------------------------------------ make_mlp networks
def _mlp_parts(seq):
    lin = [m for m in seq if isinstance(m, torch.nn.Linear)]
    ln = [m for m in seq if isinstance(m, torch.nn.LayerNorm)]
    return lin, (ln[-1] if ln else None)


def mlp_supported(seq, sources, res):
    lin, ln = _mlp_parts(seq)
    if len(lin) != 2 or len(sources) > 4:
        return False
    H, no = lin[0].out_features, lin[1].out_features
    if H % 32 != 0 or H > 256 or no > 256:
        return False
    if ln is not None and no not in (32, 64, 128, 256):
        return False
    return all(t.is_cuda and t.dtype == torch.float32 for t in sources)


def mlp_backward_py(seq, sources, res, g_out, need_src=True):
    """Gradients of ``out = (res or 0) + seq(cat(sources, -1))``.  -> ([g_source...], g_res | None, {param name: grad})"""
    lin, ln = _mlp_parts(seq)
    names = {id(p): n for n, p in seq.named_parameters()}
    B = max(t.shape[0] if t.dim() == 3 else 1 for t in sources)
    src = [_dense3(t if t.dim() == 3 else t.unsqueeze(0)).expand(B, -1, -1).contiguous() if (t.dim() == 2 or t.shape[0] != B)
           else _dense3(t) for t in sources]
    g_out = _dense3(g_out)
    K = sum(t.shape[-1] for t in src)
    Kp = (K + 31) // 32 * 32
    H, no = lin[0].out_features, lin[1].out_features
    x = src[0] if (len(src) == 1 and K == Kp) else pack(src, Kp)
    W1, ldw1 = lin[0].weight, K
    if K % 4:  # TMA wants 16-byte row pitches: zero-padded copy of the (H, K) weight (2- / 3-wide static features)
        ldw1 = (K + 3) // 4 * 4
        W1 = pack([W1.detach().unsqueeze(0)], ldw1)[0]
    z = linear(x, W1, H, ldw=ldw1, w_cols=K, bias=lin[0].bias)
    h = silu(z)
    grads = {}
    if ln is not None:
        y = linear(h, lin[1].weight, no, bias=lin[1].bias)
        g_y, dg, db = layernorm_bwd(g_out, y, ln.weight, ln.eps)
        grads[names[id(ln.weight)]] = dg
        grads[names[id(ln.bias)]] = db
    else:
        g_y = g_out
    grads[names[id(lin[1].bias)]] = colsum(g_y)
    dW2 = torch.empty_like(lin[1].weight)
    grad_weight(g_y, h, dW2)
    grads[names[id(lin[1].weight)]] = dW2
    g_h = grad_input(g_y, lin[1].weight, H)
    g_z = silu(z, gh=g_h)
    grads[names[id(lin[0].bias)]] = colsum(g_z)
    dW1 = torch.empty_like(lin[0].weight)
    grad_weight(g_z, x, dW1, x_cols=K, x_pitch=Kp)
    grads[names[id(lin[0].weight)]] = dW1
    g_src, c = [], 0
    g_x = grad_input(g_z, lin[0].weight, K) if need_src else None
    for t, orig in zip(src, sources):
        d = t.shape[-1]
        gs = None
        if g_x is not None:
            gs = g_x[..., c:c + d]
            if orig.dim() == 2:
                gs = gs.sum(0) if B > 1 else gs[0]
        c += d
        g_src.append(gs)
    return g_src, (g_out if res is not None else None), grads


# ------------------------------------------------------------------------------------------------ InteractionNet
def inet_supported(layer, send, rec, edge):
    H = layer.input_dim
    return (layer._fusable() and layer.hidden_layers == 1 and H in (64, 128, 256)
            and all(t.is_cuda and t.dtype == torch.float32 for t in (send, rec, edge)))


def inet_backward_py(layer, graph, send, rec, edge_csr, g_rec_out, g_edge_out):
    """Gradients of one InteractionNet / PropagationNet call (inputs (B, n, H), ``edge_csr`` / ``g_edge_out`` in CSR edge
    order; ``g_edge_out`` None when the layer does not update edges or the edge output is unused).
    -> (g_send, g_rec, g_edge_csr, {param name: grad})"""
    L = _lib.lib()
    H = layer.input_dim
    prop = layer.propagation
    mean = layer.aggr == "mean" or prop
    em, am = layer.edge_mlp, layer.aggr_mlp
    (e1, e2), eln = _mlp_parts(em)
    (n1, n2), nln = _mlp_parts(am)
    send, rec, edge = _dense3(send), _dense3(rec), _dense3(edge_csr)
    g_rec_out = _dense3(g_rec_out)
    B = max(send.shape[0], rec.shape[0], edge.shape[0])
    send, rec, edge = [t if t.shape[0] == B else t.expand(B, -1, -1).contiguous() for t in (send, rec, edge)]
    Ns_all, Nr, E = send.shape[1], rec.shape[1], edge.shape[1]
    h_ = graph.handle
    src, dst, rowptr = L.nlam_graph_src(h_), L.nlam_graph_dst(h_), L.nlam_graph_rowptr(h_)
    sptr, sperm = L.nlam_graph_sptr(h_), L.nlam_graph_sperm(h_)
    Ns = graph.n_send
    snd = send if Ns_all == Ns else send[:, :Ns].contiguous()
    W1, W2 = e1.weight, e2.weight                      # (H, 3H): [e | sender | receiver], (H, H)
    # ---- forward recompute (pre-activations kept)
    Ps = linear(snd, W1, H, w_off=H, ldw=3 * H)
    Pr = linear(rec, W1, H, w_off=2 * H, ldw=3 * H, bias=e1.bias)
    z1 = linear(edge, W1, H, ldw=3 * H, add=[(Ps, src, Ns * H), (Pr, dst, Nr * H)])
    h1 = silu(z1)
    y2 = linear(h1, W2, H, bias=e2.bias)
    m = layernorm_fwd(y2, eln.weight, eln.bias, eln.eps)
    if prop:
        m = add_gather(m, snd, src, None, E)
    aggr = segment_sum(m, rowptr, None, Nr, mean=mean)
    nz = linear(rec, n1.weight, H, x1=aggr, bias=n1.bias)
    nh = silu(nz)
    ny = linear(nh, n2.weight, H, bias=n2.bias)
    # ---- node update backward
    grads = {}
    g_ny, dg, db = layernorm_bwd(g_rec_out, ny, nln.weight, nln.eps)
    grads["aggr_mlp.3.weight"], grads["aggr_mlp.3.bias"] = dg, db
    grads["aggr_mlp.2.bias"] = colsum(g_ny)
    dWn2 = torch.empty_like(n2.weight)
    grad_weight(g_ny, nh, dWn2)
    grads["aggr_mlp.2.weight"] = dWn2
    g_nz = silu(nz, gh=grad_input(g_ny, n2.weight, H))
    grads["aggr_mlp.0.bias"] = colsum(g_nz)
    dWn1 = torch.empty_like(n1.weight)                 # (H, 2H): [rec | aggr]
    grad_weight(g_nz, rec, dWn1, out_off=0, out_pitch=2 * H)
    grad_weight(g_nz, aggr, dWn1, out_off=H, out_pitch=2 * H)
    grads["aggr_mlp.0.weight"] = dWn1
    # residual base: rec (InteractionNet) or the aggregate (PropagationNet)
    g_rec = grad_input(g_nz, n1.weight, H, w_off=0, ldw=2 * H, res=None if prop else g_rec_out)
    g_aggr = grad_input(g_nz, n1.weight, H, w_off=H, ldw=2 * H, res=g_rec_out if prop else None)
    # ---- message gradient: g_m[e] = g_e'[e] + g_aggr[dst(e)] (/ deg for mean)
    g_eo = _dense3(g_edge_out) if g_edge_out is not None else None
    g_m = add_gather(g_eo, g_aggr, dst, rowptr if mean else None, E)
    g_y2, dg, db = layernorm_bwd(g_m, y2, eln.weight, eln.eps)
    grads["edge_mlp.3.weight"], grads["edge_mlp.3.bias"] = dg, db
    grads["edge_mlp.2.bias"] = colsum(g_y2)
    dW2 = torch.empty_like(W2)
    grad_weight(g_y2, h1, dW2)
    grads["edge_mlp.2.weight"] = dW2
    g_z1 = silu(z1, gh=grad_input(g_y2, W2, H))
    dW1 = torch.empty_like(W1)
    grad_weight(g_z1, edge, dW1, out_off=0, out_pitch=3 * H)
    g_edge = grad_input(g_z1, W1, H, w_off=0, ldw=3 * H, res=g_eo)        # e' = e + m: the residual passes g_e' through
    # sender / receiver gathers: deterministic CSR segment sums over the edges reading each node row
    g_Ps = segment_sum(g_z1, sptr, sperm, Ns)
    g_Pr = segment_sum(g_z1, rowptr, None, Nr)
    grads["edge_mlp.0.bias"] = colsum(g_Pr)
    grad_weight(g_Ps, snd, dW1, out_off=H, out_pitch=3 * H)
    grad_weight(g_Pr, rec, dW1, out_off=2 * H, out_pitch=3 * H)
    grads["edge_mlp.0.weight"] = dW1
    g_send_post = segment_sum(g_m, sptr, sperm, Ns) if prop else None      # message = x_j + edge_mlp(...)
    g_send = grad_input(g_Ps, W1, H, w_off=H, ldw=3 * H, res=g_send_post)
    g_rec = grad_input(g_Pr, W1, H, w_off=2 * H, ldw=3 * H, res=g_rec)
    if Ns_all != Ns:
        full = torch.zeros((B, Ns_all, H), device=send.device, dtype=torch.float32)
        full[:, :Ns] = g_send
        g_send = full
    return g_send, g_rec, g_edge, grads


# ------------------------------------------------------------------------------------------------ one ABI call per layer
def _grads_struct(seq, device):
    """(NlamMlpGrads, {param name: fresh gradient tensor}) for a make_mlp Sequential"""
    from .ops import mlp_struct  # noqa: F401  (same module order as mlp_struct)

    gs = _lib.NlamMlpGrads()
    out = {}
    lin = [(n, m) for n, m in seq.named_children() if isinstance(m, torch.nn.Linear)]
    lns = [(n, m) for n, m in seq.named_children() if isinstance(m, torch.nn.LayerNorm)]
    for i, (n, m) in enumerate(lin):
        out[f"{n}.weight"] = torch.empty_like(m.weight)
        out[f"{n}.bias"] = torch.empty_like(m.bias)
        gs.w[i] = out[f"{n}.weight"].data_ptr()
        gs.b[i] = out[f"{n}.bias"].data_ptr()
    if lns:
        n, m = lns[-1]
        out[f"{n}.weight"] = torch.empty_like(m.weight)
        out[f"{n}.bias"] = torch.empty_like(m.bias)
        gs.ln_gamma = out[f"{n}.weight"].data_ptr()
        gs.ln_beta = out[f"{n}.bias"].data_ptr()
    return gs, out


def mlp_backward(seq, sources, res, g_out, need_src=True):
    """``nlam_mlp_bwd``: gradients of ``out = (res or 0) + seq(cat(sources, -1))``.
    -> ([g_source | None ...], g_res | None, {param name: grad})"""
    from .ops import as_rows, mlp_struct

    L = _lib.lib()
    prepared = [as_rows(t) for t in sources]
    B = max(p[1] for p in prepared)
    n = prepared[0][0].shape[-2]
    dev = g_out.device
    g_out = _dense3(g_out)
    if g_out.shape[0] != B:
        g_out = g_out.expand(B, -1, -1).contiguous()
    arr = (_lib.NlamRowSrc * len(prepared))()
    for i, (t, b, bs) in enumerate(prepared):
        arr[i].ptr, arr[i].idx, arr[i].bstride, arr[i].dim = t.data_ptr(), None, bs, t.shape[-1]
    mlp = mlp_struct(seq)
    gs, pg = _grads_struct(seq, dev)
    g_src = [torch.empty((B, n, t.shape[-1]), device=dev, dtype=torch.float32) if need_src else None for t, _, _ in prepared]
    gptr = (ctypes.c_void_p * len(prepared))(*[(g.data_ptr() if g is not None else None) for g in g_src])
    ws_bytes = L.nlam_mlp_bwd_workspace_bytes(ctypes.byref(mlp), arr, len(prepared), n, B)
    ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
    with torch.cuda.device(dev):
        _lib.check(L.nlam_mlp_bwd(ctypes.byref(mlp), arr, len(prepared), g_out.data_ptr(), gptr, ctypes.byref(gs), n, B,
                                  ws.data_ptr(), ws_bytes, _sp(g_out)))
    outs = []
    for g, orig in zip(g_src, sources):
        if g is not None and orig.dim() == 2:
            g = g.sum(0) if B > 1 else g[0]
        outs.append(g)
    return outs, (g_out if res is not None else None), pg


def inet_backward(layer, graph, send, rec, edge_csr, g_rec_out, g_edge_out):
    """``nlam_inet_bwd``: gradients of one InteractionNet / PropagationNet call (see ``inet_backward_py`` for the launch
    sequence).  -> (g_send, g_rec, g_edge_csr, {param name: grad})"""
    from .ops import as_rows, mlp_struct

    L = _lib.lib()
    H = layer.input_dim
    Ns = graph.n_send
    if send.shape[-2] != Ns:
        send = send[..., :Ns, :].contiguous()
    s, Bs, sbs = as_rows(send)
    r, Br, rbs = as_rows(rec)
    e, Be, ebs = as_rows(edge_csr)
    B = max(Bs, Br, Be)
    if Bs > 1 and sbs not in (0, Ns * H):
        s, sbs = s.contiguous(), Ns * H
    if Br > 1 and rbs not in (0, graph.n_rec * H):
        r, rbs = r.contiguous(), graph.n_rec * H
    if Be > 1 and ebs not in (0, graph.n_edges * H):
        e, ebs = e.contiguous(), graph.n_edges * H
    dev = r.device
    g_rec_out = _dense3(g_rec_out)
    g_eo = _dense3(g_edge_out) if g_edge_out is not None else None
    em, am = mlp_struct(layer.edge_mlp), mlp_struct(layer.aggr_mlp)
    egs, epg = _grads_struct(layer.edge_mlp, dev)
    ags, apg = _grads_struct(layer.aggr_mlp, dev)
    g_send = torch.empty((B, Ns, H), device=dev, dtype=torch.float32)
    g_rec = torch.empty((B, graph.n_rec, H), device=dev, dtype=torch.float32)
    g_edge = torch.empty((B, graph.n_edges, H), device=dev, dtype=torch.float32)
    flags = layer._flags() & (_lib.AGGR_MEAN | _lib.PROPAGATION)
    ws_bytes = L.nlam_inet_bwd_workspace_bytes(graph.handle, B, H, flags)
    ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
    with torch.cuda.device(dev):
        _lib.check(L.nlam_inet_bwd(graph.handle, ctypes.byref(em), ctypes.byref(am), s.data_ptr(), sbs, r.data_ptr(), rbs,
                                   e.data_ptr(), ebs, g_rec_out.data_ptr(), g_eo.data_ptr() if g_eo is not None else None,
                                   g_send.data_ptr(), g_rec.data_ptr(), g_edge.data_ptr(), ctypes.byref(egs), ctypes.byref(ags),
                                   B, flags, ws.data_ptr(), ws_bytes, _sp(r)))
    grads = {f"edge_mlp.{k}": v for k, v in epg.items()}
    grads.update({f"aggr_mlp.{k}": v for k, v in apg.items()})
    return g_send, g_rec, g_edge, grads
