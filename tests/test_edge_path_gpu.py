"""Which form an H = 64 edge stage takes (`-m gpu`).  The split form (node projections + K = 64 edge GEMM) and the K = 192
form round differently in TF32, and only tc_edge_rmw_kernel may write its edge output over its edge input, so one function,
tc_edge_path, decides the form and launch label of a call by the rules of DESIGN.md §4.1.

For calls on every row of those rules — both sides of the 2.5 threshold, B = 1 and B > 1, batch-shared and dense edge /
receiver tensors — this pins the launches of ops.inet_fwd and the answers of the queries that depend on the rules:
nlam_inet_inplace_supported (the call with edge_out = edge takes tc_edge_rmw_kernel), nlam_inet_chain_supported (rule 2 on
one node set) and nlam_encode_supported (the g2m call with the encoder's projections takes tc_edge_bcast_kernel).  An edge
pointer that is not 16-byte aligned is an error on every row, never a fall-back.
"""
import ctypes

import pytest
import torch

import neural_lam_b200 as nlb
from neural_lam_b200 import _lib, ops

pytestmark = pytest.mark.gpu
DEV = "cuda"
H = 64
E_INVALID = 1  # NLAM_E_INVALID


def _random_graph(ns, nr, ne, seed):
    g = torch.Generator().manual_seed(seed)
    ei = torch.stack([torch.randint(0, ns, (ne,), generator=g), torch.randint(0, nr, (ne,), generator=g)])
    ei[0, -1], ei[1, -1] = ns - 1, nr - 1  # exactly ns senders and nr receivers
    return ei[:, torch.sort(ei[1], stable=True).indices]


def _uniform_graph(ns, nr, d, seed):
    g = torch.Generator().manual_seed(seed)
    snd = torch.randint(0, ns, (nr * d,), generator=g)
    snd[0] = ns - 1
    return torch.stack([snd, torch.arange(nr).repeat_interleave(d)])


def _mlps(seed):
    torch.manual_seed(seed)
    return nlb.make_mlp([3 * H, H, H]).to(DEV), nlb.make_mlp([2 * H, H, H]).to(DEV)


SPLIT = ["tc_rowlinear_kernel", None, "tc_rowmlp_kernel"]  # None: the split-form label

CASES = [
    # name, graph (kind, ns, nr, E or d), B, senders are the receivers, receivers / edges shared by the batch,
    # update_edges, edge_inplace; expected label, inplace, chain, encode
    ("ell_b2", ("uniform", 500, 300, 4), 2, False, False, False, False, "tc_ell_window_kernel", 0, 0, 0),
    ("ell_shared_b2", ("uniform", 500, 300, 4), 2, False, True, False, False, "tc_ell_window_kernel", 0, 0, 0),
    ("ell_b1", ("uniform", 500, 300, 4), 1, False, False, False, False, "tc_ell_window_kernel", 0, 0, 0),
    # one node set, 2400 edge rows >= 2.5 x 800 node rows: rule 2 answers the in-place and chain queries
    ("ell_one_node_set", ("uniform", 200, 200, 6), 2, True, False, False, False, "tc_ell_window_kernel", 1, 1, 0),
    ("ell_graph_edge_out", ("uniform", 200, 200, 6), 2, True, False, True, False, "tc_edge3_kernel", 1, 1, 0),
    # 1000 edge rows = 2.5 x 400 node rows / 999 below
    ("at_threshold_b1", ("random", 200, 200, 1000), 1, False, False, True, False, "tc_edge3_kernel", 1, 1, 0),
    ("below_threshold_b1", ("random", 200, 200, 999), 1, False, False, True, False, "tc_edge_kernel", 0, 0, 1),
    ("below_threshold_b1_no_edge_out", ("random", 200, 200, 999), 1, False, False, False, False,
     "tc_edge_bcast_kernel", 0, 0, 1),
    # mesh-like: 7800 edge rows >= 2.5 x 1800 node rows
    ("mesh_inplace_b3", ("random", 300, 300, 2600), 3, True, False, True, True, "tc_edge_rmw_kernel", 1, 1, 0),
    ("mesh_out_of_place_b3", ("random", 300, 300, 2600), 3, True, False, True, False, "tc_edge3_kernel", 1, 1, 0),
    ("mesh_no_edge_out_b3", ("random", 300, 300, 2600), 3, True, False, False, False, "tc_edge_rmw_kernel", 1, 1, 0),
    ("mesh_shared_edges_b3", ("random", 300, 300, 2600), 3, True, "edge", True, False, "tc_edge3_kernel", 0, 1, 0),
    # shared receivers count once: 2800 edge rows >= 2.5 x (800 + 200); dense receivers: 2800 < 2.5 x 1600
    ("shared_rec_above_b4", ("random", 200, 200, 700), 4, False, True, False, False, "tc_edge_rmw_kernel", 0, 0, 0),
    ("dense_rec_below_b4", ("random", 200, 200, 700), 4, False, "edge", False, False, "tc_edge_kernel", 0, 0, 0),
    # grid -> mesh: 7500 edge rows < 2.5 x (9000 + 200)
    ("g2m_b3", ("random", 3000, 200, 2500), 3, False, True, False, False, "tc_edge_bcast_kernel", 0, 0, 1),
    ("g2m_b1", ("random", 3000, 200, 2500), 1, False, True, False, False, "tc_edge_bcast_kernel", 0, 0, 1),
    ("g2m_dense_edges_b3", ("random", 3000, 200, 2500), 3, False, "rec", False, False, "tc_edge_kernel", 0, 0, 0),
    ("g2m_edge_out_b3", ("random", 3000, 200, 2500), 3, False, True, True, False, "tc_edge_kernel", 0, 0, 1),
]


def _tensors(case, seed=0):
    """send, rec, edge as inet_fwd receives them; the shared column says which of rec / edges are (1, N, 64) expansions"""
    _, (kind, ns, nr, m), B, same, shared = case[:5]
    ne = nr * m if kind == "uniform" else m
    gen = torch.Generator(device=DEV).manual_seed(seed)
    share_rec, share_edge = shared in (True, "rec"), shared in (True, "edge")
    send = torch.randn(B, ns, H, device=DEV, generator=gen)
    rec = send if same else torch.randn(1 if share_rec else B, nr, H, device=DEV, generator=gen).expand(B, -1, -1)
    edge = torch.randn(1 if share_edge else B, ne, H, device=DEV, generator=gen).expand(B, -1, -1)
    return send, rec, edge


def _graph(case):
    kind, ns, nr, m = case[1]
    ei = _uniform_graph(ns, nr, m, 1) if kind == "uniform" else _random_graph(ns, nr, m, 1)
    return ops.Graph(ei, DEV)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_edge_path_selection_and_support_queries(case):
    name, _, B, same, shared, upd, inplace_call, label, want_inplace, want_chain, want_encode = case
    L = _lib.lib()
    g = _graph(case)
    edge_mlp, aggr_mlp = _mlps(0)
    send, rec, edge = _tensors(case)
    edge = edge.contiguous() if inplace_call else edge  # in place needs a tensor of its own
    s, _, sbs = ops.as_rows(send)
    r, _, rbs = ops.as_rows(rec)
    e, _, ebs = ops.as_rows(edge)
    assert g.n_send == send.shape[1] and g.n_rec == rec.shape[1]
    assert (g.uniform_degree != 0) == (case[1][0] == "uniform")
    em, am = ops.mlp_struct(edge_mlp), ops.mlp_struct(aggr_mlp)

    with torch.no_grad(), ops.profile_launches() as prof:
        ops.inet_fwd(g, edge_mlp, aggr_mlp, send, rec, edge, upd, 0, edge_inplace=inplace_call)
    want = ["tc_edge_kernel", "tc_rowmlp_kernel"] if label == "tc_edge_kernel" else [n or label for n in SPLIT]
    assert prof.names() == want, prof.names()

    got_inplace = L.nlam_inet_inplace_supported(g.handle, ctypes.byref(em), s.data_ptr(), sbs, r.data_ptr(), rbs, e.data_ptr(),
                                                ebs, B, 0)
    assert got_inplace == want_inplace
    for nxt in (None, edge_mlp):  # a consumer of the previous layer's projections; a producer of the next layer's too
        assert ops.inet_chain_supported(g, edge_mlp, aggr_mlp, nxt, rec, 0) == bool(want_chain)

    # the encoder's g2m call: send = its P_s (B, n_send, 64) dense, rec = the mesh, edge = the g2m edge features
    embed_mlp, grid_mlp = nlb.make_mlp([H, H, H]).to(DEV), nlb.make_mlp([H, H, H]).to(DEV)
    grid = torch.randn(B, g.n_send, H, device=DEV)
    src = (_lib.NlamRowSrc * 1)()
    src[0].ptr, src[0].idx, src[0].bstride, src[0].dim = grid.data_ptr(), None, g.n_send * H if B > 1 else 0, H
    grid_rep = torch.empty(B, g.n_send, H, device=DEV)
    proj = torch.empty((B * g.n_send + g.n_rec) * H, device=DEV)
    got_encode = L.nlam_encode_supported(g.handle, ctypes.byref(ops.mlp_struct(embed_mlp)), src, 1,
                                         ctypes.byref(ops.mlp_struct(grid_mlp)), ctypes.byref(em), None, r.data_ptr(), rbs,
                                         e.data_ptr(), ebs, grid_rep.data_ptr(), proj.data_ptr(), None, None, g.n_send, B, 0)
    assert got_encode == want_encode

    # the same call with an edge pointer one float past a 16-byte boundary
    ws_bytes = L.nlam_inet_workspace_bytes(g.handle, B, H, _lib.HINT_ONE_HIDDEN)
    ws = torch.empty(ws_bytes, device=DEV, dtype=torch.uint8)
    e_rows = e.shape[0] if e.dim() == 3 and ebs else 1
    odd = torch.zeros(e_rows * g.n_edges * H + 4, device=DEV)
    rec_out = torch.empty(B, g.n_rec, H, device=DEV)
    edge_out = torch.empty(B, g.n_edges, H, device=DEV) if upd else None
    rc = L.nlam_inet_fwd(g.handle, ctypes.byref(em), ctypes.byref(am), s.data_ptr(), sbs, r.data_ptr(), rbs,
                         odd.data_ptr() + 4, ebs, rec_out.data_ptr(), edge_out.data_ptr() if upd else None, None, B, 0,
                         ws.data_ptr(), ws_bytes, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == E_INVALID, (rc, L.nlam_last_error())
    torch.cuda.synchronize()


def test_chained_call_on_uniform_degree_graph_computes_its_own_projections():
    """On one node set with uniform in-degree (d = 6: rule 2 holds, so the chain queries say yes), a chained layer without
    edge output takes tc_ell_window_kernel, which ignores proj_in and launches its own projection pass; its outputs equal
    those of the unchained call bit for bit."""
    case = ("chain", ("uniform", 200, 200, 6), 2, True, False)
    g = _graph(case)
    x, _, e = _tensors(case, seed=3)
    first, last = _mlps(1), _mlps(2)
    assert ops.inet_chain_supported(g, *first, last[0], x, 0) and ops.inet_chain_supported(g, *last, None, x, 0)
    with torch.no_grad():
        with ops.profile_launches() as prof:
            x1, e1, _, proj = ops.inet_fwd(g, *first, x, x, e, True, 0, next_edge_seq=last[0])
        assert prof.names() == ["tc_rowlinear_kernel", "tc_edge3_kernel", "tc_node_proj_kernel"], prof.names()
        with ops.profile_launches() as prof:
            chained = ops.inet_fwd(g, *last, x1, x1, e1, False, 0, proj_in=proj)[0]
        assert prof.names() == ["tc_rowlinear_kernel", "tc_ell_window_kernel", "tc_rowmlp_kernel"], prof.names()
        plain = ops.inet_fwd(g, *last, x1, x1, e1, False, 0)[0]
    assert torch.equal(chained, plain)
