"""The fused grid encoder (`-m gpu`): tc_encode_kernel computes the grid embedder, the g2m edge MLP's node projections P_s
and P_r, and the encoding grid MLP in one launch, where the step used to run three (tc_rowmlp_kernel for the embedder,
tc_rowlinear_kernel inside the g2m call, tc_rowmlp_kernel for the encoding grid MLP).  It runs the same wgmma shapes in
the same K order and the same fp32 epilogue code on the same fp32 values, so every output must equal the three-launch
composition bit for bit:
  * config 2's graph (MEPS 268x238 grid, 63 784 rows: a partial last 64-row tile) at B = 1, 5 and 32;
  * a 31x26 grid (806 rows, 806 = 2 mod 4): the 16-byte alignment of a 17-wide source's rows of one work item differs
    between batch elements, so odd elements take the element-wise loads; its last tile is partial too;
  * the static source as a stride-0 batch expansion (as the model passes it) and as a dense batched tensor;
  * a whole config 2 step, ``forward_with_boundary`` and the no-grad ``forward``, against the same step with the encoder
    turned off.
Shapes the kernel does not cover return None and the step runs the three launches.
"""
import ctypes

import pytest
import torch

from neural_lam_b200 import _lib, models, ops, synthetic

pytestmark = pytest.mark.gpu
DEV = "cuda"
D_STATE, D_FORCING, D_STATIC = 17, 18, 4


def _model(nx, ny, hidden=64, d_state=D_STATE, d_forcing=D_FORCING, P=4):
    spec = synthetic.make_graph_spec(nx, ny, hierarchical=False)
    ds = synthetic.SyntheticDatastore(spec, d_state=d_state, d_forcing=d_forcing, d_static=D_STATIC, boundary_width=2)
    torch.manual_seed(3)
    m = models.GraphLAM(ds, spec, hidden_dim=hidden, processor_layers=P)
    fc = models.ARForecaster(m, ds).to(DEV).eval()
    return m, fc


@pytest.fixture(scope="module")
def config2():
    m, fc = _model(268, 238)
    yield m, fc
    del m, fc
    torch.cuda.empty_cache()


def _inputs(m, B, seed, dense_static=False):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    G = m.num_grid_nodes
    d = m.num_state_vars
    f = m.grid_input_dim - 2 * d - D_STATIC
    prev, prev_prev = torch.randn(B, G, d, device=DEV, generator=gen), torch.randn(B, G, d, device=DEV, generator=gen)
    forcing = torch.randn(B, G, f, device=DEV, generator=gen)
    static = m.expand_to_batch(m.grid_static_features, B)
    if dense_static:
        static = static.contiguous()
    return [prev, prev_prev, forcing, static]


def _three_launches(m, sources):
    """grid_emb (tc_rowmlp_kernel), the g2m call with its own projections (tc_rowlinear_kernel; P_s and P_r read back from the
    call's workspace) and the encoding grid MLP (tc_rowmlp_kernel) -> P_s, P_r, mesh_rep, grid_rep"""
    net = m.g2m_gnn
    B = sources[0].shape[0]
    st = m.static_embeddings()
    grid_emb = m.grid_embedder.apply_rows(sources)
    g = net._graph(grid_emb.device)
    s, _, sbs = ops.as_rows(grid_emb)
    r, _, rbs = ops.as_rows(m.expand_to_batch(st["mesh_emb"], B))
    e, _, ebs = ops.as_rows(m.expand_to_batch(st["g2m_emb"], B))
    em, am = ops.mlp_struct(net.edge_mlp), ops.mlp_struct(net.aggr_mlp)
    L = _lib.lib()
    ws_bytes = L.nlam_inet_workspace_bytes(g.handle, B, 64, net._flags() | _lib.HINT_ONE_HIDDEN)
    ws = torch.empty(ws_bytes, device=DEV, dtype=torch.uint8)
    mesh_rep = torch.empty(B, g.n_rec, 64, device=DEV)
    with ops.profile_launches() as prof:
        _lib.check(L.nlam_inet_fwd(g.handle, ctypes.byref(em), ctypes.byref(am), s.data_ptr(), sbs, r.data_ptr(), rbs,
                                   e.data_ptr(), ebs, mesh_rep.data_ptr(), None, None, B, net._flags(), ws.data_ptr(), ws_bytes,
                                   ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    assert prof.names() == ["tc_rowlinear_kernel", "tc_edge_bcast_kernel", "tc_rowmlp_kernel"], prof.names()
    agg = (B * g.n_rec * 64 * 4 + 255) // 256 * 256  # workspace: [aggregate | P_s (B) | P_r (1)]
    proj = ws[agg:].view(torch.float32)
    n_ps = B * g.n_send * 64
    ps, pr = proj[:n_ps].view(B, g.n_send, 64), proj[n_ps:n_ps + g.n_rec * 64].view(g.n_rec, 64)
    grid_rep = m.encoding_grid_mlp.apply_rows([grid_emb], res=grid_emb)
    return ps.clone(), pr.clone(), mesh_rep, grid_rep


def _fused(m, sources):
    net = m.g2m_gnn
    B, G = sources[0].shape[0], m.num_grid_nodes
    st = m.static_embeddings()
    mesh, g2m = m.expand_to_batch(st["mesh_emb"], B), m.expand_to_batch(st["g2m_emb"], B)
    g = net._graph(mesh.device)
    with ops.profile_launches() as prof:
        enc = ops.encode(g, m.grid_embedder, sources, m.encoding_grid_mlp, net.edge_mlp, mesh, g2m, flags=net._flags())
    assert enc is not None, "ops.encode does not cover this shape"
    assert prof.names() == ["tc_encode_kernel"], prof.names()
    grid_rep, (proj,), grid_emb = enc
    assert grid_emb is None
    ps, pr = proj[:B * G * 64].view(B, G, 64), proj[B * G * 64:].view(g.n_rec, 64)
    with ops.profile_launches() as prof:
        grid_rep2, (mesh_rep,), grid_emb = net.encode_step(m.grid_embedder, m.encoding_grid_mlp, sources, mesh, g2m)
    assert prof.names() == ["tc_encode_kernel", "tc_edge_bcast_kernel", "tc_rowmlp_kernel"], prof.names()
    assert grid_emb is None
    assert torch.equal(grid_rep2, grid_rep)
    return ps, pr, mesh_rep, grid_rep


def _check_equal(m, sources):
    with torch.no_grad():
        want = _three_launches(m, sources)
        got = _fused(m, sources)
    for name, a, b in zip(("P_s", "P_r", "mesh_rep", "grid_rep"), got, want):
        assert a.shape == b.shape, (name, a.shape, b.shape)
        assert torch.equal(a, b), f"{name}: max |diff| {(a - b).abs().max().item():.3e}"


@pytest.mark.parametrize("B", [1, 5, 32])
def test_fused_encode_config2_equals_three_launches(config2, B):
    m, _ = config2
    assert m.num_grid_nodes % 64 != 0 and m.num_grid_nodes % 4 == 0
    _check_equal(m, _inputs(m, B, seed=B))


@pytest.mark.parametrize("B", [1, 2, 5])
@pytest.mark.parametrize("dense_static", [False, True])
def test_fused_encode_misaligned_spans_and_partial_tile(B, dense_static):
    m, _ = _model(31, 26, P=1)
    assert m.num_grid_nodes % 4 == 2 and m.num_grid_nodes % 64 != 0
    _check_equal(m, _inputs(m, B, seed=10 + B, dense_static=dense_static))


def _step_both_ways(m, fc, B, seed):
    """(forward_with_boundary, no-grad forward) with the encoder and with encode_step returning None, plus launch names"""
    prev, prev_prev, forcing, _ = _inputs(m, B, seed)
    bnd = torch.randn_like(prev)
    res = {}
    with torch.no_grad():
        m.static_embeddings()
        for mode in ("fused", "old"):
            if mode == "old":
                m.g2m_gnn.encode_step = lambda *a, **k: None
            try:
                with ops.profile_launches() as prof:
                    a = m.forward_with_boundary(prev, prev_prev, forcing, bnd, fc.boundary_mask)
                b, _ = m(prev, prev_prev, forcing)
            finally:
                m.g2m_gnn.__dict__.pop("encode_step", None)
            res[mode] = (a, b, prof.names())
    return res


def test_model_step_equals_step_without_encoder(config2):
    m, fc = config2
    res = _step_both_ways(m, fc, 4, seed=7)
    (a, b, names), (a0, b0, names0) = res["fused"], res["old"]
    assert names.count("tc_encode_kernel") == 1 and "tc_encode_kernel" not in names0, (names, names0)
    assert len(names) == len(names0) - 2, (names, names0)
    assert names[:3] == ["tc_encode_kernel", "tc_edge_bcast_kernel", "tc_rowmlp_kernel"], names
    assert torch.equal(a, a0), (a - a0).abs().max().item()
    assert torch.equal(b, b0), (b - b0).abs().max().item()


def test_model_step_launches_same_kernels_at_b1(config2):
    m, fc = config2
    n1 = _step_both_ways(m, fc, 1, seed=8)["fused"][2]
    n32 = _step_both_ways(m, fc, 32, seed=9)["fused"][2]
    assert n1 == n32 and len(n32) == 14, (n1, n32)


def _supported(m, sources, grid_mlp_struct):
    """nlam_encode_supported for the model's g2m call on ``sources`` with the encoding grid MLP given as an NlamMlp"""
    net, B = m.g2m_gnn, sources[0].shape[0]
    st = m.static_embeddings()
    g = net._graph(torch.device(DEV, torch.cuda.current_device()))
    arr = (_lib.NlamRowSrc * len(sources))()
    for i, t in enumerate(sources):
        x, _, bs = ops.as_rows(t)
        arr[i].ptr, arr[i].idx, arr[i].bstride, arr[i].dim = x.data_ptr(), None, bs, x.shape[-1]
    out = torch.empty(B, m.num_grid_nodes, 64, device=DEV)
    proj = torch.empty((B * m.num_grid_nodes + g.n_rec) * 64, device=DEV)
    em, sm = ops.mlp_struct(m.grid_embedder), ops.mlp_struct(net.edge_mlp)
    return _lib.lib().nlam_encode_supported(g.handle, ctypes.byref(em), arr, len(sources), ctypes.byref(grid_mlp_struct),
                                            ctypes.byref(sm), None, st["mesh_emb"].data_ptr(), 0, st["g2m_emb"].data_ptr(), 0,
                                            out.data_ptr(), proj.data_ptr(), None, None, m.num_grid_nodes, B, net._flags())


def test_encode_query_declines_layernorm_without_beta():
    """The kernel reads every bias and LayerNorm parameter: an MLP whose LayerNorm has no shift is not covered."""
    m, _ = _model(31, 26, P=1)
    sources = _inputs(m, 2, seed=4)
    with torch.no_grad():
        gm = ops.mlp_struct(m.encoding_grid_mlp)
        assert _supported(m, sources, gm) == 1
        gm.ln_beta = None
        assert _supported(m, sources, gm) == 0


@pytest.mark.parametrize("kind", ["h128", "wide_input"])
def test_encode_falls_back_where_not_covered(kind):
    """H = 128, or an embedder input wider than 64 columns: ops.encode / encode_step return None and the step runs the three
    launches."""
    if kind == "h128":
        m, fc = _model(30, 27, hidden=128, P=1)
    else:
        m, fc = _model(30, 27, d_state=24, d_forcing=20, P=1)  # 24 + 24 + 20 + 4 = 72 columns
    B = 2
    sources = _inputs(m, B, seed=4)
    net = m.g2m_gnn
    with torch.no_grad():
        st = m.static_embeddings()
        mesh, g2m = m.expand_to_batch(st["mesh_emb"], B), m.expand_to_batch(st["g2m_emb"], B)
        g = net._graph(mesh.device)
        assert ops.encode(g, m.grid_embedder, sources, m.encoding_grid_mlp, net.edge_mlp, mesh, g2m, flags=net._flags()) is None
        assert net.encode_step(m.grid_embedder, m.encoding_grid_mlp, sources, mesh, g2m) is None
        prev, prev_prev, forcing, _ = sources
        with ops.profile_launches() as prof:
            out = m.forward_with_boundary(prev, prev_prev, forcing, torch.randn_like(prev), fc.boundary_mask)
    assert "tc_encode_kernel" not in prof.names(), prof.names()
    assert torch.isfinite(out).all()
