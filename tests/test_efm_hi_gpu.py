"""Graph-EFM on a hierarchical mesh (``models.GraphEFM``) on the GPU (`-m gpu`).  Reads only the golden vectors.

* every golden case (reference GraphEFM, stored noise) within DESIGN §2's bound of the fp64 oracle run on the GPU,
  max |err| <= max(3 x the reference's own TF32 error, 4e-3): the prediction, its std and the posterior through the composed
  path; case (a)'s parameter gradients within 2e-2 max|g| + 1e-4 of the reference's;
* the launch list of the fused step (at the real size): ``tc_encode2_kernel`` first, one ``tc_latent_kernel``,
  ``tc_decode_kernel``, and no projection launch over grid rows besides the decoder's m2g projections;
* ``nlam_encode_fwd`` with a second g2m edge MLP (tc_encode2_kernel): grid_rep and the first layer's projections equal
  those of the one-layer call, the second layer's equal the projections its own g2m call computes (tc_rowlinear_kernel) on
  the stored grid embedding, bit for bit, and both layers' outputs equal their plain forward; a null argument, or a second
  edge MLP together with grid_emb, returns NLAM_E_INVALID; its outputs are closer to TF32 operands rounded to nearest than
  to truncated ones;
* the stacked path that keeps its edge output (``GNNSequential(keep_stacked=True)``) equals the per-layer ``forward``;
* with the same noise the eager ``forward``, ``forward_with_boundary`` and a CUDA-graph replay are bit-identical; replays
  after the same ``torch.cuda.manual_seed`` are bit-identical, members started from one state differ;
* batch independence and one step at the real size of the MEPS hierarchy (268 x 238 grid, 4 levels) against the fp64 oracle.
"""
import ctypes

import pytest
import torch

import neural_lam_b200 as nlb
from efm_hi_golden_util import load_efm_hi_cases, oracle_cfg, oracle_graph, to_device
from neural_lam_b200 import _lib, models, ops, synthetic
from neural_lam_b200.networks import GNNSequential, make_mlp
from oracle import efm_hi_port
from oracle import reference_port as rp
from test_tf32_rounding_gpu import ABS_TOL, RATIO, _inputs as _tailed_inputs, _tail_params

pytestmark = pytest.mark.gpu
DEV = "cuda"
CASES = load_efm_hi_cases()


def _bound(got, want64, tf32):
    err = (got.double() - want64).abs().max().item()
    ref = (tf32.double() - want64).abs().max().item()
    return err, ref, max(3 * ref, 4e-3)


def _d(t):
    return None if t is None else t.to(DEV)


def _to_dev(case):
    _, ds, model = case.build()
    params = {k: v.clone() for k, v in case.params.items()}
    _, g, cfg = case.oracle_inputs(model, ds)
    g, cfg = to_device(g, cfg, DEV)
    return model.to(DEV).eval(), ds, params, g, cfg


def _p(params, dtype=None):
    return {k: (v.to(DEV, dtype) if dtype is not None and v.is_floating_point() else v.to(DEV)) for k, v in params.items()}


def _check_fused_launches(prof, G):
    """tc_encode2_kernel first, one tc_latent_kernel, tc_decode_kernel, and no projection launch over grid rows besides the
    decoder's m2g projections (the tc_rowlinear_kernel right before tc_decode_kernel)"""
    names = prof.names()
    assert names[0] == "tc_encode2_kernel", names
    assert names.count("tc_latent_kernel") == 1 and "tc_decode_kernel" in names, names
    dec = names.index("tc_decode_kernel")
    for i, (n, _, nbytes) in enumerate(prof.rows):
        if n == "tc_rowlinear_kernel" and i != dec - 1:
            assert nbytes < 8 * 64 * G, (i, nbytes, names)


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_efm_hi_golden_cases_meet_bound(case):
    model, ds, params, g, cfg = _to_dev(case)
    x = [_d(t) for t in (case.prev_state, case.prev_prev_state, case.forcing, case.eps)]
    with torch.no_grad():
        model.static_embeddings()  # the weight-only embeddings are cached outside the step
        with ops.profile_launches() as prof:
            pred, std = model(*x[:3], latent_noise=x[3])
    if case.name == "efm_hi_iso_h64":
        # the grid of this case has one grid node without a g2m edge, which the fused encoder does not cover (its senders
        # must be every grid row): the grid side composes; the launch list of the fused step is pinned at the real size
        assert prof.names().count("tc_latent_kernel") == 1, prof.names()
    p64, p32 = _p(params, torch.float64), _p(params)
    want = efm_hi_port.efm_hi_step(p64, g, cfg, *[t.double() for t in x[:3]], x[3].double())
    with rp.tf32_matmul():
        tf32 = efm_hi_port.efm_hi_step(p32, g, cfg, *x)
    err, ref, bound = _bound(pred, want["pred"], tf32["pred"])
    assert err <= bound, (err, ref, bound)
    assert (case.pred.to(DEV).double() - want["pred"]).abs().max().item() <= bound
    if case.pred_std is not None:
        err, ref, bound = _bound(std, want["pred_std"], tf32["pred_std"])
        assert err <= bound, (err, ref, bound)
    # the posterior (autograd-capable composed path)
    with torch.no_grad():
        grid_cur = model.embedd_grid_with_target(*x[:3], _d(case.target))
        post = model.encoder(grid_cur, graph_emb=model._graph_emb(x[0].shape[0]))
    pm64, ps64 = efm_hi_port.efm_hi_posterior(p64, g, cfg, *[t.double() for t in x[:3]], case.target.to(DEV).double())
    with rp.tf32_matmul():
        pm32, ps32 = efm_hi_port.efm_hi_posterior(p32, g, cfg, *x[:3], _d(case.target))
    for got, w64, w32 in ((post.mean, pm64, pm32), (post.stddev, ps64, ps32)):
        err, ref, bound = _bound(got, w64, w32)
        assert err <= bound, (err, ref, bound)


def test_efm_hi_gradients_match_reference():
    case = next(c for c in CASES if c.grads)
    model, ds, params, g, cfg = _to_dev(case)
    model.train()
    x = [_d(t) for t in (case.prev_state, case.prev_prev_state, case.forcing)]
    pred, _ = model(*x, latent_noise=_d(case.eps))
    post = model.encoder(model.embedd_grid_with_target(*x, _d(case.target)), graph_emb=model._graph_emb(x[0].shape[0]))
    loss = (pred * _d(case.w_pred)).sum() + (post.mean * _d(case.w_post)).sum() + (post.stddev * _d(case.w_post)).sum()
    loss.backward()
    got = {k: p.grad for k, p in model.named_parameters() if p.grad is not None}
    assert set(got) == set(case.grads)
    for k, want in case.grads.items():
        want = want.to(DEV)
        err = (got[k] - want).abs().max().item()
        assert err <= 2e-2 * want.abs().max().item() + 1e-4, (k, err)


# ------------------------------------------------------------------------------------------------ the two-g2m encoder
def _g2m_pair(G=3000, N=200, E=2500, B=3, tailed=False, seed=1):
    """embedder (56 -> 64 -> 64), grid MLP and two g2m InteractionNets on one receiver-sorted graph whose senders are all G
    grid rows; inputs, receivers (shared by the batch) and edge features (shared)"""
    gen = torch.Generator().manual_seed(seed)
    ei = torch.stack([torch.randint(0, G, (E,), generator=gen), torch.randint(0, N, (E,), generator=gen)])
    ei[0, 0], ei[1, -1] = G - 1, N - 1
    ei = ei[:, torch.sort(ei[1], stable=True).indices]
    torch.manual_seed(seed)
    emb, gm = make_mlp([56, 64, 64]), make_mlp([64, 64, 64])
    a = nlb.InteractionNet(ei, 64, update_edges=False)
    b = nlb.InteractionNet(ei, 64, update_edges=False)
    shapes = [(B, G, 17), (B, G, 17), (B, G, 18), (G, 4), (N, 64), (E, 64)]
    if tailed:
        for i, m in enumerate((emb, gm, a, b)):
            _tail_params(m, 20 + i)
        xs = _tailed_inputs(shapes, 5)
    else:
        with torch.no_grad():
            for m in (emb, gm, a, b):
                for n, p in m.named_parameters():
                    if p.dim() == 1:
                        p.add_(0.1 * torch.randn_like(p))
        xs = [torch.randn(sh, generator=gen) for sh in shapes]
    xs = [t.to(DEV) for t in xs]
    sources = xs[:3] + [xs[3].unsqueeze(0).expand(B, -1, -1)]
    mesh, edge = xs[4].unsqueeze(0).expand(B, -1, -1), xs[5].unsqueeze(0).expand(B, -1, -1)
    return [m.to(DEV) for m in (emb, gm, a, b)], sources, mesh, edge


def _call_projections(net, send, mesh, edge):
    """the g2m call with its own projections (tc_rowlinear_kernel), P_s and P_r read back from its workspace"""
    B = send.shape[0]
    g = net._graph(send.device)
    s, _, sbs = ops.as_rows(send)
    r, _, rbs = ops.as_rows(mesh)
    e, _, ebs = ops.as_rows(edge)
    em, am = ops.mlp_struct(net.edge_mlp), ops.mlp_struct(net.aggr_mlp)
    L = _lib.lib()
    ws_bytes = L.nlam_inet_workspace_bytes(g.handle, B, 64, net._flags() | _lib.HINT_ONE_HIDDEN)
    ws = torch.empty(ws_bytes, device=DEV, dtype=torch.uint8)
    out = torch.empty(B, g.n_rec, 64, device=DEV)
    with ops.profile_launches() as prof:
        _lib.check(L.nlam_inet_fwd(g.handle, ctypes.byref(em), ctypes.byref(am), s.data_ptr(), sbs, r.data_ptr(), rbs,
                                   e.data_ptr(), ebs, out.data_ptr(), None, None, B, net._flags(), ws.data_ptr(), ws_bytes,
                                   ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    assert prof.names() == ["tc_rowlinear_kernel", "tc_edge_bcast_kernel", "tc_rowmlp_kernel"], prof.names()
    agg = (B * g.n_rec * 64 * 4 + 255) // 256 * 256  # workspace: [aggregate | P_s (B) | P_r (1)]
    proj = ws[agg:].view(torch.float32)
    n_ps = B * g.n_send * 64
    return proj[:n_ps].view(B, g.n_send, 64).clone(), proj[n_ps:n_ps + g.n_rec * 64].view(g.n_rec, 64).clone(), out


@pytest.mark.parametrize("B", [1, 3])
def test_encode_two_g2m_equals_the_launches_it_replaces(B):
    (emb, gm, a, b), sources, mesh, edge = _g2m_pair(B=B)
    G, N = sources[0].shape[1], mesh.shape[1]
    g = a._graph(mesh.device)
    with torch.no_grad():
        with ops.profile_launches() as prof:
            grid_rep, (proj, proj_b), no_emb = ops.encode(g, emb, sources, gm, a.edge_mlp, mesh, edge, flags=a._flags(),
                                                          edge_seq_b=b.edge_mlp)
        assert prof.names() == ["tc_encode2_kernel"], prof.names()
        grid_rep0, (proj0,), grid_emb = ops.encode(g, emb, sources, gm, a.edge_mlp, mesh, edge, flags=a._flags(),
                                                   want_emb=True)
        ps_b, pr_b, out_b = _call_projections(b, grid_emb, mesh, edge)
        _, _, out_a = _call_projections(a, grid_emb, mesh, edge)
        with ops.profile_launches() as prof:
            grid_rep2, (rep_a, rep_b), no_emb2 = a.encode_step(emb, gm, sources, mesh, edge, second=b)
        assert prof.names() == ["tc_encode2_kernel", "tc_edge_bcast_kernel", "tc_rowmlp_kernel", "tc_edge_bcast_kernel",
                                "tc_rowmlp_kernel"], prof.names()
    assert no_emb is None and no_emb2 is None
    assert torch.equal(grid_rep, grid_rep0) and torch.equal(proj, proj0)
    assert torch.equal(proj_b[:B * G * 64].view(B, G, 64), ps_b), (proj_b[:B * G * 64].view(B, G, 64) - ps_b).abs().max()
    assert torch.equal(proj_b[B * G * 64:].view(N, 64), pr_b), (proj_b[B * G * 64:].view(N, 64) - pr_b).abs().max()
    assert torch.equal(grid_rep2, grid_rep) and torch.equal(rep_a, out_a) and torch.equal(rep_b, out_b)


def test_encode_two_g2m_abi_checks():
    (emb, gm, a, b), sources, mesh, edge = _g2m_pair(B=1)
    L = _lib.lib()
    em = ops.mlp_struct(emb)
    rc = L.nlam_encode_fwd(None, ctypes.byref(em), None, 0, ctypes.byref(em), ctypes.byref(em), ctypes.byref(em), None, 0, None,
                           0, None, None, None, None, 1, 1, 0, None)
    assert rc == 1  # NLAM_E_INVALID
    g = a._graph(mesh.device)
    # grid_emb is not stored with a second edge MLP: the pair is not supported, and the call is invalid
    G, N = sources[0].shape[1], mesh.shape[1]
    grid_rep, grid_emb = torch.empty(1, G, 64, device=DEV), torch.empty(1, G, 64, device=DEV)
    proj, proj_b = torch.empty((G + N) * 64, device=DEV), torch.empty((G + N) * 64, device=DEV)
    gs, sa, sb = ops.mlp_struct(gm), ops.mlp_struct(a.edge_mlp), ops.mlp_struct(b.edge_mlp)
    args = [g.handle, ctypes.byref(em), ops._row_srcs([ops.as_rows(t) for t in sources]), len(sources), ctypes.byref(gs),
            ctypes.byref(sa), ctypes.byref(sb), mesh[0].data_ptr(), 0, edge[0].data_ptr(), 0, grid_rep.data_ptr(),
            proj.data_ptr(), proj_b.data_ptr(), None, G, 1, 0]
    assert L.nlam_encode_supported(*args) == 1
    args[14] = grid_emb.data_ptr()
    assert L.nlam_encode_supported(*args) == 0
    assert L.nlam_encode_fwd(*args, None) == 1  # NLAM_E_INVALID
    # a second layer whose call does not take the batch-broadcast path (fp32 math) is declined, not approximated
    assert ops.encode(g, emb, sources, gm, a.edge_mlp, mesh, edge, flags=_lib.MATH_FP32, edge_seq_b=b.edge_mlp) is None


def test_encode_two_g2m_rounds_operands_to_nearest():
    """As test_tf32_rounding_gpu.py part B: tailed operands, fp64 references with operands rounded to nearest and truncated."""
    (emb, gm, a, b), sources, mesh, edge = _g2m_pair(G=1500, N=150, E=1400, B=2, tailed=True)
    g = a._graph(mesh.device)
    with torch.no_grad(), ops.profile_launches() as prof:
        grid_rep, projs, _ = ops.encode(g, emb, sources, gm, a.edge_mlp, mesh, edge, flags=_lib.MATH_TF32,
                                        edge_seq_b=b.edge_mlp)
    assert prof.names() == ["tc_encode2_kernel"], prof.names()
    got = [grid_rep, *projs]
    p64 = {f"{n}.{k}": v.detach().double() for n, m in (("e", emb), ("g", gm), ("a", a), ("b", b))
           for k, v in m.state_dict().items()}
    x64 = torch.cat([t.double() for t in sources], dim=-1)
    m64 = mesh[0].double()

    def lin(x, w, bias=None):
        mode = rp._TF32
        y = (rp.round_tf32(x, mode) @ rp.round_tf32(w, mode).t()) if mode else x @ w.t()
        return y if bias is None else y + bias

    def ref():
        ge = rp.mlp(x64, p64, "e")
        rep = ge + rp.mlp(ge, p64, "g")
        outs = [rep.flatten()]
        for n in ("a", "b"):
            w, bias = p64[f"{n}.edge_mlp.0.weight"], p64[f"{n}.edge_mlp.0.bias"]
            outs += [lin(ge, w[:, 64:128]).flatten(), lin(m64, w[:, 128:], bias).flatten()]
        return torch.cat(outs)

    with rp.tf32_matmul(mode="rna"):
        rna = ref()
    with rp.tf32_matmul(mode="rz"):
        rz = ref()
    got = torch.cat([t.double().flatten() for t in got])
    d_rna, d_rz = (got - rna).norm().item(), (got - rz).norm().item()
    err = (got - rna).abs().max().item()
    print(f"\ntc_encode2_kernel: ||got - ref_rna|| / ||got - ref_rz|| = {d_rna / d_rz:.3f}; max |got - ref_rna| {err:.3e}")
    assert err <= ABS_TOL, err
    assert d_rna <= RATIO * d_rz, (d_rna, d_rz)


# ------------------------------------------------------------------------------------------------ kept edge output
@pytest.mark.parametrize("n_layers", [1, 2, 4])
@pytest.mark.parametrize("B", [1, 3])
def test_stack_keeping_edges_equals_forward(n_layers, B):
    spec = synthetic.make_graph_spec(268, 238, hierarchical=True)
    ei = spec["m2m_edge_index"][0]
    ei = ei[:, torch.sort(ei[1], stable=True).indices].long()
    N = int(ei.max()) + 1
    torch.manual_seed(n_layers)
    stack = GNNSequential([nlb.InteractionNet(ei, 64) for _ in range(n_layers)]).to(DEV)
    with torch.no_grad():
        for p in stack.parameters():
            if p.dim() == 1:
                p.add_(0.1 * torch.randn_like(p))
    x = torch.randn(B, N, 64, device=DEV)
    e_static = torch.randn(ei.shape[1], 64, device=DEV).unsqueeze(0).expand(B, -1, -1)
    e_keep = e_static.clone()
    with torch.no_grad():
        want_x, want_e = x, e_static
        for i in range(n_layers):
            want_x, want_e = stack[i](want_x, want_x, want_e)
        got_x, got_e = stack(x, e_static, keep_stacked=True)
    assert torch.equal(e_static, e_keep)  # the caller's edge tensor is never written
    assert got_e is not e_static and got_e.shape == (B, ei.shape[1], 64)
    assert torch.equal(got_x, want_x), (got_x - want_x).abs().max().item()
    assert torch.equal(got_e, want_e), (got_e - want_e).abs().max().item()


# ------------------------------------------------------------------------------------------------ sampling, batches, size
def _golden_model():
    case = next(c for c in CASES if c.name == "efm_hi_iso_h64")
    model, ds, _, _, _ = _to_dev(case)
    return model, models.ARForecaster(model, ds).to(DEV)


def _inputs(m, B, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    G, d = m.num_grid_nodes, m.num_state_vars
    f = m.grid_input_dim - 2 * d - m.grid_static_features.shape[1]
    return (torch.randn(B, G, d, device=DEV, generator=gen), torch.randn(B, G, d, device=DEV, generator=gen),
            torch.randn(B, G, f, device=DEV, generator=gen))


def test_eager_boundary_and_graphed_steps_are_identical():
    model, fc = _golden_model()
    B = 3
    prev, prev_prev, forcing = _inputs(model, B, 5)
    bnd = torch.randn_like(prev)
    bufs = fc.capture(B)
    assert bufs["latent_noise"].shape == (B, model.latent_spatial_dim, model.latent_dim)
    fc.set_state(prev_prev, prev)
    bufs["forcing"].copy_(forcing)
    bufs["boundary"].copy_(bnd)
    graphed = fc.replay_step().clone()
    noise = bufs["latent_noise"].clone()
    assert noise.std().item() > 0.5
    with torch.no_grad():
        eager, _ = model(prev, prev_prev, forcing, latent_noise=noise)
        with_bnd = model.forward_with_boundary(prev, prev_prev, forcing, bnd, fc.boundary_mask, latent_noise=noise)
    mixed = fc.boundary_mask * bnd + fc.interior_mask * eager
    assert torch.equal(with_bnd, mixed), (with_bnd - mixed).abs().max().item()
    assert torch.equal(graphed, with_bnd), (graphed - with_bnd).abs().max().item()


def test_graphed_rollouts_reproducible_and_members_differ():
    model, fc = _golden_model()
    B, T = 4, 3
    G, d = model.num_grid_nodes, model.num_state_vars
    init = torch.randn(1, 2, G, d, device=DEV).expand(B, -1, -1, -1).contiguous()
    forc = torch.randn(B, T, G, 6, device=DEV)
    bnd = torch.randn(B, T, G, d, device=DEV)
    fc.capture(B)
    torch.cuda.manual_seed(123)
    a = fc.rollout_graphed(init, forc, bnd)
    torch.cuda.manual_seed(123)
    b = fc.rollout_graphed(init, forc, bnd)
    assert torch.equal(a, b)
    interior = fc.interior_mask.bool().reshape(-1)
    assert (a[0, :, interior] - a[1, :, interior]).abs().max().item() > 1e-3
    torch.cuda.manual_seed(124)
    assert not torch.equal(a, fc.rollout_graphed(init, forc, bnd))


@pytest.fixture(scope="module")
def meps_hi():
    spec = synthetic.make_graph_spec(268, 238, hierarchical=True)
    ds = synthetic.SyntheticDatastore(spec, d_state=17, d_forcing=18, d_static=4, boundary_width=10)
    torch.manual_seed(11)
    m = models.GraphEFM(ds, spec, hidden_dim=64)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if p.dim() == 1 and n.split(".")[-2] == "3":
                p.add_(0.1 * torch.randn_like(p))
    params = {k: v.detach().clone() for k, v in m.state_dict().items()}
    m = m.to(DEV).eval()
    yield m, ds, params
    del m
    torch.cuda.empty_cache()


def test_batch_member_in_a_pair_equals_its_row(meps_hi):
    """A member's row of a B = 32 step equals the member run in a batch of two, bit for bit.  Run alone (B = 1) it equals
    its row bit for bit when the step launches the same kernels at both batch sizes; otherwise it meets the fp64 bound of
    DESIGN §2.  On the MEPS hierarchy the launch lists differ: at B = 1 every input of a layer is shared by the batch, and
    layers fed by per-member tensors at B > 1 (from the prior's and the decoder's g2m onward) may then select another edge
    kernel, whose sums round differently."""
    m = meps_hi[0]
    B = 32
    prev, prev_prev, forcing = _inputs(m, B, 7)
    eps = torch.randn(B, m.latent_spatial_dim, m.latent_dim, device=DEV)
    with torch.no_grad():
        full, _ = m(prev, prev_prev, forcing, latent_noise=eps)
        for b in (0, 17, 31):
            pair = [b, (b + 5) % B]
            with ops.profile_launches() as p2:
                two, _ = m(prev[pair], prev_prev[pair], forcing[pair], latent_noise=eps[pair])
            assert torch.equal(two[:1], full[b:b + 1]), (b, (two[:1] - full[b:b + 1]).abs().max().item())
            with ops.profile_launches() as p1:
                alone, _ = m(prev[b:b + 1], prev_prev[b:b + 1], forcing[b:b + 1], latent_noise=eps[b:b + 1])
            print(f"\nmember {b}: same launches alone and in a pair: {p1.names() == p2.names()}; max |alone - row| "
                  f"{(alone - full[b:b + 1]).abs().max().item():.3e}")
            if p1.names() == p2.names():
                assert torch.equal(alone, full[b:b + 1]), (b, (alone - full[b:b + 1]).abs().max().item())
            else:
                assert (alone - full[b:b + 1]).abs().max().item() <= 4e-3


def test_real_size_step_meets_fp64_bound(meps_hi):
    m, ds, params = meps_hi
    assert [n for n in m.level_mesh_sizes] == [6561, 729, 81, 9]
    B = 2
    prev, prev_prev, forcing = _inputs(m, B, 8)
    eps = torch.randn(B, m.latent_spatial_dim, m.latent_dim, device=DEV)
    with torch.no_grad():
        with ops.profile_launches() as prof:
            got, _ = m(prev, prev_prev, forcing, latent_noise=eps)
    _check_fused_launches(prof, m.num_grid_nodes)
    g, cfg = to_device(oracle_graph(m), oracle_cfg(m, {}), DEV)
    want = efm_hi_port.efm_hi_step(_p(params, torch.float64), g, cfg, prev.double(), prev_prev.double(), forcing.double(),
                                eps.double())["pred"]
    with rp.tf32_matmul():
        tf32 = efm_hi_port.efm_hi_step(_p(params), g, cfg, prev, prev_prev, forcing, eps)["pred"]
    err, ref, bound = _bound(got, want, tf32)
    assert err <= bound, (err, ref, bound)
