"""Graph-EFM on the GPU (`-m gpu`).

* ``tc_latent_kernel`` (prior latent_param_map + reparameterised sample + latent_embedder in one launch) against the
  composed path and the fp64 oracle, isotropic and diagonal, at the real mesh size of BASELINE config 2 (6 561 rows: the
  last 64-row tile is partial) and B = 1, 5, 32.  Bound (DESIGN §2): max |err| vs fp64 <= max(3 x the reference's own TF32
  error, 4e-3).
* shapes the kernel does not cover (latent_dim 32, H = 128, hidden_layers 2, math fp32) compose and meet the same bound;
* ``nlam_encode_fwd`` storing grid_emb: grid_emb equals ``grid_prev_embedder.apply_rows`` bit for bit, its other outputs
  equal those of the call without grid_emb;
* every golden case (reference Graph-EFM, stored noise) within the bound, and the parameter gradients of the case that has
  them within 2e-2 max|g| + 1e-4;
* with the same noise the eager ``forward``, ``forward_with_boundary`` and a CUDA-graph replay are bit-identical; replays
  after the same ``torch.cuda.manual_seed`` are bit-identical, members started from one state differ; a member of a
  B = 32 batch run alone equals its row of the batch; a real-size MEPS step meets the fp64 bound.
"""
import ctypes

import pytest
import torch

from efm_golden_util import load_efm_cases
from neural_lam_b200 import _lib, models, ops, synthetic
from neural_lam_b200.networks import make_mlp
from oracle import efm_port
from oracle import reference_port as rp

pytestmark = pytest.mark.gpu
DEV = "cuda"
CASES = load_efm_cases()


def _bound(got, want64, tf32):
    err = (got.double() - want64).abs().max().item()
    ref = (tf32.double() - want64).abs().max().item()
    return err, ref, max(3 * ref, 4e-3)


def _perturb_ln(mods):
    with torch.no_grad():
        for m in mods:
            for n, p in m.named_parameters():
                if n.split(".")[-2] == "3":  # the LayerNorm of a make_mlp with one hidden layer
                    p.add_(0.1 * torch.randn_like(p))


def _latent_modules(diag, L=64, H=64, hl=1, seed=0):
    torch.manual_seed(seed)
    pm = make_mlp([H] * (hl + 1) + [2 * L if diag else L], layer_norm=False).to(DEV)
    em = make_mlp([L] + [H] * (hl + 1)).to(DEV)
    _perturb_ln([em])
    return pm, em


def _oracle(pm, em, x, eps, diag, hl=1, dtype=torch.float64, tf32=False):
    params = {**{f"p.{k}": v.to(dtype) for k, v in pm.state_dict().items()},
              **{f"e.{k}": v.to(dtype) for k, v in em.state_dict().items()}}
    with rp.tf32_matmul(tf32):
        p = rp.mlp(x.to(dtype), params, "p", hl, layer_norm=False)
        mean, std = efm_port.mean_std(p, "diagonal" if diag else "isotropic")
        return rp.mlp(mean + eps.to(dtype) * std, params, "e", hl)


def _composed(pm, em, x, eps, diag):
    p = pm(x)
    if diag:
        mean, raw = p.chunk(2, dim=-1)
        std = 1e-4 + torch.nn.functional.softplus(raw)
    else:
        mean, std = p, torch.ones_like(p)
    return em.apply_rows([mean + eps * std])


@pytest.mark.parametrize("diag", [False, True], ids=["isotropic", "diagonal"])
@pytest.mark.parametrize("B", [1, 5, 32])
def test_latent_kernel_vs_composed_and_fp64(diag, B):
    N = 6561  # mesh rows of BASELINE config 2; 6561 = 102 x 64 + 33
    pm, em = _latent_modules(diag, seed=B)
    gen = torch.Generator(device=DEV).manual_seed(B)
    x = torch.randn(B, N, 64, device=DEV, generator=gen)
    eps = torch.randn(B, N, 64, device=DEV, generator=gen)
    with torch.no_grad():
        with ops.profile_launches() as prof:
            got = ops.latent_sample(pm, em, x, eps)
        assert got is not None and prof.names() == ["tc_latent_kernel"], prof.names()
        comp = _composed(pm, em, x, eps, diag)
        want = _oracle(pm, em, x, eps, diag)
        tf32 = _oracle(pm, em, x, eps, diag, dtype=torch.float32, tf32=True)
    assert got.shape == (B, N, 64) and torch.isfinite(got).all()
    err, ref, bound = _bound(got, want, tf32)
    assert err <= bound, (err, ref, bound)
    err_c, _, _ = _bound(comp, want, tf32)
    assert err_c <= bound, (err_c, bound)
    assert (got - comp).abs().max().item() <= 2 * bound


def test_latent_kernel_shared_inputs_and_batch_rows():
    """A stride-0 batch expansion of x reads the same rows for every element; each element's output depends only on its
    own rows."""
    pm, em = _latent_modules(True, seed=9)
    x = torch.randn(1, 700, 64, device=DEV)
    eps = torch.randn(4, 700, 64, device=DEV)
    with torch.no_grad():
        full = ops.latent_sample(pm, em, x.expand(4, -1, -1), eps)
        for b in range(4):
            assert torch.equal(ops.latent_sample(pm, em, x, eps[b:b + 1]), full[b:b + 1])


@pytest.mark.parametrize("kind", ["latent32", "h128", "hidden2", "fp32"])
def test_latent_uncovered_shapes_compose(kind):
    """The library declines these shapes (ops.latent_sample -> None); the model composes the step and meets the bound."""
    kw = dict(hidden_dim=64, prior_m2m_layers=1, encoder_m2m_layers=1, decoder_m2m_layers=1)
    if kind == "latent32":
        kw["latent_dim"] = 32
    elif kind == "h128":
        kw["hidden_dim"] = 128
    elif kind == "hidden2":
        kw["hidden_layers"] = 2
    spec = synthetic.make_graph_spec(30, 27, hierarchical=False)
    ds = synthetic.SyntheticDatastore(spec, d_state=5, d_forcing=6, d_static=1, boundary_width=2)
    torch.manual_seed(4)
    m = models.GraphEFMMultiScale(ds, spec, math="fp32" if kind == "fp32" else None, **kw)
    params = {k: v.detach().clone() for k, v in m.state_dict().items()}
    m = m.to(DEV)
    B, G = 2, m.num_grid_nodes
    gen = torch.Generator(device=DEV).manual_seed(1)
    prev, prev_prev = torch.randn(B, G, 5, device=DEV, generator=gen), torch.randn(B, G, 5, device=DEV, generator=gen)
    forcing = torch.randn(B, G, 6, device=DEV, generator=gen)
    eps = torch.randn(B, m.num_mesh_nodes, m.latent_dim, device=DEV, generator=gen)
    with torch.no_grad():
        with ops.profile_launches() as prof:
            got, _ = m(prev, prev_prev, forcing, latent_noise=eps)
    assert "tc_latent_kernel" not in prof.names(), prof.names()
    g = {k: getattr(m, k).detach() for k in ("grid_static_features", "g2m_features", "m2g_features", "g2m_edge_index",
                                              "m2g_edge_index", "diff_std", "diff_mean", "m2m_features", "m2m_edge_index",
                                              "mesh_static_features")}
    cfg = dict(hidden_layers=kw.get("hidden_layers", 1), prior_m2m_layers=1, encoder_m2m_layers=1, decoder_m2m_layers=1,
               num_mesh_nodes=m.num_mesh_nodes, latent_dim=m.latent_dim)
    p64 = {k: v.to(DEV, torch.float64) if v.is_floating_point() else v.to(DEV) for k, v in params.items()}
    p32 = {k: v.to(DEV) for k, v in params.items()}
    want = efm_port.efm_step(p64, g, cfg, prev.double(), prev_prev.double(), forcing.double(), eps.double())["pred"]
    with rp.tf32_matmul(kind != "fp32"):
        tf32 = efm_port.efm_step(p32, g, cfg, prev, prev_prev, forcing, eps)["pred"]
    err, ref, bound = _bound(got, want, tf32)
    assert err <= bound, (err, ref, bound)


@pytest.fixture(scope="module")
def config2():
    spec = synthetic.make_graph_spec(268, 238, hierarchical=False)
    ds = synthetic.SyntheticDatastore(spec, d_state=17, d_forcing=18, d_static=4, boundary_width=10)
    torch.manual_seed(11)
    m = models.GraphEFMMultiScale(ds, spec, hidden_dim=64).to(DEV).eval()
    _perturb_ln([m])
    params = {k: v.detach().clone() for k, v in m.state_dict().items()}
    fc = models.ARForecaster(m, ds).to(DEV)
    yield m, ds, fc, params
    del m, fc
    torch.cuda.empty_cache()


def _inputs(m, B, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    G, d = m.num_grid_nodes, m.num_state_vars
    f = m.grid_input_dim - 2 * d - m.grid_static_features.shape[1]
    return (torch.randn(B, G, d, device=DEV, generator=gen), torch.randn(B, G, d, device=DEV, generator=gen),
            torch.randn(B, G, f, device=DEV, generator=gen))


def test_encode_grid_emb_outputs(config2):
    m = config2[0]
    B = 3
    prev, prev_prev, forcing = _inputs(m, B, 1)
    sources = m._grid_sources(prev, prev_prev, forcing)
    ge = m._graph_emb(B)
    net = m.prior_model.g2m_gnn
    g = net._graph(prev.device)
    with torch.no_grad():
        with ops.profile_launches() as prof:
            grid_rep, (proj,), grid_emb = ops.encode(g, m.grid_prev_embedder, sources, m.decoder.grid_update_mlp, net.edge_mlp,
                                                     ge["mesh"], ge["g2m"], flags=net._flags(), want_emb=True)
        assert prof.names() == ["tc_encode_kernel"], prof.names()
        grid_rep0, (proj0,), no_emb = ops.encode(g, m.grid_prev_embedder, sources, m.decoder.grid_update_mlp, net.edge_mlp,
                                                 ge["mesh"], ge["g2m"], flags=net._flags())
        want_emb = m.grid_prev_embedder.apply_rows(sources)
    assert no_emb is None
    assert torch.equal(grid_emb, want_emb), (grid_emb - want_emb).abs().max().item()
    assert torch.equal(grid_rep, grid_rep0) and torch.equal(proj, proj0)


def test_encode_grid_emb_abi_checks(config2):
    m = config2[0]
    em = ops.mlp_struct(m.grid_prev_embedder)
    rc = _lib.lib().nlam_encode_fwd(None, ctypes.byref(em), None, 0, ctypes.byref(em), ctypes.byref(em), None, None, 0, None, 0,
                                    None, None, None, None, 1, 1, 0, None)
    assert rc == 1  # NLAM_E_INVALID


def _to_dev(case):
    spec, ds, model = case.build()
    params = {k: v.clone() for k, v in case.params.items()}
    _, g, cfg = case.oracle_inputs(model, ds)
    if "clamp" in cfg:
        cfg["clamp"] = dict(cfg["clamp"], state_mean=cfg["clamp"]["state_mean"].to(DEV), state_std=cfg["clamp"]["state_std"].to(DEV))
    return model.to(DEV).eval(), ds, params, g, cfg


def _d(t):
    return None if t is None else t.to(DEV)


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_efm_golden_cases_meet_bound(case):
    model, ds, params, g, cfg = _to_dev(case)
    x = [_d(t) for t in (case.prev_state, case.prev_prev_state, case.forcing, case.eps)]
    with torch.no_grad():
        with ops.profile_launches() as prof:
            pred, std = model(*x[:3], latent_noise=x[3])
    if case.name == "efm_iso_h64":
        assert prof.names().count("tc_latent_kernel") == 1, prof.names()
    g = {k: v.to(DEV) for k, v in g.items()}
    p64 = {k: v.to(DEV, torch.float64) if v.is_floating_point() else v.to(DEV) for k, v in params.items()}
    p32 = {k: v.to(DEV) for k, v in params.items()}
    want = efm_port.efm_step(p64, g, cfg, *[t.double() for t in x[:3]], x[3].double())
    with rp.tf32_matmul():
        tf32 = efm_port.efm_step(p32, g, cfg, *x)
    err, ref, bound = _bound(pred, want["pred"], tf32["pred"])
    assert err <= bound, (err, ref, bound)
    # the golden prediction itself (reference fp32 on the CPU) is within the same bound of the fp64 oracle
    assert (case.pred.to(DEV).double() - want["pred"]).abs().max().item() <= bound
    if case.pred_std is not None:
        err, ref, bound = _bound(std, want["pred_std"], tf32["pred_std"])
        assert err <= bound, (err, ref, bound)
    # the posterior (autograd-capable composed path)
    with torch.no_grad():
        grid_cur = model.embedd_grid_with_target(*x[:3], _d(case.target))
        post = model.encoder(grid_cur, graph_emb=model._graph_emb(x[0].shape[0]))
    pm64, ps64 = efm_port.efm_posterior(p64, g, cfg, *[t.double() for t in x[:3]], case.target.to(DEV).double())
    with rp.tf32_matmul():
        pm32, ps32 = efm_port.efm_posterior(p32, g, cfg, *x[:3], _d(case.target))
    for got, w64, w32 in ((post.mean, pm64, pm32), (post.stddev, ps64, ps32)):
        err, ref, bound = _bound(got, w64, w32)
        assert err <= bound, (err, ref, bound)


def test_efm_gradients_match_reference():
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


def _golden_model():
    case = next(c for c in CASES if c.name == "efm_iso_h64")
    model, ds, _, _, _ = _to_dev(case)
    fc = models.ARForecaster(model, ds).to(DEV)
    return model, fc


def test_eager_boundary_and_graphed_steps_are_identical():
    model, fc = _golden_model()
    B = 3
    prev, prev_prev, forcing = _inputs(model, B, 5)
    bnd = torch.randn_like(prev)
    bufs = fc.capture(B)
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
    init = torch.randn(1, 2, G, d, device=DEV).expand(B, -1, -1, -1).contiguous()  # one initial state for every member
    forc = torch.randn(B, T, G, 6, device=DEV)
    bnd = torch.randn(B, T, G, d, device=DEV)
    fc.capture(B)  # outside the seeded sequences: the warm-up steps of a capture draw noise too
    torch.cuda.manual_seed(123)
    a = fc.rollout_graphed(init, forc, bnd)
    torch.cuda.manual_seed(123)
    b = fc.rollout_graphed(init, forc, bnd)
    assert torch.equal(a, b)
    interior = fc.interior_mask.bool().reshape(-1)
    assert (a[0, :, interior] - a[1, :, interior]).abs().max().item() > 1e-3
    torch.cuda.manual_seed(124)
    c = fc.rollout_graphed(init, forc, bnd)
    assert not torch.equal(a, c)


def test_batch_member_alone_equals_its_row(config2):
    """Each member's row of a B = 32 step equals the member run in a batch of two, bit for bit, and the member run alone
    within the fp64 bound.  Alone (B = 1) the decoder's g2m layer has receivers shared by the batch and takes the
    batch-broadcast edge kernel; with B > 1 its receivers (the embedded latent) differ per member and it takes the K = 192 edge
    kernel, whose sums round differently."""
    m = config2[0]
    B = 32
    prev, prev_prev, forcing = _inputs(m, B, 7)
    eps = torch.randn(B, m.num_mesh_nodes, m.latent_dim, device=DEV)
    with torch.no_grad():
        full, _ = m(prev, prev_prev, forcing, latent_noise=eps)
        for b in (0, 17, 31):
            pair = [b, (b + 5) % B]
            two, _ = m(prev[pair], prev_prev[pair], forcing[pair], latent_noise=eps[pair])
            assert torch.equal(two[:1], full[b:b + 1]), (b, (two[:1] - full[b:b + 1]).abs().max().item())
            alone, _ = m(prev[b:b + 1], prev_prev[b:b + 1], forcing[b:b + 1], latent_noise=eps[b:b + 1])
            assert (alone - full[b:b + 1]).abs().max().item() <= 4e-3


def test_real_size_step_meets_fp64_bound(config2):
    m, ds, fc, params = config2
    B = 2
    prev, prev_prev, forcing = _inputs(m, B, 8)
    eps = torch.randn(B, m.num_mesh_nodes, m.latent_dim, device=DEV)
    with torch.no_grad():
        with ops.profile_launches() as prof:
            got, _ = m(prev, prev_prev, forcing, latent_noise=eps)
    names = prof.names()
    assert names.count("tc_latent_kernel") == 1 and names[0] == "tc_encode_kernel", names
    g = {k: getattr(m, k).detach() for k in ("grid_static_features", "g2m_features", "m2g_features", "g2m_edge_index",
                                              "m2g_edge_index", "diff_std", "diff_mean", "m2m_features", "m2m_edge_index",
                                              "mesh_static_features")}
    cfg = dict(hidden_layers=1, prior_m2m_layers=2, encoder_m2m_layers=2, decoder_m2m_layers=4,
               num_mesh_nodes=m.num_mesh_nodes, latent_dim=m.latent_dim)
    p64 = {k: v.to(DEV, torch.float64) if v.is_floating_point() else v.to(DEV) for k, v in params.items()}
    p32 = {k: v.to(DEV) for k, v in params.items()}
    want = efm_port.efm_step(p64, g, cfg, prev.double(), prev_prev.double(), forcing.double(), eps.double())["pred"]
    with rp.tf32_matmul():
        tf32 = efm_port.efm_step(p32, g, cfg, prev, prev_prev, forcing, eps)["pred"]
    err, ref, bound = _bound(got, want, tf32)
    assert err <= bound, (err, ref, bound)
