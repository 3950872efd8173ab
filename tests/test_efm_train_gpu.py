"""Training Graph-EFM on the GPU (`-m gpu`): the gradient of the ensemble scores (``ens_stats_bwd_kernel``),
``BaseGraphEFM.forward_posterior`` and ``ARForecaster.efm_loss`` (DESIGN §4.5, §4.6).

* score gradients against fp64 (autograd through ``oracle/ensemble_port.py`` where its K² G d pair differences fit, the
  closed form of ``oracle/efm_loss_port.py``, pinned to that autograd on the CPU, elsewhere) for K in {2, 3, 8, 32, 64},
  B in {1, 3}, d in {1, 17}, G in {63 784, 1 001}, random and all-interior masks; odd K read a strided time slice of a
  (B, K, T, G, d) leaf and the gradient lands in that slice only.  Bound per tensor: max |g - g64| <= 1e-5 max |g64| (the
  gradients scale with 1/N ~ 1.6e-5 at MEPS size, so an absolute bound would be vacuous); with only the A or the D
  upstream the signs equal fp64's exactly;
* ties meet the bound, identical members give an exactly 0 s² and D gradient;
* two backward passes are bit-identical, row b of a B = 3 call equals a B = 1 call on its rows;
* with ``requires_grad`` the forward outputs equal the no-grad call bit for bit; K = 65 raises, the C ABI returns
  NLAM_E_UNSUPPORTED for it;
* ``forward_posterior`` on every flat and hierarchical golden case: the posterior against the golden vectors, pred and kl
  against the fp64 port with the same noise, within max(3 x the reference TF32 error, 4e-3);
* ``efm_loss`` (T = 2, K = 2 or 3, pinned noise): the terms within that bound, every parameter's gradient within
  2e-2 max|g| + 1e-4 of fp64 autograd through the port, no library GEMM launched where the library's MLP backward covers
  the width (the two H = 64 cases; the H = 16 constant-prior case takes the ATen MLP backward every H = 16 model takes);
* 20 AdamW steps on one batch lower the loss, and the captured step graphs follow the updated weights.
"""
import ctypes

import pytest
import torch

from efm_golden_util import load_efm_cases
from efm_hi_golden_util import load_efm_hi_cases, to_device
from neural_lam_b200 import _lib, ensemble, models
from oracle import efm_loss_port as lp
from oracle import ensemble_port as ep
from oracle import reference_port as rp

pytestmark = pytest.mark.gpu
DEV = "cuda"
QUANTITIES = ("se", "var", "abs_err", "pair_diff")
FLAT = {c.name: c for c in load_efm_cases()}
HI = {c.name: c for c in load_efm_hi_cases()}


# ------------------------------------------------------------------------------------------------ score gradients
def _leaf(B, K, G, d, seed, strided):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    shape = (B, K, 3, G, d) if strided else (B, K, G, d)
    leaf = (torch.randn(*shape, device=DEV, generator=gen) * 0.7 + 0.3).requires_grad_()
    y = torch.randn(B, G, d, device=DEV, generator=gen)
    w = torch.randn(B, d, 4, device=DEV, generator=gen)
    return leaf, y, w


def _members(leaf, strided):
    return leaf[:, :, 1] if strided else leaf


def _grad(leaf, strided, mask, y, w):
    leaf.grad = None
    _, _, sc = ensemble.ensemble_stats(_members(leaf, strided), mask, y)
    (torch.stack([getattr(sc, q) for q in QUANTITIES], dim=-1) * w).sum().backward()
    return leaf.grad


def _grad64(x, mask, y, w):
    B, K, G, d = x.shape
    if B * K * K * G * d <= 2 ** 27:  # autograd through the port keeps K (B, K, G, d) pair differences
        x64 = x.detach().double().requires_grad_()
        _, _, means = ep.ensemble_stats(x64, mask, y)
        (means * w.double()).sum().backward()
        return x64.grad
    return lp.ensemble_stats_grad(x.detach(), mask, y, w)


def _check_grad(leaf, strided, mask, y, w, label):
    g = _grad(leaf, strided, mask, y, w)
    x = _members(leaf, strided)
    if strided:  # the gradient lands in the slice only
        assert torch.count_nonzero(g[:, :, 0]) == 0 and torch.count_nonzero(g[:, :, 2]) == 0
        g = g[:, :, 1]
    want = _grad64(x, mask, y, w)
    err = (g.double() - want).abs().max().item()
    scale = want.abs().max().item()
    print(f"GRADERR {label}: max |g - g64| {err:.2e}, max |g64| {scale:.2e}, relative {err / scale:.2e}")
    assert err <= 1e-5 * scale, (err, scale)
    for q in (2, 3):  # a pure sign term: the signs agree with fp64 exactly
        wq = torch.zeros_like(w)
        wq[..., q] = w[..., q]
        gq = _grad(leaf, strided, mask, y, wq)
        gq = gq[:, :, 1] if strided else gq
        assert torch.equal(torch.sign(gq).double(), torch.sign(_grad64(x, mask, y, wq))), (label, q)


@pytest.mark.parametrize("G", [63784, 1001])
@pytest.mark.parametrize("d", [1, 17])
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("K", [2, 3, 8, 32, 64])
def test_score_grads_vs_fp64(K, B, d, G):
    strided = K % 2 == 1
    leaf, y, w = _leaf(B, K, G, d, seed=K * 1000 + B * 100 + d, strided=strided)
    mask = torch.rand(G, device=DEV, generator=torch.Generator(device=DEV).manual_seed(G)) > 0.3
    _check_grad(leaf, strided, mask, y, w, f"K={K} B={B} d={d} G={G}")


@pytest.mark.parametrize("K", [2, 32])
def test_score_grads_all_interior(K):
    G, d, B = 63784, 17, 3
    leaf, y, w = _leaf(B, K, G, d, seed=K, strided=False)
    _check_grad(leaf, False, torch.ones(G, device=DEV), y, w, f"all-interior K={K}")


def test_score_grads_ties():
    B, K, G, d = 2, 8, 1001, 17
    leaf, y, w = _leaf(B, K, G, d, seed=4, strided=False)
    with torch.no_grad():
        leaf[:, 4:] = leaf[:, :4]  # every member has a twin
        leaf[:, 0, :50] = y[:, :50]  # a member equal to the target
        leaf[:, :, 100:200] = leaf[:, :1, 100:200].round()  # all members equal on these nodes
    mask = torch.rand(G, device=DEV, generator=torch.Generator(device=DEV).manual_seed(5)) > 0.5
    _check_grad(leaf, False, mask, y, w, "ties")
    # identical members: the s² and D gradients are exactly 0
    same = leaf[:, :1].detach().expand(B, K, G, d).contiguous().requires_grad_()
    for q in (1, 3):
        wq = torch.zeros_like(w)
        wq[..., q] = w[..., q]
        g = _grad(same, False, mask, y, wq)
        assert torch.count_nonzero(g) == 0, q


def test_score_grads_deterministic_and_batch_independent():
    B, K, G, d = 3, 32, 63784, 17
    leaf, y, w = _leaf(B, K, G, d, seed=9, strided=True)
    mask = torch.rand(G, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1)) > 0.2
    a = _grad(leaf, True, mask, y, w).clone()
    b = _grad(leaf, True, mask, y, w).clone()
    assert torch.equal(a, b)
    for i in range(B):
        row = leaf[i:i + 1].detach().clone().requires_grad_()
        assert torch.equal(_grad(row, True, mask, y[i:i + 1], w[i:i + 1])[0], a[i]), i


def test_forward_unchanged_and_errors():
    B, K, G, d = 3, 8, 63784, 17
    leaf, y, _ = _leaf(B, K, G, d, seed=2, strided=True)
    mask = torch.rand(G, device=DEV) > 0.3
    with torch.no_grad():
        want = ensemble.ensemble_stats(leaf[:, :, 1], mask, y)
    got = ensemble.ensemble_stats(leaf[:, :, 1], mask, y)
    assert not got[0].requires_grad and not got[1].requires_grad and got[2].se.requires_grad
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    for q in QUANTITIES:
        assert torch.equal(getattr(got[2], q), getattr(want[2], q)), q
    with pytest.raises(ValueError, match="2 <= K <= 64"):
        ensemble.ensemble_stats(torch.zeros(1, 65, 100, 3, device=DEV, requires_grad=True), torch.ones(100, device=DEV),
                                torch.zeros(1, 100, 3, device=DEV))
    x65 = torch.zeros(1, 65, 100, 3, device=DEV)
    gm, out = torch.zeros(1, 3, 4, device=DEV), torch.empty(1, 65, 100, 3, device=DEV)
    t, mk = torch.zeros(1, 100, 3, device=DEV), torch.ones(100, device=DEV)
    rc = _lib.lib().nlam_ensemble_stats_bwd(x65.data_ptr(), x65.stride(0), x65.stride(1), 1, 65, 100, 3, t.data_ptr(), t.stride(0),
                                            mk.data_ptr(), gm.data_ptr(), out.data_ptr(),
                                            ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == _lib.E_UNSUPPORTED


# ------------------------------------------------------------------------------------------------ posterior step
def _bound(got, want64, tf32):
    err = (got.double() - want64).abs().max().item()
    ref = (tf32.double() - want64).abs().max().item()
    return err, ref, max(3 * ref, 4e-3)


def _d(t):
    return None if t is None else t.to(DEV)


def _setup(case):
    _, ds, model = case.build()
    params, g, cfg = case.oracle_inputs(model, ds)
    if case.name in HI:
        g, cfg = to_device(g, cfg, DEV)
    else:
        g = {k: v.to(DEV) for k, v in g.items()}
        if "clamp" in cfg:
            cfg["clamp"] = dict(cfg["clamp"], state_mean=cfg["clamp"]["state_mean"].to(DEV),
                                state_std=cfg["clamp"]["state_std"].to(DEV))
    return model.to(DEV), ds, params, g, cfg


def _p(params, dtype=None):
    return {k: (v.to(DEV, dtype) if dtype is not None and v.is_floating_point() else v.to(DEV)) for k, v in params.items()}


@pytest.mark.parametrize("name", list(FLAT) + list(HI))
def test_forward_posterior_golden_cases(name):
    case = FLAT.get(name) or HI[name]
    hi = name in HI
    model, ds, params, g, cfg = _setup(case)
    x = [_d(t) for t in (case.prev_state, case.prev_prev_state, case.forcing, case.target, case.eps)]
    with torch.no_grad():
        pred, pred_std, kl = model.forward_posterior(*x[:4], latent_noise=x[4])
        post = model.encoder(model.embedd_grid_with_target(*x[:4]), graph_emb=model._graph_emb(x[0].shape[0]))
    assert kl.shape == (case.B,)
    want = lp.posterior_step(_p(params, torch.float64), g, cfg, *[t.double() for t in x], hierarchical=hi)
    with rp.tf32_matmul():
        tf32 = lp.posterior_step(_p(params), g, cfg, *x, hierarchical=hi)
    checks = [("post_mean", post.mean, case.post_mean), ("post_std", post.stddev, case.post_std), ("pred", pred, None),
              ("kl", kl, None)]
    if pred_std is not None:
        checks.append(("pred_std", pred_std, None))
    for key, got, golden in checks:
        err, ref, bound = _bound(got, want[key], tf32[key])
        print(f"POSTERR {name} {key}: {err:.2e} (bound {bound:.2e})")
        assert err <= bound, (key, err, ref, bound)
        if golden is not None:  # the reference's own fp32 posterior is within the same bound
            assert (golden.to(DEV).double() - want[key]).abs().max().item() <= bound, key


# ------------------------------------------------------------------------------------------------ objective gradients
def _loss_inputs(model, B, T, K, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    G, d = model.num_grid_nodes, model.num_state_vars
    f = model.grid_input_dim - 2 * d - model.grid_static_features.shape[1]
    r = lambda *s: torch.randn(*s, device=DEV, generator=gen)  # noqa: E731
    lat = (model.latent_spatial_dim, model.latent_dim)
    return dict(init_states=r(B, 2, G, d), forcing_features=r(B, T, G, f), boundary_states=r(B, T, G, d),
                target_states=r(B, T, G, d), per_var_std=0.5 + torch.rand(d, device=DEV, generator=gen),
                latent_noise=(r(T, B, *lat), r(T, B * K, *lat)))


def _cuda_kernel_names(fn):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.key for e in prof.key_averages()]


@pytest.mark.parametrize("name,K", [("efm_iso_h64", 2), ("efm_hi_iso_h64", 3), ("efm_hi_const_h16", 2)])
def test_efm_loss_gradients_vs_fp64(name, K):
    case = FLAT.get(name) or HI[name]
    hi = name in HI
    model, ds, params, g, cfg = _setup(case)
    model.train()
    fc = models.ARForecaster(model, ds).to(DEV)
    B, T = case.B, 2
    inp = _loss_inputs(model, B, T, K, seed=3)
    kw = dict(members=K, kl_weight=0.5, crps_weight=0.3)
    out = {}

    def step():
        model.zero_grad(set_to_none=True)
        out["loss"] = fc.efm_loss(**inp, **kw)
        out["loss"].loss.backward()

    kernels = _cuda_kernel_names(step)
    if model.hidden_dim % 32 == 0:
        # the library's MLP backward covers H = 32k (backward.mlp_supported); the H = 16 constant-prior case composes its MLP
        # backward from ATen, as every H = 16 model does
        bad = [k for k in kernels if any(t in k.lower() for t in ("gemm", "cublas", "cutlass", "gemv"))]
        assert not bad, f"library GEMMs in the training step: {bad}"
    assert "ens_stats_bwd_kernel" in " ".join(kernels), kernels
    res = out["loss"]
    got = {k: p.grad for k, p in model.named_parameters()}
    missing = [k for k, v in got.items() if v is None]
    assert not missing, missing
    assert any(k.startswith("encoder.") for k in got) and any(k.startswith("grid_current_embedder.") for k in got)

    oracle_args = lambda p, cast: dict(  # noqa: E731
        params=p, graph=g, cfg=cfg, init_states=cast(inp["init_states"]), forcing=cast(inp["forcing_features"]),
        boundary=cast(inp["boundary_states"]), target=cast(inp["target_states"]), per_var_std=cast(inp["per_var_std"]),
        boundary_mask=fc.boundary_mask, post_eps=cast(inp["latent_noise"][0]), prior_eps=cast(inp["latent_noise"][1]),
        hierarchical=hi, **kw)
    p64 = {k: (v.to(DEV, torch.float64).requires_grad_() if v.is_floating_point() else v.to(DEV)) for k, v in params.items()}
    want = lp.efm_loss(**oracle_args(p64, lambda t: t.double()))
    want["loss"].backward()
    with torch.no_grad(), rp.tf32_matmul():
        tf32 = lp.efm_loss(**oracle_args(_p(params), lambda t: t))
    for key in ("loss", "recon", "kl", "crps"):
        err, ref, bound = _bound(getattr(res, key).detach(), want[key].detach(), tf32[key])
        print(f"LOSSERR {name} {key}: {err:.2e} (bound {bound:.2e})")
        assert err <= bound, (key, err, ref, bound)
    worst = 0.0
    for k, gk in got.items():
        w64 = p64[k].grad
        assert w64 is not None, k
        err = (gk.double() - w64).abs().max().item()
        bound = 2e-2 * w64.abs().max().item() + 1e-4
        worst = max(worst, err / bound)
        assert err <= bound, (k, err, bound)
    print(f"LOSSGRAD {name}: {len(got)} parameters, worst error / bound {worst:.2f}")


def test_efm_loss_argument_checks():
    case = FLAT["efm_iso_h64"]
    model, ds, _, _, _ = _setup(case)
    fc = models.ARForecaster(model, ds).to(DEV)
    inp = _loss_inputs(model, 2, 1, 2, seed=1)
    with pytest.raises(ValueError, match="members"):
        fc.efm_loss(**inp, members=65, crps_weight=0.1)
    with pytest.raises(ValueError, match="per_var_std"):
        fc.efm_loss(**dict(inp, per_var_std=-inp["per_var_std"]))
    with pytest.raises(ValueError, match="target_states"):
        fc.efm_loss(**dict(inp, target_states=inp["target_states"][:, :, :-1]))
    with pytest.raises(ValueError, match="latent_noise"):
        fc.efm_loss(**dict(inp, latent_noise=(inp["latent_noise"][0][:, :1], None)))


# ------------------------------------------------------------------------------------------------ training smoke
def test_adamw_training_lowers_loss_and_graphs_follow_weights():
    case = FLAT["efm_iso_h64"]
    model, ds, _, _, _ = _setup(case)
    fc = models.ARForecaster(model, ds).to(DEV)
    B, T, K = 2, 2, 2
    inp = _loss_inputs(model, B, T, K, seed=11)
    fc.capture(B)  # the step graphs exist before training
    graphs = fc._graph[1]
    opt = torch.optim.AdamW(model.parameters(), lr=1e-3)
    losses = []
    model.train()
    for _ in range(20):
        opt.zero_grad(set_to_none=True)
        res = fc.efm_loss(**inp, members=K, kl_weight=0.5, crps_weight=0.3)
        res.loss.backward()
        opt.step()
        losses.append(res.loss.item())
    print("TRAIN losses", " ".join(f"{v:.4f}" for v in losses))
    assert all(torch.isfinite(torch.tensor(losses))) and losses[-1] < losses[0], losses
    model.eval()
    init, forc, bnd = inp["init_states"], inp["forcing_features"][:, :1], inp["boundary_states"][:, :1]
    out = fc.rollout_graphed(init, forc, bnd)
    assert fc._graph[1] is not graphs  # the updated weights forced a re-capture
    noise = fc._graph[2]["latent_noise"].clone()
    with torch.no_grad():
        want = model.forward_with_boundary(init[:, 1], init[:, 0], forc[:, 0], bnd[:, 0], fc.boundary_mask, latent_noise=noise)
    assert torch.equal(out[:, 0], want), (out[:, 0] - want).abs().max().item()
