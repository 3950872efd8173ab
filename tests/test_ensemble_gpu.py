"""Ensemble statistics on the GPU (`-m gpu`): ``ens_stats_kernel`` through ``ensemble.ensemble_stats`` and
``ARForecaster.rollout_ensemble`` (DESIGN §4.5).

* ``ensemble_stats`` against the fp64 oracle (``oracle/ensemble_port.py``) for K in {2, 3, 8, 32, 64}, B in {1, 3},
  d in {1, 17}, G = 63 784 (MEPS) and G = 1 001 (the last CTA partial), a random interior mask and an all-interior mask;
  odd K read a strided time slice of a (B, K, T, G, d) tensor.  Bounds: m and s rtol = atol = 2e-5 per element (DESIGN
  §2's exact-fp32 bound); the four interior means relative 1e-5;
* identical members give s = 0 and D = 0 exactly and A = |x - y|; tied members meet the bounds; K = 1, K = 65, CPU and
  float64 tensors raise, and the C ABI returns NLAM_E_UNSUPPORTED for K = 65;
* two calls are bit-identical, and initial condition b of a B = 3 call equals a B = 1 call on its rows bit for bit;
* ``rollout_ensemble`` of GraphEFMMultiScale and GraphEFM equals ``ensemble_stats`` applied per step to ``rollout_graphed``
  on the inputs expanded to B·K rows, bit for bit, after the same ``torch.cuda.manual_seed``; ``rollout_graphed``'s
  capture and results are unaffected;
* GraphEFMMultiScale at MEPS size, K = 32, two steps: the bounds against the fp64 oracle on the expanded members.
"""
import ctypes

import pytest
import torch

from neural_lam_b200 import _lib, ensemble, models, synthetic
from oracle import ensemble_port as ep

pytestmark = pytest.mark.gpu
DEV = "cuda"
QUANTITIES = ("se", "var", "abs_err", "pair_diff")


def _case(B, K, G, d, seed, strided=False):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    if strided:  # a time slice of a stored (B, K, T, G, d) ensemble: member stride T·G·d, batch stride K·T·G·d
        x = torch.randn(B, K, 3, G, d, device=DEV, generator=gen)[:, :, 1]
    else:
        x = torch.randn(B, K, G, d, device=DEV, generator=gen)
    x = x * 0.7 + 0.3
    y = torch.randn(B, G, d, device=DEV, generator=gen)
    return x, y


def _check(x, mask, y, label):
    mean, std, sc = ensemble.ensemble_stats(x, mask, y)
    wm, ws, wq = ep.ensemble_stats(x, mask, y)
    torch.testing.assert_close(mean.double(), wm, rtol=2e-5, atol=2e-5)
    torch.testing.assert_close(std.double(), ws, rtol=2e-5, atol=2e-5)
    got = torch.stack([getattr(sc, q) for q in QUANTITIES], dim=-1).double()
    rel = ((got - wq).abs() / wq.abs().clamp_min(1e-30)).max().item()
    err_m = ((mean.double() - wm).abs() / (2e-5 + 2e-5 * wm.abs())).max().item()
    err_s = ((std.double() - ws).abs() / (2e-5 + 2e-5 * ws.abs())).max().item()
    print(f"ENSERR {label}: m {(mean.double() - wm).abs().max().item():.2e} (bound use {err_m:.2f}), "
          f"s {(std.double() - ws).abs().max().item():.2e} (bound use {err_s:.2f}), means rel {rel:.2e}")
    assert rel < 1e-5, rel
    return mean, std, sc


@pytest.mark.parametrize("G", [63784, 1001])
@pytest.mark.parametrize("d", [1, 17])
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("K", [2, 3, 8, 32, 64])
def test_stats_vs_fp64_oracle(K, B, d, G):
    x, y = _case(B, K, G, d, seed=K * 1000 + B * 100 + d, strided=K % 2 == 1)
    mask = torch.rand(G, device=DEV, generator=torch.Generator(device=DEV).manual_seed(G)) > 0.3
    _check(x, mask, y, f"K={K} B={B} d={d} G={G}")


@pytest.mark.parametrize("K", [2, 32])
def test_stats_all_interior(K):
    G, d, B = 63784, 17, 3
    x, y = _case(B, K, G, d, seed=K)
    _check(x, torch.ones(G, device=DEV), y, f"all-interior K={K}")


def test_identical_members():
    B, K, G, d = 2, 5, 1001, 17
    base, y = _case(B, 1, G, d, seed=3)
    x = base.expand(B, K, G, d)  # member stride 0: every member is the same tensor
    mask = torch.ones(G, device=DEV)
    mean, std, sc = ensemble.ensemble_stats(x, mask, y)
    assert torch.equal(mean, base[:, 0])
    assert torch.equal(std, torch.zeros_like(std))
    assert torch.equal(sc.var, torch.zeros_like(sc.var))
    assert torch.equal(sc.pair_diff, torch.zeros_like(sc.pair_diff))
    want_a = (base[:, 0].double() - y.double()).abs().mean(dim=1)
    torch.testing.assert_close(sc.abs_err.double(), want_a, rtol=1e-5, atol=0)


def test_tied_members():
    B, K, G, d = 2, 8, 1001, 17
    x, y = _case(B, K, G, d, seed=4)
    x = x.clone()
    x[:, 4:] = x[:, :4]  # every member has a twin
    x[:, :, :100] = x[:, :1, :100].round()  # and on the first 100 nodes all members are equal
    _check(x, torch.rand(G, device=DEV) > 0.5, y, "ties")


def test_invalid_arguments_raise():
    G, d = 100, 3
    x, y = _case(1, 4, G, d, seed=0)
    mask = torch.ones(G, device=DEV)
    for K in (1, 65):
        with pytest.raises(ValueError, match="2 <= K <= 64"):
            ensemble.ensemble_stats(torch.zeros(1, K, G, d, device=DEV), mask, y)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ensemble.ensemble_stats(x.cpu(), mask.cpu(), y.cpu())
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ensemble.ensemble_stats(x, mask, y.cpu())
    with pytest.raises(TypeError, match="float32"):
        ensemble.ensemble_stats(x.double(), mask, y)
    with pytest.raises(TypeError, match="float32"):
        ensemble.ensemble_stats(x, mask, y.double())
    # the C ABI itself refuses K outside 2 .. 64
    x65 = torch.zeros(1, 65, G, d, device=DEV)
    mean, std = torch.empty(1, G, d, device=DEV), torch.empty(1, G, d, device=DEV)
    rc = _lib.lib().nlam_ensemble_stats(x65.data_ptr(), x65.stride(0), x65.stride(1), 1, 65, G, d, None, 0, None,
                                        mean.data_ptr(), std.data_ptr(), None, None, 0,
                                        ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == _lib.E_UNSUPPORTED


def test_deterministic_and_batch_independent():
    B, K, G, d = 3, 32, 63784, 17
    x, y = _case(B, K, G, d, seed=9, strided=True)
    mask = torch.rand(G, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1)) > 0.2
    a = ensemble.ensemble_stats(x, mask, y)
    b = ensemble.ensemble_stats(x, mask, y)
    for u, v in ((a[0], b[0]), (a[1], b[1]), (a[2].se, b[2].se), (a[2].var, b[2].var), (a[2].abs_err, b[2].abs_err),
                 (a[2].pair_diff, b[2].pair_diff)):
        assert torch.equal(u, v)
    for i in range(B):
        m1, s1, q1 = ensemble.ensemble_stats(x[i:i + 1], mask, y[i:i + 1])
        assert torch.equal(m1[0], a[0][i]) and torch.equal(s1[0], a[1][i])
        for q in QUANTITIES:
            assert torch.equal(getattr(q1, q)[0], getattr(a[2], q)[i]), (i, q)


# ------------------------------------------------------------------------------------------------------------- rollouts
def _small_forecaster(kind):
    spec = synthetic.make_graph_spec(30, 27, hierarchical=kind == "hi")
    ds = synthetic.SyntheticDatastore(spec, d_state=5, d_forcing=6, d_static=1, boundary_width=2)
    torch.manual_seed(2)
    cls = models.GraphEFM if kind == "hi" else models.GraphEFMMultiScale
    m = cls(ds, spec, hidden_dim=64).to(DEV).eval()
    return m, models.ARForecaster(m, ds).to(DEV)


def _rollout_inputs(m, B, T, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    G, d = m.num_grid_nodes, m.num_state_vars
    f = m.grid_input_dim - 2 * d - m.grid_static_features.shape[1]
    return (torch.randn(B, 2, G, d, device=DEV, generator=gen), torch.randn(B, T, G, f, device=DEV, generator=gen),
            torch.randn(B, T, G, d, device=DEV, generator=gen), torch.randn(B, T, G, d, device=DEV, generator=gen))


def _expand(t, K):
    return t.unsqueeze(1).expand(t.shape[0], K, *t.shape[1:]).reshape(t.shape[0] * K, *t.shape[1:])


@pytest.mark.parametrize("kind", ["multiscale", "hi"])
def test_rollout_ensemble_equals_stats_of_graphed_rollout(kind):
    m, fc = _small_forecaster(kind)
    B, K, T = 2, 4, 3
    init, forc, bnd, tgt = _rollout_inputs(m, B, T, seed=1)
    G, d = m.num_grid_nodes, m.num_state_vars
    ex = [_expand(t, K) for t in (init, forc, bnd)]
    fc.rollout_graphed(*ex)  # capture outside the seeded runs (the warm-up steps draw noise)
    graphs = fc._graph[1]
    torch.cuda.manual_seed(77)
    traj = fc.rollout_graphed(*ex)
    fc.rollout_ensemble(init, forc, bnd, K, targets=tgt)
    torch.cuda.manual_seed(77)
    mean, std, sc = fc.rollout_ensemble(init, forc, bnd, K, targets=tgt)
    assert mean.shape == std.shape == (B, T, G, d) and sc.se.shape == (B, T, d)
    for t in range(T):
        wm, ws, wq = ensemble.ensemble_stats(traj[:, t].view(B, K, G, d), fc.interior_mask, tgt[:, t])
        assert torch.equal(mean[:, t], wm) and torch.equal(std[:, t], ws), t
        for q in QUANTITIES:
            assert torch.equal(getattr(sc, q)[:, t], getattr(wq, q)), (t, q)
    # members really differ, and the mean is not a single member
    assert std[:, :, fc.interior_mask.reshape(-1) > 0].min().item() > 0
    # without targets: its own capture, the same mean and spread
    fc.rollout_ensemble(init, forc, bnd, K)
    torch.cuda.manual_seed(77)
    mean2, std2, none = fc.rollout_ensemble(init, forc, bnd, K)
    assert none is None and torch.equal(mean2, mean) and torch.equal(std2, std)
    # rollout_graphed's capture is neither evicted nor reused for the ensemble's shape, and its results are unchanged
    torch.cuda.manual_seed(77)
    assert torch.equal(fc.rollout_graphed(*ex), traj)
    assert fc._graph[1] is graphs
    # the other batch shape of rollout_graphed is not served by the ensemble capture either
    torch.cuda.manual_seed(77)
    small = fc.rollout_graphed(init, forc, bnd)
    assert small.shape == (B, T, G, d) and fc._graph[0] == B


def test_real_size_rollout_ensemble_vs_fp64():
    spec = synthetic.make_graph_spec(268, 238, hierarchical=False)
    ds = synthetic.SyntheticDatastore(spec, d_state=17, d_forcing=18, d_static=4, boundary_width=10)
    torch.manual_seed(11)
    m = models.GraphEFMMultiScale(ds, spec, hidden_dim=64, prior_m2m_layers=2, decoder_m2m_layers=4).to(DEV).eval()
    fc = models.ARForecaster(m, ds).to(DEV)
    B, K, T = 1, 32, 2
    init, forc, bnd, tgt = _rollout_inputs(m, B, T, seed=5)
    G, d = m.num_grid_nodes, 17
    ex = [_expand(t, K) for t in (init, forc, bnd)]
    fc.rollout_graphed(*ex)
    fc.rollout_ensemble(init, forc, bnd, K, targets=tgt)
    torch.cuda.manual_seed(3)
    traj = fc.rollout_graphed(*ex)
    torch.cuda.manual_seed(3)
    mean, std, sc = fc.rollout_ensemble(init, forc, bnd, K, targets=tgt)
    for t in range(T):
        wm, ws, wq = ep.ensemble_stats(traj[:, t].view(B, K, G, d), fc.interior_mask, tgt[:, t])
        torch.testing.assert_close(mean[:, t].double(), wm, rtol=2e-5, atol=2e-5)
        torch.testing.assert_close(std[:, t].double(), ws, rtol=2e-5, atol=2e-5)
        got = torch.stack([getattr(sc, q)[:, t] for q in QUANTITIES], dim=-1).double()
        rel = ((got - wq).abs() / wq.abs()).max().item()
        print(f"ENSERR real-size rollout step {t}: m {(mean[:, t].double() - wm).abs().max().item():.2e}, "
              f"s {(std[:, t].double() - ws).abs().max().item():.2e}, means rel {rel:.2e}")
        assert rel < 1e-5, rel
        want = ep.derived(wq, K)
        for name in ("rmse", "spread", "ssr", "crps_fair", "crps_ecdf"):
            torch.testing.assert_close(getattr(sc, name)[:, t].double(), want[name], rtol=1e-5, atol=1e-6)
