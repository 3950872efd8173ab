"""Forecast steps at the benchmark's batch sizes (`-m gpu`): bench.py config 2 (MEPS 268x238 grid, multiscale GraphLAM
H = 64, P = 4) at B = 32 and config 3 (the same grid, three-level HiLAM H = 128, P = 6) at B = 8, built as bench.py builds
them.

Every persistent kernel of the step loops over work items indexed by batch element, and the small-batch tests never reach
the later iterations of those loops.  A forecast step has no reduction across the batch (no batch norm, no atomics; the
summation order inside a row is fixed), which gives checks without a tolerance:
  * permuting the batch permutes the output bit for bit (a wrong batch index, a stale prefetch or bleed between items
    breaks it);
  * where the step launches the same kernels at B and at B = 1, every element run alone equals its row of the batched
    run bit for bit;
and anchors the whole batch to the fp64 oracle through two of its elements (0 and B - 1, the bound of
``test_real_size._check``).  Config 2 also checks the eager no-grad forward against the graph replay (1e-6, as in
test_models.py) and ``rollout_from_host`` over 6 steps, on dense pinned host tensors and on a layout that takes the
per-sample copies, against the graph replay bit for bit.

Wall time on an H100 80GB HBM3 (700 W) with 8 host cores: about 80 s, most of it in the CPU oracle of the two elements.
"""
from types import SimpleNamespace

import pytest
import torch

from neural_lam_b200 import models, ops, synthetic
from oracle import reference_port as rp
from test_models import _oracle_graph
from test_real_size import _check

pytestmark = pytest.mark.gpu
DEV = "cuda"
T = 2
D_STATE, D_FORCING = 17, 18

CONFIGS = {
    "config2": dict(hierarchical=False, n_levels=None, model="graph_lam", hidden=64, layers=4, B=32),
    "config3": dict(hierarchical=True, n_levels=3, model="hi_lam", hidden=128, layers=6, B=8),
}


def _inputs(B, steps, G, seed):
    gen = torch.Generator().manual_seed(seed)
    return (torch.randn(B, 2, G, D_STATE, generator=gen), torch.randn(B, steps, G, D_FORCING, generator=gen),
            torch.randn(B, steps, G, D_STATE, generator=gen))


@pytest.fixture(scope="module", params=sorted(CONFIGS))
def case(request):
    """The model, B seeded inputs (a distinct draw per element) and their T-step graph replay, shared by the tests of one
    config: building the graph is the expensive part."""
    c = CONFIGS[request.param]
    spec = synthetic.make_graph_spec(268, 238, hierarchical=c["hierarchical"], n_levels=c["n_levels"])
    ds = synthetic.SyntheticDatastore(spec, d_state=D_STATE, d_forcing=D_FORCING, d_static=4, boundary_width=10)
    torch.manual_seed(42)
    model = models.MODELS[c["model"]](ds, spec, hidden_dim=c["hidden"], processor_layers=c["layers"])
    fc = models.ARForecaster(model, ds)
    graph = _oracle_graph(model, fc)
    B = c["B"]
    host = _inputs(B, T, model.num_grid_nodes, 123)
    fc = fc.to(DEV).eval()
    dev = tuple(t.to(DEV) for t in host)
    with torch.no_grad():
        out = fc.rollout_graphed(*dev)
    label = f"{request.param} ({c['model']} H={c['hidden']} P={c['layers']}, B={B})"
    yield SimpleNamespace(name=request.param, label=label, cfg=c, B=B, model=model, fc=fc, graph=graph, host=host, dev=dev,
                          out=out)
    del fc, model, dev, out
    torch.cuda.empty_cache()


def _step_launches(case, sl):
    """launch names of one eager forecast step (the step rollout_graphed captures) on the batch elements ``sl``"""
    init, forc, bnd = case.dev
    m = case.fc.predictor
    with torch.no_grad():
        m.static_embeddings()  # weight-only, cached: not part of the step
        with ops.profile_launches() as prof:
            m.forward_with_boundary(init[sl, 1], init[sl, 0], forc[sl, 0], bnd[sl, 0], case.fc.boundary_mask)
    return prof.names()


def test_batch_permutation_is_exact(case):
    B = case.B
    perm = torch.arange(B).flip(0).roll(2)  # reversal, then a rotation: no element keeps its place
    assert not (perm == torch.arange(B)).any()
    perm = perm.to(DEV)
    init, forc, bnd = case.dev
    with torch.no_grad():
        got = case.fc.rollout_graphed(init[perm], forc[perm], bnd[perm])
    want = case.out[perm]
    bad = [b for b in range(B) if not torch.equal(got[b], want[b])]
    assert not bad, (f"{case.label}: permuted positions {bad} differ from the permuted output "
                     f"(max |diff| {(got - want).abs().max().item():.3e})")


def test_batch_size_independence(case):
    """Each element alone (B = 1, one capture replayed per element) against its row of the batched run.  The step at B = 1
    launches the same kernels as at B (no shape-dependent choice flips between the two), so the rows must be equal bit
    for bit."""
    B = case.B
    names_b, names_1 = _step_launches(case, slice(None)), _step_launches(case, slice(0, 1))
    print(f"\n{case.label}: {len(names_b)} launches per step at B={B}, {len(names_1)} at B=1")
    if case.name == "config2":
        assert "tc_decode_kernel" in names_b, names_b  # the fused decoder runs at the bench's batch
    assert names_b == names_1, (f"{case.label}: the step launches other kernels at B={B} than at B=1; name the "
                                f"B-dependent choice here and compare those elements under the TF32 bound:\n"
                                f"B={B}: {names_b}\nB=1: {names_1}")
    init, forc, bnd = case.dev
    with torch.no_grad():
        single = torch.cat([case.fc.rollout_graphed(init[b:b + 1], forc[b:b + 1], bnd[b:b + 1]) for b in range(B)])
    bad = [b for b in range(B) if not torch.equal(single[b], case.out[b])]
    assert not bad, (f"{case.label}: elements {bad} run alone differ from their rows of the batch "
                     f"(max |diff| {(single - case.out).abs().max().item():.3e})")


def test_batch_ends_against_fp64_oracle(case):
    """Elements 0 and B - 1 of the batched run against the fp64 oracle, bound max(3 x reference-TF32 error, 1e-2) per
    step.  With the two exact checks above this ties every element of the batch to the oracle."""
    c, sel = case.cfg, [0, case.B - 1]
    params = {f"predictor.{k}": v.detach().cpu() for k, v in case.model.state_dict().items()}
    cfg = dict(model=c["model"], hidden_layers=1, processor_layers=c["layers"], mesh_aggr="sum")
    init, forc, bnd = (t[sel] for t in case.host)
    with torch.no_grad():
        want64 = rp.ar_rollout({k: v.double() for k, v in params.items()}, case.graph, cfg, init.double(), forc.double(),
                               bnd.double())
        with rp.tf32_matmul():
            ref_tf32 = rp.ar_rollout(params, case.graph, cfg, init, forc, bnd)
    _check(f"{case.label}, elements {sel}, {T} AR steps", case.out[sel].cpu(), want64, ref_tf32)


@pytest.mark.parametrize("case", ["config2"], indirect=True)
def test_eager_forward_matches_graph_replay(case):
    """The no-grad ``ARForecaster.forward`` (the decoder branch of ``forward()``) at B = 32 against the graph replay."""
    init, forc, bnd = case.dev
    with torch.no_grad(), ops.profile_launches() as prof:
        eager, _ = case.fc(init, forc, bnd)
    assert prof.names().count("tc_decode_kernel") == T, prof.names()
    torch.testing.assert_close(eager, case.out, rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("case", ["config2"], indirect=True)
def test_rollout_from_host_at_bench_batch(case):
    """``rollout_from_host`` at B = 32 over 6 steps, so that the waits of its double buffering (``in_free``, ``out_free``,
    from step 2 on) run several times: on dense pinned host tensors (one strided copy per step and tensor) and with the
    forcing sliced out of a wider last dimension (per-sample copies).  Both equal the graph replay bit for bit."""
    B, steps = case.B, 6
    init, forc, bnd = (t.pin_memory() for t in _inputs(B, steps, case.model.num_grid_nodes, 7))
    with torch.no_grad():
        want = case.fc.rollout_graphed(init.to(DEV), forc.to(DEV), bnd.to(DEV)).cpu()
    dense = case.fc.rollout_from_host(init, forc, bnd)
    assert dense.shape == want.shape and dense.is_pinned()
    assert torch.equal(dense, want), (dense - want).abs().max().item()
    wide = torch.empty(*forc.shape[:3], D_FORCING + 3).pin_memory()
    wide[..., :D_FORCING] = forc
    forc_strided = wide[..., :D_FORCING]
    assert forc_strided.is_pinned() and forc_strided.stride(2) != D_FORCING
    strided = case.fc.rollout_from_host(init, forc_strided, bnd)
    assert torch.equal(strided, want), (strided - want).abs().max().item()
