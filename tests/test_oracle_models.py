"""Model-level oracle pinning (SURVEY.md 8 rows a10-a16): the CPU restatement
``oracle/reference_port.graph_model_forward`` / ``ar_rollout`` against golden vectors produced by the reference's
OWN ``graph/base.py`` + ``graph_lam.py`` + ``hierarchical.py`` + ``hi_lam.py`` + ``hi_lam_parallel.py`` +
``forecasters/autoregressive.py`` (``oracle/gen_golden_models.py``), and the graph loader / generator against the
reference's results stored by ``oracle/gen_golden_refchecks.py``."""
import os
import tempfile

import pytest
import torch

from golden_util import load_shards
from model_golden_util import load_model_cases
from oracle import reference_port as rp

CASES = load_model_cases()


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_oracle_port_matches_reference_golden(case):
    _, ds, model, fc = case.build()
    params, g, cfg = case.oracle_inputs(model, fc, ds)
    with torch.no_grad():
        pred, std = rp.ar_rollout(params, g, cfg, case.init, case.forcing, case.boundary)
    # fp32 on both sides, same op sequence up to summation order of index_add_/scatter_add_ and cat-vs-split GEMMs
    torch.testing.assert_close(pred, case.pred, rtol=2e-5, atol=2e-5)
    if case.pred_std is None:
        assert std is None
    else:
        torch.testing.assert_close(std, case.pred_std, rtol=2e-5, atol=2e-5)
    # boundary rows carry the true state (autoregressive.py:128-131)
    bm = g["boundary_mask"].bool().reshape(-1)
    torch.testing.assert_close(pred[:, :, bm], case.boundary[:, :, bm], rtol=0, atol=0)


def test_state_dict_names_match_reference():
    """The golden state_dicts come from the reference classes; strict loading into the product models is the
    checkpoint-compatibility check (parameter names AND shapes)."""
    for case in CASES:
        _, _, model, _ = case.build()
        assert set(model.state_dict()) == set(case.params), case.name


REFCHECKS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_checks")


def _stored(blob, pre):
    """one tensor, or the per-level list stored as <pre>/0, <pre>/1, ..."""
    if pre in blob:
        return torch.from_numpy(blob[pre])
    out = []
    while f"{pre}/{len(out)}" in blob:
        out.append(torch.from_numpy(blob[f"{pre}/{len(out)}"]))
    return out


def test_reference_load_graph_reads_generated_files():
    """``synthetic.load_graph`` + ``normalize_graph`` on the directories ``synthetic.save_graph`` writes arrive at the
    tensors the reference's own ``load_graph`` read from the same directories (stored in
    tests/golden/reference_checks.*.npz by oracle/gen_golden_refchecks.py)."""
    from neural_lam_b200 import synthetic

    blob = load_shards(REFCHECKS)
    for hier in (False, True):
        spec = synthetic.make_graph_spec(30, 27, hierarchical=hier)
        with tempfile.TemporaryDirectory() as tmp:
            synthetic.save_graph(spec, tmp)
            ours = synthetic.normalize_graph(synthetic.load_graph(tmp, spec["grid_xy"]))
        g = lambda k: _stored(blob, f"load_graph/{int(hier)}/{k}")  # noqa: E731
        for k in ("g2m_features", "m2g_features", "g2m_edge_index", "m2g_edge_index"):
            torch.testing.assert_close(ours[k], g(k), rtol=0, atol=0)
        for k in ("m2m_features", "m2m_edge_index", "mesh_static_features", "mesh_up_features", "mesh_down_edge_index"):
            if hier:
                a, b = ours[k], g(k)
                assert len(a) == len(b) > 0
                for x, y in zip(a, b):
                    torch.testing.assert_close(x, y, rtol=0, atol=0)
            elif k in ("m2m_features", "m2m_edge_index", "mesh_static_features"):
                torch.testing.assert_close(ours[k], g(k), rtol=0, atol=0)


def test_legacy_graph_directory_is_zero_indexed(tmp_path):
    """A directory without metainfo.yaml is the legacy format: offset node labels, normalised mesh coordinates
    (reference utils/graph.py:272-328)."""
    from neural_lam_b200 import synthetic

    spec = synthetic.make_graph_spec(30, 27, hierarchical=False)
    norm = synthetic.normalize_graph(spec)
    legacy = dict(spec)
    n_mesh = spec["mesh_static_features"].shape[0]
    legacy["mesh_static_features"] = norm["mesh_static_features"]
    legacy["g2m_edge_index"] = torch.stack((spec["g2m_edge_index"][0] + n_mesh, spec["g2m_edge_index"][1]))
    legacy["m2g_edge_index"] = torch.stack((spec["m2g_edge_index"][0], spec["m2g_edge_index"][1] + n_mesh))
    synthetic.save_graph(legacy, str(tmp_path))
    os.remove(tmp_path / "metainfo.yaml")
    got = synthetic.normalize_graph(synthetic.load_graph(str(tmp_path), spec["grid_xy"]))
    for k in ("g2m_edge_index", "m2g_edge_index", "mesh_static_features", "g2m_features"):
        torch.testing.assert_close(got[k], norm[k], rtol=0, atol=0)
    (tmp_path / "metainfo.yaml").write_text("spec_version: 9.9\n")
    with pytest.raises(ValueError):
        synthetic.load_graph(str(tmp_path), spec["grid_xy"])


def _edge_set(ei, feat):
    return sorted((int(a), int(b)) + tuple(round(float(x), 4) for x in f) for a, b, f in zip(ei[0], ei[1], feat))


@pytest.mark.parametrize("hier", [False, True])
def test_graph_generator_matches_reference_create_graph(hier):
    """``synthetic.make_graph_spec`` (vectorised) against the reference's own ``create_graph`` (networkx loops,
    create_graph.py:356-862, run unmodified through oracle/load_create_graph.py; its graphs are stored in
    tests/golden/reference_checks.*.npz) on a NON-square grid: identical edge sets and edge features for g2m (radius
    0.67 x the mesh spacing along the first axis), m2g (4 nearest), every m2m level, the up / down edges, and identical
    mesh node positions."""
    from neural_lam_b200 import synthetic

    blob = load_shards(REFCHECKS)
    ref = {k: _stored(blob, f"create_graph/{int(hier)}/{k}") for k in (
        "g2m_edge_index", "g2m_features", "m2g_edge_index", "m2g_features", "m2m_edge_index", "m2m_features", "mesh_features",
        "mesh_up_edge_index", "mesh_up_features", "mesh_down_edge_index", "mesh_down_features")}
    mine = synthetic.make_graph_spec(30, 27, hierarchical=hier)
    for k in ("g2m", "m2g"):
        assert _edge_set(ref[f"{k}_edge_index"], ref[f"{k}_features"]) == _edge_set(mine[f"{k}_edge_index"], mine[f"{k}_features"]), k
    m_ei = mine["m2m_edge_index"] if hier else [mine["m2m_edge_index"]]
    m_f = mine["m2m_features"] if hier else [mine["m2m_features"]]
    mesh = mine["mesh_static_features"] if hier else [mine["mesh_static_features"]]
    assert len(ref["m2m_edge_index"]) == len(m_ei)
    for l in range(len(m_ei)):
        assert _edge_set(ref["m2m_edge_index"][l], ref["m2m_features"][l]) == _edge_set(m_ei[l], m_f[l]), f"m2m level {l}"
        torch.testing.assert_close(ref["mesh_features"][l].float(), mesh[l], rtol=1e-6, atol=1e-5)
    if hier:
        for k in ("mesh_up", "mesh_down"):
            for l in range(len(mine[f"{k}_edge_index"])):
                assert _edge_set(ref[f"{k}_edge_index"][l], ref[f"{k}_features"][l]) == \
                    _edge_set(mine[f"{k}_edge_index"][l], mine[f"{k}_features"][l]), f"{k} level {l}"
