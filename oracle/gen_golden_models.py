"""Generate model-level golden vectors FROM THE REFERENCE SOURCE (SURVEY.md 8 rows a10-a16).

TEST INFRASTRUCTURE ONLY.  Run in the build container (needs /root/reference):

    python -m oracle.gen_golden_models

``oracle/load_reference.load_models`` imports the reference's ``step_predictors/base.py``,
``graph/{base,graph_lam,hierarchical,hi_lam,hi_lam_parallel}.py``, ``forecasters/autoregressive.py`` and
``utils/{graph,buffer_list,tensor}.py`` UNMODIFIED (PyG behind ``oracle/pyg_standin.py``, the datastore behind
``load_reference.StubDatastore``).  For every case below a synthetic graph is written in the reference's on-disk
format (``neural_lam_b200.synthetic.save_graph``), the reference model reads it with ITS OWN ``load_graph``, is
initialised under ``torch.manual_seed``, and ``ARForecaster.forward`` is run on seeded CPU fp32 inputs.  Stored:
the state_dict, the inputs, the rollout (and the predicted std where the model has one) ->
``tests/golden/model_cases.*.npz``.  Both the CPU restatement (tests/test_oracle_models.py) and the CUDA path
(tests/test_models_golden.py, ``-m gpu``) are checked against this file.
"""
import os
import sys
import tempfile

import numpy as np
import torch

from . import load_reference
from .shards import save_shards

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "model_cases")

# name -> (reference class, graph kwargs, datastore kwargs, model kwargs, B, T)
CASES = {
    # BASELINE config 2's model family (multiscale GraphLAM, H=64: the fused tensor-core kernels) on a small grid
    "graph_lam_ms_h64": ("GraphLAM", dict(Nx=30, Ny=27, hierarchical=False),
                         dict(d_state=5, d_forcing=6, d_static=1, boundary_width=2),
                         dict(hidden_dim=64, processor_layers=2), 2, 3),
    # BASELINE config 3's family: HiLAM with THREE mesh levels (27/9/3 nodes a side), H=64
    "hi_lam_l3_h64": ("HiLAM", dict(Nx=81, Ny=81, hierarchical=True),
                      dict(d_state=5, d_forcing=6, d_static=1, boundary_width=3),
                      dict(hidden_dim=64, processor_layers=1), 1, 2),
    # HiLAMParallel (SplitMLPs path), two levels
    "hi_lam_parallel_h16": ("HiLAMParallel", dict(Nx=30, Ny=27, hierarchical=True),
                            dict(d_state=5, d_forcing=6, d_static=1, boundary_width=2),
                            dict(hidden_dim=16, processor_layers=2), 2, 2),
    # BASELINE config 1's shape (16x16, one mesh level, hidden 16) with everything optional switched on:
    # predicted std, output clamping of all three kinds, PropagationNet encoder/decoder, mean aggregation
    "graph_lam_opts_h16": ("GraphLAM", dict(Nx=16, Ny=16, hierarchical=False, n_levels=1),
                           dict(d_state=5, d_forcing=6, d_static=1, boundary_width=1),
                           dict(hidden_dim=16, processor_layers=2, mesh_aggr="mean", output_std=True,
                                g2m_gnn_type="PropagationNet", m2g_gnn_type="PropagationNet",
                                output_clamping_lower={"var1": -2.5, "var3": -3.0},
                                output_clamping_upper={"var1": 2.0, "var4": 3.5}), 2, 3),
}


def build_inputs(B, T, G, d_state, d_forcing, seed=123):
    g = torch.Generator().manual_seed(seed)
    init = torch.randn(B, 2, G, d_state, generator=g)
    forc = torch.randn(B, T, G, d_forcing, generator=g)
    bnd = torch.randn(B, T, G, d_state, generator=g)
    return init, forc, bnd


def run_case(ref, name, tmp):
    from neural_lam_b200 import synthetic

    cls, gkw, dkw, mkw, B, T = CASES[name]
    spec = synthetic.make_graph_spec(**gkw)
    ds = synthetic.SyntheticDatastore(spec, **dkw)
    root = os.path.join(tmp, name)
    synthetic.save_graph(spec, os.path.join(root, "graph", "g"))
    stub = load_reference.StubDatastore(ds, root)
    torch.manual_seed(42)
    model = getattr(ref, cls)(stub, graph_name="g", num_past_forcing_steps=0, num_future_forcing_steps=0, **mkw)
    with torch.no_grad():  # non-trivial LayerNorm affine parameters
        for n_, p_ in model.named_parameters():
            if p_.dim() == 1 and p_.shape[0] == mkw["hidden_dim"] and (n_.endswith(".3.weight") or n_.endswith(".3.bias")):
                p_.add_(0.1 * torch.randn_like(p_))
    fc = ref.ARForecaster(model, stub)
    fc.eval()
    init, forc, bnd = build_inputs(B, T, ds.num_grid_nodes, dkw["d_state"], dkw["d_forcing"])
    with torch.no_grad():
        pred, std = fc(init, forc, bnd)
    blob = {"init": init.numpy(), "forcing": forc.numpy(), "boundary": bnd.numpy(), "pred": pred.numpy()}
    if std is not None:
        blob["pred_std"] = std.numpy()
    for k, v in model.state_dict().items():
        blob["param/" + k] = v.numpy()
    blob["meta"] = np.array([cls, repr(gkw), repr(dkw), repr(mkw), str(B), str(T)]).astype(str)
    n_par = sum(p.numel() for p in model.parameters())
    print(f"  {name}: {cls} G={ds.num_grid_nodes} params={n_par} |pred| max={pred.abs().max():.3f}")
    return blob


def main():
    ref = load_reference.load_models()
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name in CASES:
            for k, v in run_case(ref, name, tmp).items():
                out[f"{name}/{k}"] = v
    out["__names__"] = np.array(list(CASES))
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    paths = save_shards(OUT, out)
    print(f"wrote {len(paths)} files {OUT}.*.npz")


if __name__ == "__main__":
    sys.exit(main())
