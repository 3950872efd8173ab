"""Loader for tests/golden/model_cases.*.npz (generated from the reference's own model source by
oracle/gen_golden_models.py) + builders of the product model / oracle inputs for a case."""
import ast
import os

import numpy as np
import torch

from golden_util import load_shards

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "model_cases")

KIND = {"GraphLAM": "graph_lam", "HiLAM": "hi_lam", "HiLAMParallel": "hi_lam_parallel"}


class ModelCase:
    def __init__(self, blob, name):
        self.name = name
        pre = name + "/"
        meta = [str(x) for x in blob[pre + "meta"]]
        self.cls = meta[0]
        self.graph_kw, self.ds_kw, self.model_kw = (ast.literal_eval(m) for m in meta[1:4])
        self.B, self.T = int(meta[4]), int(meta[5])
        self.params = {k[len(pre) + 6:]: torch.from_numpy(blob[k]) for k in blob.files if k.startswith(pre + "param/")}
        self.init, self.forcing, self.boundary, self.pred = (torch.from_numpy(blob[pre + k])
                                                             for k in ("init", "forcing", "boundary", "pred"))
        self.pred_std = torch.from_numpy(blob[pre + "pred_std"]) if pre + "pred_std" in blob.files else None

    def build(self, math="auto"):
        """(spec, datastore, product model with the case's weights loaded, ARForecaster) on the CPU."""
        from neural_lam_b200 import models, synthetic

        spec = synthetic.make_graph_spec(**self.graph_kw)
        ds = synthetic.SyntheticDatastore(spec, **self.ds_kw)
        model = models.MODELS[KIND[self.cls]](ds, spec, math=math, **self.model_kw)
        missing = model.load_state_dict(self.params, strict=True)
        assert not missing.missing_keys and not missing.unexpected_keys
        return spec, ds, model, models.ARForecaster(model, ds)

    def oracle_inputs(self, model, fc, ds):
        """(params, graph dict, cfg) for oracle/reference_port.ar_rollout."""
        from neural_lam_b200 import models

        g = {"boundary_mask": fc.boundary_mask.detach().cpu()}
        for k in ("grid_static_features", "g2m_features", "m2g_features", "g2m_edge_index", "m2g_edge_index", "diff_std",
                  "diff_mean", "m2m_features", "m2m_edge_index", "mesh_static_features", "mesh_up_features",
                  "mesh_up_edge_index", "mesh_down_features", "mesh_down_edge_index"):
            if hasattr(model, k):
                v = getattr(model, k)
                g[k] = [t.detach().cpu() for t in v] if isinstance(v, models.BufferList) else v.detach().cpu()
        kw = self.model_kw
        cfg = dict(model=KIND[self.cls], hidden_layers=kw.get("hidden_layers", 1), processor_layers=kw["processor_layers"],
                   mesh_aggr=kw.get("mesh_aggr", "sum"), output_std=kw.get("output_std", False), return_std=True)
        for t in ("g2m_gnn_type", "m2g_gnn_type", "mesh_up_gnn_type", "mesh_down_gnn_type"):
            if t in kw:
                cfg[t] = kw[t]
        if kw.get("output_clamping_lower") or kw.get("output_clamping_upper"):
            cfg["clamp"] = dict(names=list(ds.state_var_names), lower=kw.get("output_clamping_lower") or {},
                                upper=kw.get("output_clamping_upper") or {}, state_mean=ds.state_mean, state_std=ds.state_std)
        params = {f"predictor.{k}": v for k, v in self.params.items()}
        return params, g, cfg


def load_model_cases():
    blob = load_shards(GOLDEN)
    return [ModelCase(blob, str(n)) for n in blob["__names__"]]
