"""Loader for tests/golden/efm_cases.*.npz (generated from the reference's own Graph-EFM source by
oracle/gen_golden_efm.py) + builders of the product model / oracle inputs for a case."""
import ast
import os

import torch

from golden_util import load_shards

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "efm_cases")
GRAPH_KEYS = ("grid_static_features", "g2m_features", "m2g_features", "g2m_edge_index", "m2g_edge_index", "diff_std",
              "diff_mean", "m2m_features", "m2m_edge_index", "mesh_static_features")


class EfmCase:
    def __init__(self, blob, name):
        self.name = name
        pre = name + "/"
        meta = [str(x) for x in blob[pre + "meta"]]
        self.graph_kw, self.ds_kw, self.model_kw = (ast.literal_eval(m) for m in meta[:3])
        self.B = int(meta[3])
        t = lambda k: torch.from_numpy(blob[pre + k]) if pre + k in blob else None  # noqa: E731
        self.params = {k[len(pre) + 6:]: torch.from_numpy(blob[k]) for k in blob.files if k.startswith(pre + "param/")}
        self.grads = {k[len(pre) + 5:]: torch.from_numpy(blob[k]) for k in blob.files if k.startswith(pre + "grad/")}
        for k in ("prev_state", "prev_prev_state", "forcing", "target", "eps", "prior_mean", "prior_std", "pred", "pred_std",
                  "post_mean", "post_std", "w_pred", "w_post"):
            setattr(self, k, t(k))

    def build(self, math="auto"):
        """(spec, datastore, GraphEFMMultiScale with the case's weights loaded strictly) on the CPU."""
        from neural_lam_b200 import models, synthetic

        spec = synthetic.make_graph_spec(**self.graph_kw)
        ds = synthetic.SyntheticDatastore(spec, **self.ds_kw)
        model = models.GraphEFMMultiScale(ds, spec, math=math, **self.model_kw)
        res = model.load_state_dict(self.params, strict=True)
        assert not res.missing_keys and not res.unexpected_keys
        return spec, ds, model

    def oracle_inputs(self, model, ds):
        """(params, graph dict, cfg) for oracle/efm_port."""
        g = {k: getattr(model, k).detach().cpu() for k in GRAPH_KEYS}
        kw = self.model_kw
        cfg = dict(hidden_layers=kw.get("hidden_layers", 1), prior_m2m_layers=kw.get("prior_m2m_layers", 2),
                   encoder_m2m_layers=kw.get("encoder_m2m_layers", 2), decoder_m2m_layers=kw.get("decoder_m2m_layers", 4),
                   learn_prior=kw.get("learn_prior", True), prior_dist=kw.get("prior_dist", "isotropic"),
                   output_std=kw.get("output_std", False), num_mesh_nodes=model.num_mesh_nodes, latent_dim=model.latent_dim)
        if kw.get("output_clamping_lower") or kw.get("output_clamping_upper"):
            cfg["clamp"] = dict(names=list(ds.state_var_names), lower=kw.get("output_clamping_lower") or {},
                                upper=kw.get("output_clamping_upper") or {}, state_mean=ds.state_mean, state_std=ds.state_std)
        return dict(self.params), g, cfg


def load_efm_cases():
    blob = load_shards(GOLDEN)
    return [EfmCase(blob, str(n)) for n in blob["__names__"]]
