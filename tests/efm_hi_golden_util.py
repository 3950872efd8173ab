"""Loader for tests/golden/efm_hi_cases.*.npz (generated from the reference's own hierarchical Graph-EFM source by
oracle/gen_golden_efm_hi.py) + builders of the product model / oracle inputs for a case."""
import ast
import os

import torch

from golden_util import load_shards

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "efm_hi_cases")
GRAPH_KEYS = ("grid_static_features", "g2m_features", "m2g_features", "g2m_edge_index", "m2g_edge_index", "diff_std",
              "diff_mean")
LEVEL_KEYS = ("mesh_static_features", "m2m_features", "m2m_edge_index", "mesh_up_features", "mesh_up_edge_index",
              "mesh_down_features", "mesh_down_edge_index")


def oracle_graph(model):
    """The tensors of a ``models.GraphEFM`` that ``oracle/efm_hi_port`` read."""
    g = {k: getattr(model, k).detach() for k in GRAPH_KEYS}
    g.update({k: [t.detach() for t in getattr(model, k)] for k in LEVEL_KEYS})
    return g


def oracle_cfg(model, model_kw, ds=None):
    kw = model_kw
    cfg = dict(hidden_layers=kw.get("hidden_layers", 1), prior_intra_level_layers=kw.get("prior_intra_level_layers", 2),
               encoder_intra_level_layers=kw.get("encoder_intra_level_layers", 2),
               decoder_intra_level_layers=kw.get("decoder_intra_level_layers", 4), learn_prior=kw.get("learn_prior", True),
               prior_dist=kw.get("prior_dist", "isotropic"), output_std=kw.get("output_std", False),
               num_top_nodes=model.latent_spatial_dim, latent_dim=model.latent_dim)
    if kw.get("output_clamping_lower") or kw.get("output_clamping_upper"):
        cfg["clamp"] = dict(names=list(ds.state_var_names), lower=kw.get("output_clamping_lower") or {},
                            upper=kw.get("output_clamping_upper") or {}, state_mean=ds.state_mean, state_std=ds.state_std)
    return cfg


def to_device(g, cfg, dev):
    g = {k: ([t.to(dev) for t in v] if isinstance(v, list) else v.to(dev)) for k, v in g.items()}
    if "clamp" in cfg:
        cfg = dict(cfg, clamp=dict(cfg["clamp"], state_mean=cfg["clamp"]["state_mean"].to(dev),
                                   state_std=cfg["clamp"]["state_std"].to(dev)))
    return g, cfg


class EfmHiCase:
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
        """(spec, datastore, GraphEFM with the case's weights loaded strictly) on the CPU."""
        from neural_lam_b200 import models, synthetic

        spec = synthetic.make_graph_spec(**self.graph_kw)
        ds = synthetic.SyntheticDatastore(spec, **self.ds_kw)
        model = models.GraphEFM(ds, spec, math=math, **self.model_kw)
        res = model.load_state_dict(self.params, strict=True)
        assert not res.missing_keys and not res.unexpected_keys
        return spec, ds, model

    def oracle_inputs(self, model, ds):
        """(params, graph dict, cfg) for oracle/efm_hi_port."""
        return dict(self.params), oracle_graph(model), oracle_cfg(model, self.model_kw, ds)


def load_efm_hi_cases():
    blob = load_shards(GOLDEN)
    return [EfmHiCase(blob, str(n)) for n in blob["__names__"]]
