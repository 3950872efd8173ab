"""Run the reference source on the inputs of three checks and store what they compare against as
``tests/golden/reference_checks.*.npz``, so that the checks run without the reference:

  * ``oracle_random/s<seed>/<cls>_<aggr>/...``: InteractionNet / PropagationNet of the reference on fresh random graphs and
    weights (fp32 CPU): inputs, state_dict and outputs (tests/test_oracle.py);
  * ``load_graph/<hier>/<key>[/<level>]``: the reference's ``load_graph`` on the directory ``synthetic.save_graph`` writes
    for the 30 x 27 grid (tests/test_oracle_models.py);
  * ``create_graph/<hier>/<key>[/<level>]``: the reference's ``create_graph`` on the same grid (tests/test_oracle_models.py).

Build-container tool: needs the reference checkout (``NLAM_REFERENCE_ROOT``) and networkx."""
import os
import sys
import tempfile

import numpy as np
import torch

from . import load_create_graph as lcg
from . import load_reference
from .shards import save_shards

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "reference_checks")


def oracle_random(blob):
    ref = load_reference.load()
    for seed in (0, 1, 2):
        torch.manual_seed(seed)
        ns, nr, ne, H, B = 11 + seed, 7, 40, 8 * (seed + 1), 2
        ei = torch.stack([torch.randint(0, ns, (ne,)), torch.randint(0, nr, (ne,))])
        ei[1, -1] = nr - 1
        for cls in ("InteractionNet", "PropagationNet"):
            for aggr in ("sum", "mean"):
                net = getattr(ref, cls)(ei.clone(), H, aggr=aggr)
                send, rec, edge = torch.randn(B, ns, H), torch.randn(B, nr, H), torch.randn(B, ne, H)
                with torch.no_grad():
                    r_ref, e_ref = net(send, rec, edge)
                pre = f"oracle_random/s{seed}/{cls}_{aggr}/"
                for k, v in dict(ei=ei, send=send, rec=rec, edge=edge, rec_out=r_ref, edge_out=e_ref).items():
                    blob[pre + k] = v.numpy()
                for k, v in net.state_dict().items():
                    blob[pre + "param/" + k] = v.numpy()


def _put(blob, pre, v):
    if isinstance(v, (list, tuple)) or not isinstance(v, torch.Tensor):
        for i, x in enumerate(v):
            blob[f"{pre}/{i}"] = torch.as_tensor(x).detach().numpy()
    else:
        blob[pre] = v.detach().numpy()


def graphs(blob):
    from neural_lam_b200 import synthetic

    ref = load_reference.load_models()
    for hier in (False, True):
        spec = synthetic.make_graph_spec(30, 27, hierarchical=hier)
        with tempfile.TemporaryDirectory() as tmp:
            synthetic.save_graph(spec, tmp)
            span = float(max(spec["grid_xy"][:, 0].max() - spec["grid_xy"][:, 0].min(),
                             spec["grid_xy"][:, 1].max() - spec["grid_xy"][:, 1].min()))
            is_hier, g = ref.load_graph(tmp, mesh_node_features_scaling=span)
        assert is_hier == hier
        for k in ("g2m_features", "m2g_features", "g2m_edge_index", "m2g_edge_index", "m2m_features", "m2m_edge_index",
                  "mesh_static_features", "mesh_up_features", "mesh_down_edge_index"):
            if hier or k in ("g2m_features", "m2g_features", "g2m_edge_index", "m2g_edge_index", "m2m_features",
                             "m2m_edge_index", "mesh_static_features"):
                _put(blob, f"load_graph/{int(hier)}/{k}", g[k])
        cg = lcg.reference_create_graph(30, 27, hierarchical=hier)
        keys = ["g2m_edge_index", "g2m_features", "m2g_edge_index", "m2g_features", "m2m_edge_index", "m2m_features",
                "mesh_features"]
        if hier:
            keys += ["mesh_up_edge_index", "mesh_up_features", "mesh_down_edge_index", "mesh_down_features"]
        for k in keys:
            _put(blob, f"create_graph/{int(hier)}/{k}", cg[k])


def main():
    blob = {}
    oracle_random(blob)
    graphs(blob)
    paths = save_shards(OUT, blob)
    print(f"wrote {len(paths)} files {OUT}.*.npz")


if __name__ == "__main__":
    sys.exit(main())
