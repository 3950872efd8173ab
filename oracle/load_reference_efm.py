"""Load the reference's Graph-EFM source UNMODIFIED: ``models/latent/*.py`` and ``step_predictors/graph/graph_efm.py``.

TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``), on top of ``load_reference.load_models``.  The latent files import
``from neural_lam import utils`` / ``from neural_lam.gnn_layers import ...`` absolutely, so while they load ``neural_lam``
is an alias of the synthetic parent package that ``load_reference`` builds (and ``neural_lam.utils`` /
``neural_lam.gnn_layers`` of its modules).  ``utils.make_gnn_seq`` imports ``neural_lam.gnn_layers`` when it is called, so the
aliases stay in place after loading.
"""
import sys

from . import load_reference
from .load_reference import _PKG, _load_file, _synthetic_package


def load_efm():
    """Namespace of ``load_reference.load_models`` plus ``GraphEFMMultiScale``, ``GraphEFM``, ``GraphLatentEncoder``,
    ``ConstantLatentEncoder`` and ``GraphLatentDecoder`` from the reference files."""
    ns = load_reference.load_models()
    if hasattr(ns, "GraphEFMMultiScale"):
        return ns
    aliases = {"neural_lam": _PKG, "neural_lam.utils": f"{_PKG}.utils", "neural_lam.gnn_layers": f"{_PKG}.gnn_layers"}
    if "neural_lam" in sys.modules and sys.modules["neural_lam"] is not sys.modules[_PKG]:
        raise RuntimeError("a real neural_lam package is imported; the reference Graph-EFM files need the synthetic one")
    for k, v in aliases.items():
        sys.modules[k] = sys.modules[v]
    lat = _synthetic_package("models.latent")
    ldir = "neural_lam/models/latent/"
    for name in ("base_encoder", "base_decoder", "constant_encoder", "graph_encoder", "graph_decoder",
                 "hi_graph_encoder", "hi_graph_decoder"):
        mod = _load_file(f"models.latent.{name}", ldir + name + ".py")
        # what the package's __init__.py re-exports: the classes of its files
        for k, v in vars(mod).items():
            if isinstance(v, type) and v.__module__ == mod.__name__:
                setattr(lat, k, v)
    efm = _load_file("models.step_predictors.graph.graph_efm", "neural_lam/models/step_predictors/graph/graph_efm.py")
    ns.GraphEFMMultiScale, ns.GraphEFM = efm.GraphEFMMultiScale, efm.GraphEFM
    ns.GraphLatentEncoder, ns.ConstantLatentEncoder = lat.GraphLatentEncoder, lat.ConstantLatentEncoder
    ns.GraphLatentDecoder = lat.GraphLatentDecoder
    return ns
