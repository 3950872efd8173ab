"""neural_lam_b200 — H100 (sm_90a) kernels for Neural-LAM's InteractionNet message-passing
hot path behind the reference's Python API (``neural_lam.gnn_layers`` /
``neural_lam.models`` GraphLAM / HiLAM).  See DESIGN.md and INTEGRATION.md."""
from . import _lib, ops  # noqa: F401
from .gnn_layers import (  # noqa: F401
    GNN_TYPES,
    InteractionNet,
    PropagationNet,
    SplitMLPs,
    get_default_math,
    get_gnn_class,
    set_default_math,
)
from .networks import make_gnn_seq, make_mlp  # noqa: F401

__version__ = "0.1.0"
