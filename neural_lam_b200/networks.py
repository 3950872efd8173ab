"""MLP and GNN-stack factories with the reference's interface
(reference neural_lam/utils/networks.py: ``make_mlp`` :8-40, ``make_gnn_seq`` :43-106).

The modules built here are ordinary ``torch.nn`` containers so that ``state_dict`` keys and
shapes equal the reference's (``edge_mlp.0.weight`` ...); they only HOLD parameters — on the
forward path the math runs in libnlam_b200.so (see ``ops.rowmlp`` / ``FusedMLP``).
"""
import torch
from torch import nn

from . import _lib, backward, ops


class FusedMLP(nn.Sequential):
    """``nn.Sequential(Linear, SiLU, ..., Linear[, LayerNorm])`` whose ``forward`` is one
    fused row-MLP kernel launch.  Under autograd the backward re-evaluates the ATen modules
    (``ops.RecomputeFn``)."""

    nlam_flags = 0

    def forward(self, x):  # noqa: D102
        return self.apply_rows([x])

    def apply_rows(self, sources, res=None):
        """``(res or 0) + mlp(cat(sources, -1))`` in ONE kernel: the concatenation of up to 4
        row-aligned inputs (e.g. prev_state | prev_prev_state | forcing | static features,
        reference graph/base.py:275-283) and the residual add (base.py:308-310) are fused into
        the row-MLP kernel instead of being materialised."""
        for t in sources:
            if not t.is_cuda:
                raise RuntimeError("neural_lam_b200: CUDA tensors only (no CPU fallback)")
        params = list(self.parameters())
        names = [n for n, _ in self.named_parameters()]
        n_src = len(sources)
        has_res = res is not None

        def kernel_fn(*args):
            srcs = list(args[:n_src])
            r = args[n_src] if has_res else None
            return ops.rowmlp(self, srcs, res=r, flags=self.nlam_flags)

        def torch_fn(*args):
            srcs = list(args[:n_src])
            r = args[n_src] if has_res else None
            p_ = args[n_src + (1 if has_res else 0):]
            B = max((t.shape[0] for t in srcs if t.dim() == 3), default=None)
            if B is not None:
                srcs = [t if t.dim() == 3 and t.shape[0] == B else (t if t.dim() == 3 else t.unsqueeze(0)).expand(B, -1, -1)
                        for t in srcs]
            y = _aten_forward(self, dict(zip(names, p_)), torch.cat(srcs, dim=-1) if n_src > 1 else srcs[0])
            return y if r is None else r + y

        bwd_fn = None
        if not (self.nlam_flags & _lib.MATH_FP32) and backward.mlp_supported(self, sources, res):
            def bwd_fn(saved, gouts, needs=None):
                srcs = list(saved[:n_src])
                r = saved[n_src] if has_res else None
                need_src = needs is None or any(needs[:n_src])
                g_src, g_res, pg = backward.mlp_backward(self, srcs, r, gouts[0].contiguous(), need_src=need_src)
                g_src = [g if (g is None or g.shape == t.shape) else g.reshape(t.shape) for g, t in zip(g_src, srcs)]
                if g_res is not None and g_res.shape != r.shape:
                    g_res = g_res.reshape(r.shape) if g_res.numel() == r.numel() else g_res.sum(0)
                return (*g_src, *([g_res] if has_res else []), *[pg[n] for n in names])

        tensors = [*sources, *([res] if has_res else []), *params]
        return ops.run_with_recompute(kernel_fn, torch_fn, tensors, bwd_fn=bwd_fn)


def _aten_forward(seq, params, x):
    """Differentiable ATen evaluation of a make_mlp Sequential with explicit parameter tensors."""
    h = x
    for name, mod in seq.named_children():
        if isinstance(mod, nn.Linear):
            h = torch.nn.functional.linear(h, params[f"{name}.weight"], params[f"{name}.bias"])
        elif isinstance(mod, nn.SiLU):
            h = torch.nn.functional.silu(h)
        elif isinstance(mod, nn.LayerNorm):
            h = torch.nn.functional.layer_norm(h, mod.normalized_shape, params[f"{name}.weight"], params[f"{name}.bias"], mod.eps)
        else:
            raise TypeError(f"unexpected module {type(mod)} in make_mlp network")
    return h


def make_mlp(blueprint, layer_norm=True):
    """Widths ``blueprint[0] -> ... -> blueprint[-1]``; SiLU after every Linear but the
    last; optional trailing LayerNorm (torch defaults)."""
    n_hidden = len(blueprint) - 2
    if n_hidden < 0:
        raise AssertionError("Invalid MLP blueprint")
    mods = []
    for k in range(n_hidden + 1):
        mods.append(nn.Linear(blueprint[k], blueprint[k + 1]))
        if k < n_hidden:
            mods.append(nn.SiLU())
    if layer_norm:
        mods.append(nn.LayerNorm(blueprint[-1]))
    return FusedMLP(*mods)


class GNNSequential(nn.Module):
    """Stand-in for ``pyg.nn.Sequential("mesh_rep, edge_rep", [(gnn, "mesh_rep, mesh_rep,
    edge_rep -> mesh_rep, edge_rep"), ...])`` (reference networks.py:93-106,
    graph_lam.py:117-126).  Children are named ``module_{i}`` like PyG's so checkpoints map."""

    def __init__(self, gnns):
        super().__init__()
        self._n = len(gnns)
        for i, g in enumerate(gnns):
            self.add_module(f"module_{i}", g)

    def __len__(self):
        return self._n

    def __getitem__(self, i):
        return getattr(self, f"module_{i}")

    def forward(self, mesh_rep, edge_rep, keep_edge_rep=True, keep_stacked=False):
        """``keep_edge_rep=False``: the caller discards the final edge representation (GraphLAM.process_step,
        reference graph_lam.py:185 ``mesh_rep, _ = self.processor(...)``): in no-grad mode the last layer then
        skips writing it, and the layers in between update their (private) edge tensor IN PLACE.
        ``keep_stacked=True``: the same stacked path in no-grad mode, but the final edge representation is returned: the
        last layer writes it in place into the stack's private tensor (out of place when it is also the first layer, whose
        input belongs to the caller).  Graph-EFM's hierarchical decoder hands it to its down sweep."""
        grad = torch.is_grad_enabled()
        fast = (keep_stacked or not keep_edge_rep) and not grad
        keep = keep_stacked or keep_edge_rep
        proj = None  # node projections of the next layer's edge MLP, computed by the previous layer's node kernel
        for i in range(self._n):
            mod = getattr(self, f"module_{i}")
            if fast and hasattr(mod, "forward_stacked"):
                nxt = getattr(self, f"module_{i + 1}") if i + 1 < self._n else None
                mesh_rep, edge_rep, proj = mod.forward_stacked(mesh_rep, edge_rep, first=(i == 0), last=(i == self._n - 1),
                                                               proj_in=proj, next_layer=nxt, keep_edges=keep)
            else:
                assert proj is None
                mesh_rep, edge_rep = mod(mesh_rep, mesh_rep, edge_rep)
        return mesh_rep, edge_rep


def make_gnn_seq(edge_index, num_gnn_layers, hidden_layers, hidden_dim, gnn_type="InteractionNet"):
    """Stack of ``num_gnn_layers`` GNN layers mapping (mesh_rep, edge_rep) -> (mesh_rep, edge_rep)."""
    from .gnn_layers import get_gnn_class

    if num_gnn_layers < 1:
        raise ValueError(
            f"make_gnn_seq requires num_gnn_layers >= 1 (got {num_gnn_layers}); skip the stage for a no-op."
        )
    cls = get_gnn_class(gnn_type)
    return GNNSequential([cls(edge_index, hidden_dim, hidden_layers=hidden_layers) for _ in range(num_gnn_layers)])
