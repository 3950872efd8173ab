"""Generate golden vectors for the InteractionNet hot path FROM THE REFERENCE SOURCE.

TEST INFRASTRUCTURE ONLY.  Run in the build container (needs /root/reference):

    python -m oracle.gen_golden

It imports the reference's ``neural_lam/gnn_layers.py`` / ``utils/networks.py``
unmodified (``oracle/load_reference.py``), builds ``InteractionNet`` /
``PropagationNet`` instances exactly as the reference constructs them, runs
forward + backward on seeded CPU fp32 inputs and stores inputs, weights, outputs
and gradients as ``tests/golden/inet_cases.*.npz``.  The GPU box has no
``/root/reference``; its tests compare against this file.
"""
import os
import sys

import numpy as np
import torch

from . import load_reference
from .shards import save_shards

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "inet_cases")


def _rand_edge_index(n_send, n_rec, n_edges, seed=0):
    # reference tests/test_gnn_layers.py:15-20
    torch.manual_seed(seed)
    senders = torch.randint(0, n_send, (n_edges,))
    receivers = torch.randint(0, n_rec, (n_edges,))
    # make sure the highest receiver id is present so that num_rec == n_rec
    receivers[-1] = n_rec - 1
    return torch.stack([senders, receivers])


CASES = [
    # name, cls, n_send, n_rec, E, H, B (0 = unbatched), kwargs, same_nodes
    ("inet_sum_h8", "InteractionNet", 5, 4, 10, 8, 0, dict(update_edges=True), False),
    ("inet_mean_b3_h16", "InteractionNet", 7, 6, 24, 16, 3, dict(update_edges=True, aggr="mean"), False),
    ("inet_noedge_h4", "InteractionNet", 100, 10, 200, 4, 2, dict(update_edges=False), False),
    ("pnet_h8", "PropagationNet", 5, 4, 10, 8, 0, dict(update_edges=True), False),
    ("pnet_noedge_b2_h16", "PropagationNet", 9, 5, 31, 16, 2, dict(update_edges=False), False),
    ("inet_m2m_h64", "InteractionNet", 40, 40, 200, 64, 2, dict(update_edges=True), True),
    ("inet_g2m_h64_highdeg", "InteractionNet", 300, 3, 500, 64, 1, dict(update_edges=False), False),
    ("inet_chunks_h8", "InteractionNet", 6, 4, 12, 8, 0, dict(update_edges=True, edge_chunk_sizes=[5, 7], aggr_chunk_sizes=[2, 2]), False),
    ("pnet_chunks_h8", "PropagationNet", 6, 4, 12, 8, 2, dict(update_edges=True, edge_chunk_sizes=[5, 7], aggr_chunk_sizes=[1, 3]), False),
    ("inet_hl2_h8", "InteractionNet", 5, 4, 10, 8, 0, dict(update_edges=True, hidden_layers=2), False),
]


def main():
    ref = load_reference.load()
    blob = {}
    names = []
    for name, cls, ns, nr, ne, H, B, kw, same in CASES:
        ei = _rand_edge_index(ns, nr, ne)
        torch.manual_seed(42)
        net = getattr(ref, cls)(ei.clone(), H, **kw)
        # non-trivial LayerNorm affine so gamma/beta are exercised
        with torch.no_grad():
            for n_, p_ in net.named_parameters():
                if p_.dim() == 1 and (".3." in n_ or n_.endswith(("5.weight", "5.bias"))):
                    p_.add_(0.1 * torch.randn_like(p_))
        gen = torch.Generator().manual_seed(123)
        shp = (lambda n: (B, n, H)) if B else (lambda n: (n, H))
        send = torch.randn(*shp(ns), generator=gen)
        rec = send.clone() if same else torch.randn(*shp(nr), generator=gen)
        edge = torch.randn(*shp(ne), generator=gen)
        w_rec = torch.randn(*shp(nr), generator=gen)
        w_edge = torch.randn(*shp(ne), generator=gen)
        send.requires_grad_(True)
        edge.requires_grad_(True)
        if same:
            out = net(send, send, edge)
        else:
            rec.requires_grad_(True)
            out = net(send, rec, edge)
        if kw.get("update_edges", True):
            rec_out, edge_out = out
            loss = (rec_out * w_rec).sum() + (edge_out * w_edge).sum()
        else:
            rec_out, edge_out = out, None
            loss = (rec_out * w_rec).sum()
        loss.backward()
        names.append(name)
        pre = name + "/"
        blob[pre + "edge_index"] = ei.numpy()
        blob[pre + "send"] = send.detach().numpy()
        blob[pre + "rec"] = (send if same else rec).detach().numpy()
        blob[pre + "edge"] = edge.detach().numpy()
        blob[pre + "w_rec"] = w_rec.numpy()
        blob[pre + "w_edge"] = w_edge.numpy()
        blob[pre + "rec_out"] = rec_out.detach().numpy()
        if edge_out is not None:
            blob[pre + "edge_out"] = edge_out.detach().numpy()
        blob[pre + "g_send"] = send.grad.numpy()
        if not same:
            blob[pre + "g_rec"] = rec.grad.numpy()
        blob[pre + "g_edge"] = edge.grad.numpy()
        for k, v in net.state_dict().items():
            blob[pre + "param/" + k] = v.numpy()
        for k, v in net.named_parameters():
            blob[pre + "gparam/" + k] = v.grad.numpy()
        # meta
        blob[pre + "meta"] = np.array(
            [cls, str(B), str(int(same)), repr(kw)], dtype=object
        ).astype(str)
    blob["__names__"] = np.array(names)
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    paths = save_shards(OUT, blob)
    print(f"wrote {len(paths)} files {OUT}.*.npz")


if __name__ == "__main__":
    sys.exit(main())
