"""Time the grid side of the encoder of one forecast step at bench.py config 2 size (MEPS 268x238 grid, GraphLAM H = 64), two
ways on the same inputs, alternating:

  old:   grid embedder (tc_rowmlp_kernel), the g2m node projections P_s / P_r (tc_rowlinear_kernel, launched by the g2m call's
         edge stage), encoding grid MLP (tc_rowmlp_kernel)
  fused: tc_encode_kernel (``ops.encode``)

The old projections have no entry of their own: nlam_inet_fwd launches them inside the g2m call's edge stage.  So "old"
times the embedder, the g2m edge stage (NLAM_EDGE_ONLY: projections + tc_edge_bcast_kernel) and the grid MLP, minus the
same edge stage run on the fused kernel's projections (tc_edge_bcast_kernel alone), timed in the same rounds.  Each round
times ITERS calls of one variant with CUDA events; rounds alternate old / fused / edge stage.  Prints one JSON line: median, min and max ms per call of each, the launch names of each, the
speed-up of the medians, and the maximum absolute difference of grid_rep, P_s and P_r between the two.

    python scripts/bench_encode.py [--batch 32] [--rounds 7] [--iters 50]
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from neural_lam_b200 import _lib, models, ops, synthetic  # noqa: E402


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = torch.cuda.get_device_name()
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_encode.py needs a CUDA device"
    dev = torch.device("cuda")
    B = args.batch
    spec = synthetic.make_graph_spec(268, 238, hierarchical=False)
    ds = synthetic.SyntheticDatastore(spec, d_state=17, d_forcing=18, d_static=4, boundary_width=10)
    torch.manual_seed(0)
    m = models.GraphLAM(ds, spec, hidden_dim=64, processor_layers=4).to(dev).eval()
    net = m.g2m_gnn
    with torch.no_grad():
        st = m.static_embeddings()
    G = m.num_grid_nodes
    gen = torch.Generator(device=dev).manual_seed(1)
    sources = [torch.randn(B, G, 17, device=dev, generator=gen), torch.randn(B, G, 17, device=dev, generator=gen),
               torch.randn(B, G, 18, device=dev, generator=gen), m.expand_to_batch(m.grid_static_features, B)]
    mesh, g2m = m.expand_to_batch(st["mesh_emb"], B), m.expand_to_batch(st["g2m_emb"], B)
    g = net._graph(dev)
    L = _lib.lib()
    em, am = ops.mlp_struct(net.edge_mlp), ops.mlp_struct(net.aggr_mlp)
    flags = net._flags()
    ws_bytes = L.nlam_inet_workspace_bytes(g.handle, B, 64, flags | _lib.HINT_ONE_HIDDEN)
    ws = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
    aggr = torch.empty(B, g.n_rec, 64, device=dev)
    agg_bytes = (B * g.n_rec * 64 * 4 + 255) // 256 * 256
    proj_old = ws[agg_bytes:].view(torch.float32)
    state = {}

    @torch.no_grad()
    def old():
        grid_emb = m.grid_embedder.apply_rows(sources)
        _lib.check(L.nlam_inet_fwd(g.handle, ctypes.byref(em), ctypes.byref(am), grid_emb.data_ptr(), G * 64, mesh.data_ptr(), 0,
                                   g2m.data_ptr(), 0, None, None, aggr.data_ptr(), B, flags | _lib.EDGE_ONLY, ws.data_ptr(),
                                   ws_bytes, ops._stream_ptr(dev)))
        state["old"] = m.encoding_grid_mlp.apply_rows([grid_emb], res=grid_emb)

    @torch.no_grad()
    def fused():
        r = ops.encode(g, m.grid_embedder, sources, m.encoding_grid_mlp, net.edge_mlp, mesh, g2m, flags=flags)
        assert r is not None, "ops.encode does not cover this shape"
        state["fused"] = r

    @torch.no_grad()
    def edge_only_with_proj():
        # the same edge stage on the fused projections: its time is subtracted from old() so that both sides time the
        # three launches the kernel replaces
        ps = state["fused"][1][0]
        _lib.check(L.nlam_inet_fwd_chain(g.handle, ctypes.byref(em), ctypes.byref(am), None, ps.data_ptr(), G * 64,
                                         mesh.data_ptr(), 0, g2m.data_ptr(), 0, None, None, aggr.data_ptr(), ps.data_ptr(),
                                         None, B, flags | _lib.EDGE_ONLY, ws.data_ptr(), ws_bytes, ops._stream_ptr(dev)))

    with ops.profile_launches() as prof:
        old()
    rows_old = prof.rows
    with ops.profile_launches() as prof:
        fused()
    rows_new = prof.rows
    for _ in range(3):
        old()
        fused()
        edge_only_with_proj()
    torch.cuda.synchronize()
    times = {"old": [], "fused": [], "edge": []}
    for _ in range(args.rounds):
        for name, fn in (("old", old), ("fused", fused), ("edge", edge_only_with_proj)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                fn()
            e1.record()
            e1.synchronize()
            times[name].append(e0.elapsed_time(e1) / args.iters)
    old()
    fused()
    torch.cuda.synchronize()
    grid_rep, (proj,), _ = state["fused"]
    n_ps = B * G * 64
    diff = max((grid_rep - state["old"]).abs().max().item(),
               (proj[:n_ps] - proj_old[:n_ps]).abs().max().item(),
               (proj[n_ps:n_ps + g.n_rec * 64] - proj_old[n_ps:n_ps + g.n_rec * 64]).abs().max().item())
    res = {"gpu": gpu_info(), "batch": B, "grid_nodes": G, "rounds": args.rounds, "iters": args.iters,
           "launches_old": [r[0] for r in rows_old if r[0] != "tc_edge_bcast_kernel"],
           "launches_fused": [r[0] for r in rows_new],
           "profile_us_old": [[r[0], round(r[1], 1)] for r in rows_old], "profile_us_fused": [[r[0], round(r[1], 1)] for r in rows_new],
           "max_abs_diff": diff}
    # old: embedder + projections + edge stage + grid MLP, minus the edge stage timed on its own
    t_old = [a - e for a, e in zip(times["old"], times["edge"])]
    for name, t in (("old", t_old), ("fused", times["fused"]), ("g2m_edge_stage", times["edge"])):
        res[name] = {"median_ms": round(statistics.median(t), 4), "min_ms": round(min(t), 4), "max_ms": round(max(t), 4)}
    res["speedup"] = round(res["old"]["median_ms"] / res["fused"]["median_ms"], 3)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
