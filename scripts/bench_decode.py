"""Time the mesh -> grid decoder of one forecast step at bench.py config 2 size (MEPS 268x238 grid, GraphLAM H = 64), two ways
on the same inputs, alternating:

  old:   edge-only InteractionNet (tc_rowlinear_kernel for P_s / P_r, tc_ell_window_kernel) + tc_node_out_kernel
         (``aggregate_only`` + ``ops.node_update_step``)
  fused: tc_rowlinear_kernel for P_s / P_e + tc_decode_kernel (``decode_step``)

Each round times ITERS calls of one variant with CUDA events; rounds alternate old / fused.  Prints one JSON line: median,
min and max ms per call of each, the speed-up of the medians, and the maximum absolute difference of the two outputs.

    python scripts/bench_decode.py [--batch 32] [--rounds 7] [--iters 50]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from neural_lam_b200 import models, ops, synthetic  # noqa: E402


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
    assert torch.cuda.is_available(), "bench_decode.py needs a CUDA device"
    dev = torch.device("cuda")
    B = args.batch
    spec = synthetic.make_graph_spec(268, 238, hierarchical=False)
    ds = synthetic.SyntheticDatastore(spec, d_state=17, d_forcing=18, d_static=4, boundary_width=10)
    torch.manual_seed(0)
    m = models.GraphLAM(ds, spec, hidden_dim=64, processor_layers=4)
    fc = models.ARForecaster(m, ds).to(dev).eval()
    net, out_map = m.m2g_gnn, m.output_map
    with torch.no_grad():
        st = m.static_embeddings()
    G, D = m.num_grid_nodes, ds.num_state_vars
    gen = torch.Generator(device=dev).manual_seed(1)
    mesh = torch.randn(B, st["mesh_emb"].shape[0], 64, device=dev, generator=gen)
    grid = torch.randn(B, G, 64, device=dev, generator=gen)
    m2g = m.expand_to_batch(st["m2g_emb"], B)
    prev = torch.randn(B, G, D, device=dev, generator=gen)
    bnd = torch.randn(B, G, D, device=dev, generator=gen)
    mask = fc.boundary_mask
    out_old, out_new = torch.empty_like(prev), torch.empty_like(prev)

    @torch.no_grad()
    def old():
        aggr = net.aggregate_only(mesh, grid, m2g)
        r = ops.node_update_step(net.aggr_mlp, out_map, grid, aggr, prev, bnd, mask, m.diff_std, m.diff_mean, out=out_old)
        assert r is not None

    @torch.no_grad()
    def fused():
        r = net.decode_step(mesh, grid, m2g, out_map, prev, bnd, mask, m.diff_std, m.diff_mean, out=out_new)
        assert r is not None, "decode_step does not cover this shape"

    with ops.profile_launches() as prof:
        old()
    names_old = prof.names()
    with ops.profile_launches() as prof:
        fused()
    names_new = prof.names()
    for _ in range(3):
        old()
        fused()
    torch.cuda.synchronize()
    times = {"old": [], "fused": []}
    for _ in range(args.rounds):
        for name, fn in (("old", old), ("fused", fused)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                fn()
            e1.record()
            e1.synchronize()
            times[name].append(e0.elapsed_time(e1) / args.iters)
    diff = (out_new - out_old).abs().max().item()
    res = {"gpu": gpu_info(), "batch": B, "grid_nodes": G, "rounds": args.rounds, "iters": args.iters,
           "launches_old": names_old, "launches_fused": names_new,
           "max_abs_diff": diff}
    for name, t in times.items():
        res[name] = {"median_ms": round(statistics.median(t), 4), "min_ms": round(min(t), 4), "max_ms": round(max(t), 4)}
    res["speedup"] = round(res["old"]["median_ms"] / res["fused"]["median_ms"], 3)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
