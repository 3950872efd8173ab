"""Graph-EFM ensemble forecasts reduced on the device, at BASELINE config 2 size (MEPS 268x238 grid, multiscale mesh,
H = 64, prior 2 / decoder 4 m2m layers, latent_dim 64), one initial condition, K members, for each K of ``--members``:

  1. ms per step of ``ARForecaster.rollout_ensemble`` (member expansion, predictor step on K rows, ens_stats_kernel; mean,
     spread and scores stored) against ms per step of ``rollout_graphed`` on the inputs expanded to K rows (every member's
     trajectory stored), each a ``--steps``-step rollout timed with CUDA events, alternating for ``--rounds`` rounds;
  2. ``nlam_ensemble_stats`` alone on one step's (1, K, G, 17) members with a target: µs per call (CUDA events over
     ``--iters`` calls; ens_stats_kernel and the fixed-order ens_reduce_kernel), the per-kernel split from
     ``ops.profile_launches``, and ens_stats_kernel's algorithmic bytes ((K + 1)·G·d·4 read + 2·G·d·4 written) over its
     time against the data sheet's 3.35 TB/s;
  3. the card's name, power limit and SM clocks (nvidia-smi), read in the same run.

Prints one JSON line.

    python scripts/bench_ensemble.py [--members 8 32 64] [--steps 19] [--rounds 5] [--iters 50]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from neural_lam_b200 import ensemble, models, ops, synthetic  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name()


def timed(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


def spread(v):
    return {"median": round(statistics.median(v), 4), "min": round(min(v), 4), "max": round(max(v), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--members", type=int, nargs="+", default=[8, 32, 64])
    ap.add_argument("--steps", type=int, default=19, help="forecast steps per rollout (the reference's T = 19)")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ensemble.py needs a CUDA device"
    dev = torch.device("cuda")
    info_before = gpu_info()
    spec = synthetic.make_graph_spec(268, 238, hierarchical=False)
    ds = synthetic.SyntheticDatastore(spec, d_state=17, d_forcing=18, d_static=4, boundary_width=10)
    torch.manual_seed(0)
    m = models.GraphEFMMultiScale(ds, spec, hidden_dim=64, prior_m2m_layers=2, decoder_m2m_layers=4).to(dev).eval()
    fc = models.ARForecaster(m, ds).to(dev)
    G, d, T = m.num_grid_nodes, 17, args.steps
    gen = torch.Generator(device=dev).manual_seed(1)
    init = torch.randn(1, 2, G, d, device=dev, generator=gen)
    forc = torch.randn(1, T, G, 18, device=dev, generator=gen)
    bnd = torch.randn(1, T, G, d, device=dev, generator=gen)
    results = []
    for K in args.members:
        ex = [t.expand(K, *t.shape[1:]).contiguous() for t in (init, forc, bnd)]
        ens = lambda: fc.rollout_ensemble(init, forc, bnd, K, targets=bnd)  # noqa: E731
        graphed = lambda: fc.rollout_graphed(*ex)  # noqa: E731
        for _ in range(2):  # capture + warm up both
            ens()
            graphed()
        times = {"ensemble": [], "graphed": []}
        for _ in range(args.rounds):
            times["ensemble"].append(timed(ens, 1) / T)
            times["graphed"].append(timed(graphed, 1) / T)

        # the statistics kernel alone on one step's members
        members = torch.randn(1, K, G, d, device=dev, generator=gen)
        mean, std = torch.empty(1, G, d, device=dev), torch.empty(1, G, d, device=dev)
        scores = torch.empty(1, d, 4, device=dev)
        ws = torch.empty(ensemble.workspace_bytes(1, G, d), dtype=torch.uint8, device=dev)
        interior = fc.interior_mask.reshape(-1).contiguous()
        call = lambda: ensemble.launch(members, interior, mean, std, target=bnd[:, 0], scores=scores, workspace=ws)  # noqa: E731
        for _ in range(5):
            call()
        call_us = [timed(call, args.iters) * 1e3 for _ in range(args.rounds)]
        with ops.profile_launches() as prof:
            for _ in range(args.iters):
                call()
        per_kernel = {}
        for name, us, _ in prof.rows:
            per_kernel.setdefault(name, []).append(us)
        k_us = statistics.median(per_kernel["ens_stats_kernel"])
        nbytes = (K + 1) * G * d * 4 + 2 * G * d * 4
        med = {k: statistics.median(v) for k, v in times.items()}
        results.append({
            "K": K,
            "rollout_ensemble_ms_per_step": spread(times["ensemble"]),
            "rollout_graphed_ms_per_step": spread(times["graphed"]),
            "ensemble_vs_graphed": round(med["ensemble"] / med["graphed"], 4),
            "stats_call_us": spread(call_us),
            "kernels_us": {n: round(statistics.median(v), 2) for n, v in per_kernel.items()},
            "ens_stats_kernel_MB": round(nbytes / 1e6, 1),
            "ens_stats_kernel_GBps": round(nbytes / (k_us * 1e-6) / 1e9, 1),
            "ens_stats_kernel_share_of_3.35TBps": round(nbytes / (k_us * 1e-6) / HBM_BYTES_PER_S, 3),
            "stats_share_of_step": round(statistics.median(call_us) * 1e-3 / med["ensemble"], 4),
        })
        del ex, members
        torch.cuda.empty_cache()
    print(json.dumps({
        "workload": f"GraphEFMMultiScale MEPS 268x238, H=64, prior 2 / decoder 4 m2m, latent 64, 1 initial condition, "
                    f"T={T} steps, targets given",
        "gpu_before": info_before, "gpu_after": gpu_info(), "results": results,
    }))


if __name__ == "__main__":
    main()
