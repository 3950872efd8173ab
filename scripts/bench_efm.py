"""Graph-EFM ensemble forecasting at BASELINE config 2 size (MEPS 268x238 grid, multiscale mesh, H = 64, prior 2 / decoder 4
m2m layers, latent_dim 64), B ensemble members, in one run:

  1. forecast steps/s from the captured step graphs (``ARForecaster.capture``: fresh noise per replay), CUDA events around
     ``--steps`` replays after ``--warmup``; one step advances all B members;
  2. the kernel table of one no-grad step (``ops.profile_launches``: name, µs, algorithmic bytes);
  3. the latent step two ways on the same inputs, alternating rounds of ``--iters`` calls: tc_latent_kernel
     (``ops.latent_sample``) against the composition it replaces (latent_param_map, mean + eps * std, latent_embedder),
     with the maximum absolute difference of their outputs;
  4. the card's name, power limit and max SM clock (nvidia-smi), read in the same run.

Prints one JSON line.

    python scripts/bench_efm.py [--batch 32] [--steps 50] [--warmup 10] [--rounds 7] [--iters 50]
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
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32, help="ensemble members (independent forecasts) per step")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_efm.py needs a CUDA device"
    dev = torch.device("cuda")
    B = args.batch
    spec = synthetic.make_graph_spec(268, 238, hierarchical=False)
    ds = synthetic.SyntheticDatastore(spec, d_state=17, d_forcing=18, d_static=4, boundary_width=10)
    torch.manual_seed(0)
    m = models.GraphEFMMultiScale(ds, spec, hidden_dim=64, prior_m2m_layers=2, decoder_m2m_layers=4).to(dev).eval()
    fc = models.ARForecaster(m, ds).to(dev)
    G, N = m.num_grid_nodes, m.num_mesh_nodes
    gen = torch.Generator(device=dev).manual_seed(1)
    prev, prev_prev = torch.randn(B, G, 17, device=dev, generator=gen), torch.randn(B, G, 17, device=dev, generator=gen)
    forcing, bnd = torch.randn(B, G, 18, device=dev, generator=gen), torch.randn(B, G, 17, device=dev, generator=gen)

    # 1. captured forecast steps
    bufs = fc.capture(B)
    fc.set_state(prev_prev, prev)
    bufs["forcing"].copy_(forcing)
    bufs["boundary"].copy_(bnd)
    for _ in range(args.warmup):
        fc.replay_step()
    ms_step = timed(fc.replay_step, args.steps)

    # 2. kernel table of one step
    eps = torch.randn(B, N, m.latent_dim, device=dev, generator=gen)
    with torch.no_grad(), ops.profile_launches() as prof:
        m.forward_with_boundary(prev, prev_prev, forcing, bnd, fc.boundary_mask, latent_noise=eps)
    table = [{"kernel": n, "us": round(us, 1), "MB": round(b / 1e6, 1)} for n, us, b in prof.rows]

    # 3. latent kernel vs the composition it replaces
    pm, em = m.prior_model.latent_param_map, m.decoder.latent_embedder
    x = torch.randn(B, N, 64, device=dev, generator=gen)
    out = {}

    @torch.no_grad()
    def fused():
        out["fused"] = ops.latent_sample(pm, em, x, eps)

    @torch.no_grad()
    def composed():
        mean, std = m.prior_model.mean_std(pm(x))
        out["composed"] = em.apply_rows([mean + eps * std])

    with ops.profile_launches() as prof:
        fused()
    names_fused = prof.names()
    with ops.profile_launches() as prof:
        composed()
    names_composed = prof.names()
    for _ in range(3):
        fused()
        composed()
    times = {"fused": [], "composed": []}
    for _ in range(args.rounds):
        for name, fn in (("fused", fused), ("composed", composed)):
            times[name].append(timed(fn, args.iters))
    fused()
    composed()
    torch.cuda.synchronize()
    diff = (out["fused"] - out["composed"]).abs().max().item()
    med = {k: statistics.median(v) for k, v in times.items()}
    print(json.dumps({
        "workload": f"GraphEFMMultiScale MEPS 268x238, H=64, prior 2 / decoder 4 m2m, latent 64, B={B}",
        "gpu": gpu_info(),
        "forecast_steps_per_s": round(1e3 / ms_step, 2), "ms_per_step": round(ms_step, 3),
        "member_steps_per_s": round(B * 1e3 / ms_step, 1),
        "launches_per_step": len(table), "kernels": table,
        "latent": {"fused_ms": {"median": round(med["fused"], 4), "min": round(min(times["fused"]), 4),
                                "max": round(max(times["fused"]), 4)},
                   "composed_ms": {"median": round(med["composed"], 4), "min": round(min(times["composed"]), 4),
                                   "max": round(max(times["composed"]), 4)},
                   "speedup": round(med["composed"] / med["fused"], 2), "fused_launches": names_fused,
                   "composed_launches": names_composed, "max_abs_diff": diff},
    }))


if __name__ == "__main__":
    main()
