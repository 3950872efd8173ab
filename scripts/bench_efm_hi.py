"""Graph-EFM on the hierarchical MEPS mesh (268x238 grid, levels of 6 561 / 729 / 81 / 9 nodes, H = latent = 64, intra-level
layers prior 2 / encoder 2 / decoder 4), B ensemble members, in one run:

  1. forecast steps/s from the captured step graphs (``ARForecaster.capture``: fresh noise per replay), CUDA events around
     ``--steps`` replays after ``--warmup``; one step advances all B members;
  2. the kernel table of one no-grad step (``ops.profile_launches``: name, µs, algorithmic bytes);
  3. the grid side of the step two ways on the same inputs, alternating rounds of ``--iters`` calls: one tc_encode2_kernel
     launch for the projections of both g2m layers, then both g2m layers on them (``encode_step(second=...)``), against
     tc_encode_kernel storing grid_emb (EMIT_EMB) and the decoder's g2m call computing its own projections from it
     (tc_rowlinear_kernel); the maximum absolute difference of the three outputs (prior and decoder level-0
     representations, grid_rep);
  4. the card's name, power limit and max SM clock (nvidia-smi), read in the same run.

Prints one JSON line.

    python scripts/bench_efm_hi.py [--batch 32] [--steps 30] [--warmup 5] [--rounds 7] [--iters 20]
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


def stats(v):
    return {"median": round(statistics.median(v), 4), "min": round(min(v), 4), "max": round(max(v), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32, help="ensemble members (independent forecasts) per step")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_efm_hi.py needs a CUDA device"
    dev = torch.device("cuda")
    B = args.batch
    spec = synthetic.make_graph_spec(268, 238, hierarchical=True)
    ds = synthetic.SyntheticDatastore(spec, d_state=17, d_forcing=18, d_static=4, boundary_width=10)
    torch.manual_seed(0)
    m = models.GraphEFM(ds, spec, hidden_dim=64, prior_intra_level_layers=2, encoder_intra_level_layers=2,
                        decoder_intra_level_layers=4).to(dev).eval()
    fc = models.ARForecaster(m, ds).to(dev)
    G = m.num_grid_nodes
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
    del bufs
    fc._graph = None
    torch.cuda.empty_cache()

    # 2. kernel table of one step
    eps = torch.randn(B, m.latent_spatial_dim, m.latent_dim, device=dev, generator=gen)
    with torch.no_grad(), ops.profile_launches() as prof:
        m.forward_with_boundary(prev, prev_prev, forcing, bnd, fc.boundary_mask, latent_noise=eps)
    table = [{"kernel": n, "us": round(us, 1), "MB": round(b / 1e6, 1)} for n, us, b in prof.rows]

    # 3. the grid side: one launch for both g2m layers' projections, against EMIT_EMB + the decoder g2m's own projections
    prior_g2m, dec = m.prior_model.g2m_gnn, m.decoder
    sources = m._grid_sources(prev, prev_prev, forcing)
    ge = m._graph_emb(B)
    mesh0, g2m = ge["mesh"][0], ge["g2m"]
    out = {}

    @torch.no_grad()
    def two_g2m():
        grid_rep, (prior_rep, dec_rep), _ = prior_g2m.encode_step(m.grid_prev_embedder, dec.grid_update_mlp, sources, mesh0,
                                                                  g2m, second=dec.g2m_gnn)
        out["two_g2m"] = (prior_rep, grid_rep, dec_rep)

    @torch.no_grad()
    def emit_emb():
        grid_rep, (prior_rep,), grid_emb = prior_g2m.encode_step(m.grid_prev_embedder, dec.grid_update_mlp, sources, mesh0,
                                                                 g2m, want_grid_emb=True)
        out["emit_emb"] = (prior_rep, grid_rep, dec.g2m_gnn(grid_emb, mesh0, g2m))

    launches = {}
    for name, fn in (("two_g2m", two_g2m), ("emit_emb", emit_emb)):
        with ops.profile_launches() as prof:
            fn()
        launches[name] = [{"kernel": n, "us": round(us, 1), "MB": round(b / 1e6, 1)} for n, us, b in prof.rows]
    for _ in range(3):
        two_g2m()
        emit_emb()
    times = {"two_g2m": [], "emit_emb": []}
    for _ in range(args.rounds):
        for name, fn in (("two_g2m", two_g2m), ("emit_emb", emit_emb)):
            times[name].append(timed(fn, args.iters))
    two_g2m()
    emit_emb()
    torch.cuda.synchronize()
    diff = max((a - b).abs().max().item() for a, b in zip(out["two_g2m"], out["emit_emb"]))
    med = {k: statistics.median(v) for k, v in times.items()}
    print(json.dumps({
        "workload": f"GraphEFM MEPS 268x238 hierarchy {m.level_mesh_sizes}, H=64, latent 64, intra 2/2/4, B={B}",
        "gpu": gpu_info(),
        "forecast_steps_per_s": round(1e3 / ms_step, 2), "ms_per_step": round(ms_step, 3),
        "member_steps_per_s": round(B * 1e3 / ms_step, 1),
        "launches_per_step": len(table), "kernels": table,
        "encoder": {"two_g2m_ms": stats(times["two_g2m"]), "emit_emb_ms": stats(times["emit_emb"]),
                    "speedup": round(med["emit_emb"] / med["two_g2m"], 3), "launches": launches, "max_abs_diff": diff},
    }))


if __name__ == "__main__":
    main()
