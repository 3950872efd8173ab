"""The forecast step of a model that predicts its std, at BASELINE config 2 size (MEPS 268x238 grid, GraphLAM H = 64, 4
processor layers, 17 state variables, output_std=True: output_map 64 -> 64 -> 34), B forecasts per step, in one run:

  1. alternating rounds of ``--iters`` steps each, CUDA events around each round, of
       * the captured std step (``ARForecaster.capture``: the fused decoder writes the softplus std beside the new state),
       * the captured step of the same model without a std (output_map 64 -> 64 -> 17),
       * the eager no-grad ``forward`` of the std model (the m2g layer, output_map and the step epilogue as separate
         launches, the updated grid representation through HBM), which the captured std step replaces;
  2. the kernel table of one captured-path step of the std model (``ops.profile_launches``: name, µs, algorithmic bytes);
  3. the card's name, power limit and max SM clock (nvidia-smi), read in the same run.

Prints one JSON line.

    python scripts/bench_std.py [--batch 32] [--rounds 7] [--iters 20] [--warmup 5]
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
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_std.py needs a CUDA device"
    dev = torch.device("cuda")
    B = args.batch
    spec = synthetic.make_graph_spec(268, 238, hierarchical=False)
    ds = synthetic.SyntheticDatastore(spec, d_state=17, d_forcing=18, d_static=4, boundary_width=10)
    fcs = {}
    for std in (True, False):
        torch.manual_seed(0)
        m = models.GraphLAM(ds, spec, hidden_dim=64, processor_layers=4, output_std=std)
        fcs[std] = models.ARForecaster(m, ds).to(dev).eval()
    m_std = fcs[True].predictor
    G, d = m_std.num_grid_nodes, m_std.num_state_vars
    gen = torch.Generator(device=dev).manual_seed(1)
    forcing = torch.randn(B, G, 18, device=dev, generator=gen)
    bnd = torch.randn(B, G, d, device=dev, generator=gen)
    prev, prev_prev = torch.randn(B, G, d, device=dev, generator=gen), torch.randn(B, G, d, device=dev, generator=gen)
    for fc in fcs.values():
        bufs = fc.capture(B)
        bufs["forcing"].copy_(forcing)
        bufs["boundary"].copy_(bnd)
        fc.set_state(prev_prev, prev)

    def eager():
        m_std(prev, prev_prev, forcing)

    runs = {"captured_std_step": fcs[True].replay_step, "captured_step_no_std": fcs[False].replay_step, "eager_std_forward": eager}
    with torch.no_grad():
        for fn in runs.values():
            timed(fn, args.warmup)
        ms = {k: [] for k in runs}
        for _ in range(args.rounds):
            for k, fn in runs.items():
                ms[k].append(timed(fn, args.iters))
        # one captured-path step of the std model, eagerly, with per-launch events
        std_out = torch.empty(B, G, d, device=dev)
        out = torch.empty(B, G, d, device=dev)
        m_std.forward_with_boundary(prev, prev_prev, forcing, bnd, fcs[True].boundary_mask, out=out, std_out=std_out)
        with ops.profile_launches() as prof:
            m_std.forward_with_boundary(prev, prev_prev, forcing, bnd, fcs[True].boundary_mask, out=out, std_out=std_out)
    result = {
        "workload": f"config 2 GraphLAM H=64 P=4, d_state=17, output_std, B={B}",
        "gpu": gpu_info(),
        "rounds": args.rounds, "iters_per_round": args.iters,
        **{f"{k}_ms": {"median": statistics.median(v), "min": min(v), "max": max(v)} for k, v in ms.items()},
        "std_write_bytes_per_step": 4 * B * G * d,
        "kernels": [{"name": n, "us": round(us, 1), "bytes": b} for n, us, b in prof.rows],
    }
    print(json.dumps(result))


if __name__ == "__main__":
    main()
