"""Training Graph-EFM: the gradient of the ensemble scores and one training step, at BASELINE config 2 size (MEPS 268x238
grid, d = 17, multiscale mesh, H = 64, prior 2 / encoder 2 / decoder 4 m2m layers, latent_dim 64).

  1. the fair CRPS of stored members, forward + backward, B = 1, for each K of ``--members``: ``ensemble.ensemble_stats``
     (ens_stats_kernel, ens_stats_bwd_kernel) against a torch composition that autograds through ``abs`` of the member
     differences one member at a time (as oracle/ensemble_port.py sums them).  ms per call (CUDA events, the two arms
     alternating for ``--rounds`` rounds, medians) and peak memory above the inputs for both; ens_stats_bwd_kernel's µs
     from ``torch.profiler`` in a run of its own and its algorithmic bytes ((K + 1)·G·d·4 read + K·G·d·4 written) over it;
  2. one training step of ``ARForecaster.efm_loss`` (forward + backward + AdamW) for GraphEFMMultiScale, B = 1, K = 2,
     T = 1, with ``crps_weight = 0`` and with ``crps_weight = 0.3`` alternating: ms per step and peak memory ("unavailable"
     with the error on out-of-memory);
  3. the card's name, power limit and SM clocks (nvidia-smi), read in the same run.

Prints one JSON line.

    python scripts/bench_efm_train.py [--members 2 8 32] [--rounds 7] [--iters 20]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from neural_lam_b200 import ensemble, models, synthetic  # noqa: E402


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


def peak_mb(fn):
    """peak device memory allocated during ``fn`` above what was allocated before it, MB"""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return round((torch.cuda.max_memory_allocated() - base) / 1e6, 1)


def spread(v):
    return {"median": round(statistics.median(v), 4), "min": round(min(v), 4), "max": round(max(v), 4)}


def torch_crps(x, interior, y):
    """fair CRPS A - D/2, interior mean, summed over the variables, by autograd through abs one member at a time"""
    K = x.shape[1]
    a = (x - y.unsqueeze(1)).abs().mean(dim=1)
    pairs = torch.zeros_like(a)
    for k in range(K):
        pairs = pairs + (x[:, k:k + 1] - x).abs().sum(dim=1)
    crps = a - 0.5 * pairs / (K * (K - 1))
    return ((crps * interior).sum(dim=1) / interior.sum()).sum()


def kernel_us(fn, name, iters):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    for e in prof.key_averages():
        if name in e.key:
            total = getattr(e, "device_time_total", None)
            total = e.cuda_time_total if total is None else total
            return total / e.count
    raise RuntimeError(f"{name} not found in the profile")


def bench_scores(fc, G, d, K, rounds, iters, dev):
    gen = torch.Generator(device=dev).manual_seed(K)
    x = torch.randn(1, K, G, d, device=dev, generator=gen).requires_grad_()
    y = torch.randn(1, G, d, device=dev, generator=gen)
    interior = fc.interior_mask  # (G, 1)

    def lib():
        x.grad = None
        _, _, sc = ensemble.ensemble_stats(x, interior, y)
        sc.crps_fair.sum().backward()

    def ref():
        x.grad = None
        torch_crps(x, interior, y).backward()

    for _ in range(3):
        lib()
        ref()
    g_lib = x.grad.clone()
    ref()
    rel = ((x.grad - g_lib).abs().max() / x.grad.abs().max()).item()
    times = {"library": [], "torch": []}
    for _ in range(rounds):
        times["library"].append(timed(lib, iters))
        times["torch"].append(timed(ref, iters))
    us = kernel_us(lib, "ens_stats_bwd_kernel", iters)
    nbytes = (K + 1) * G * d * 4 + K * G * d * 4
    return {"K": K, "library_ms": spread(times["library"]), "torch_ms": spread(times["torch"]),
            "torch_over_library": round(statistics.median(times["torch"]) / statistics.median(times["library"]), 2),
            "library_peak_MB": peak_mb(lib), "torch_peak_MB": peak_mb(ref),
            "ens_stats_bwd_kernel_us": round(us, 2), "ens_stats_bwd_kernel_MB": round(nbytes / 1e6, 1),
            "ens_stats_bwd_kernel_GBps": round(nbytes / (us * 1e-6) / 1e9, 1),
            "grad_max_rel_diff_vs_torch": float(f"{rel:.2e}")}


def bench_train_step(ds, spec, rounds, dev):
    torch.manual_seed(0)
    m = models.GraphEFMMultiScale(ds, spec, hidden_dim=64, prior_m2m_layers=2, encoder_m2m_layers=2,
                                  decoder_m2m_layers=4).to(dev).train()
    fc = models.ARForecaster(m, ds).to(dev)
    opt = torch.optim.AdamW(m.parameters(), lr=1e-4)
    G, d, B, T, K = m.num_grid_nodes, 17, 1, 1, 2
    gen = torch.Generator(device=dev).manual_seed(2)
    r = lambda *s: torch.randn(*s, device=dev, generator=gen)  # noqa: E731
    inp = dict(init_states=r(B, 2, G, d), forcing_features=r(B, T, G, 18), boundary_states=r(B, T, G, d),
               target_states=r(B, T, G, d), per_var_std=torch.ones(d, device=dev))
    out = {}
    arms = {f"crps_weight={w}": (lambda w=w: step(w)) for w in (0.0, 0.3)}

    def step(w):
        opt.zero_grad(set_to_none=True)
        fc.efm_loss(**inp, members=K, kl_weight=1.0, crps_weight=w).loss.backward()
        opt.step()

    times = {k: [] for k in arms}
    try:
        for fn in arms.values():
            for _ in range(3):
                fn()
        for _ in range(rounds):
            for k, fn in arms.items():
                times[k].append(timed(fn, 3))
        for k, fn in arms.items():
            out[k] = {"ms_per_step": spread(times[k]), "peak_MB": peak_mb(fn)}
    except torch.cuda.OutOfMemoryError as e:  # noqa: F841
        for k in arms:
            out.setdefault(k, f"unavailable: {str(e).splitlines()[0]}")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--members", type=int, nargs="+", default=[2, 8, 32])
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_efm_train.py needs a CUDA device"
    dev = torch.device("cuda")
    info_before = gpu_info()
    spec = synthetic.make_graph_spec(268, 238, hierarchical=False)
    ds = synthetic.SyntheticDatastore(spec, d_state=17, d_forcing=18, d_static=4, boundary_width=10)
    fc = models.ARForecaster(models.GraphEFMMultiScale(ds, spec, hidden_dim=64), ds).to(dev)
    G = fc.predictor.num_grid_nodes
    scores = []
    for K in args.members:
        scores.append(bench_scores(fc, G, 17, K, args.rounds, args.iters, dev))
        torch.cuda.empty_cache()
    del fc
    torch.cuda.empty_cache()
    train = bench_train_step(ds, spec, args.rounds, dev)
    print(json.dumps({
        "workload": "MEPS 268x238 (G = 63 784), d = 17; scores: B = 1, fair CRPS forward + backward; training step: "
                    "GraphEFMMultiScale H = 64, prior 2 / encoder 2 / decoder 4 m2m, latent 64, B = 1, K = 2, T = 1, "
                    "efm_loss forward + backward + AdamW",
        "gpu_before": info_before, "gpu_after": gpu_info(), "scores": scores, "train_step": train,
    }))


if __name__ == "__main__":
    main()
