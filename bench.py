#!/usr/bin/env python
"""bench.py — forecast-steps/sec of the GraphLAM hot path on one H100.

Workload (BASELINE.json configs[1]): MEPS-shaped 268x238 grid (xy shape (268, 238), as the reference's create_graph takes it), multiscale
mesh (6 561 nodes, 57 616 m2m / 100 656 g2m / 255 136 m2g edges), GraphLAM hidden_dim=64,
4 processor layers, fp32 I/O, synthetic inputs (seeded), random-init weights (seed 42).

One "step" = one autoregressive forecast step (StepPredictor.forward + boundary mix) for a
batch of B independent forecasts (default 32: every sample shares graph and weights, so the batch is
a pure extra row dimension; it also pushes the working set far past the 50 MB L2) on each GPU;
value = forecast-steps/sec = N*B*K / t.
  * `value`     : inputs resident in HBM, the step replayed from a CUDA graph.
  * `e2e`       : ARForecaster public call path with HOST (pinned) buffers: every step copies that
                  step's forcing + boundary states host->device and the predicted state
                  device->host inside the timed region.
  * `roofline`  : the fused m2m InteractionNet layer (all launches of one nlam_inet_fwd call),
                  algorithmic bytes (SURVEY.md 8d) / CUDA-event time with L2 flushed between
                  iterations, against MEASURED_PEAKS.json hbm_gbs.
  * `cpu_baseline` / `--impl reference`: the CPU oracle port of the reference op sequence
                  (oracle/reference_port.py) on the host cores, bounded sample, SAME batch as our arm.
  * `ref_cuda`  : the reference op sequence (index_select + cat + Linear/SiLU/LayerNorm + index_add_, what
                  PyG 2.3.1 without torch-scatter executes) moved to the GPU with TF32 matmuls on, as the
                  reference configures itself (train_model.py:484-488), same batch, CUDA-event timed.
  * `kernels`   : per-launch table of one eager step (library-side CUDA events around every launch):
                  kernel, µs, algorithmic bytes, GB/s, fraction of the measured HBM peak.
  * `parity`    : our step vs the fp64 oracle on the same inputs at the workload's real size (B=2, 1 step).
N>1: one process per GPU (torchrun), independent replicas (the reference's only parallelism is
DDP replicas, README.md:486-514): weak scaling, no data-path collective.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

D_STATE, D_FORCING, D_STATIC = 17, 18, 4
# BASELINE.json configs (1-based as listed there).  Config 2 is the one the metric is quoted on (default); 3 and 4 are
# the H = 128 / 256 workloads (generic wgmma path, tc7.cu), 4 as its single-GPU form (B = 1).
CONFIGS = {
    2: dict(grid=(268, 238), hierarchical=False, n_levels=None, model="graph_lam", hidden=64, layers=4, batch=32,
            workload="MEPS 268x238 grid, multiscale mesh, GraphLAM hidden_dim=64, 4 processor layers (BASELINE.json configs[1])"),
    3: dict(grid=(268, 238), hierarchical=True, n_levels=3, model="hi_lam", hidden=128, layers=6, batch=8,
            workload="MEPS 268x238 grid, 3-level hierarchical mesh, HiLAM hidden_dim=128, 6 processor layers "
                     "(BASELINE.json configs[2])"),
    4: dict(grid=(1024, 1024), hierarchical=False, n_levels=None, model="graph_lam", hidden=256, layers=4, batch=1,
            workload="synthetic 1024x1024 grid, multiscale mesh, GraphLAM hidden_dim=256, 4 processor layers, whole graph on "
                     "ONE GPU (single-GPU form of BASELINE.json configs[3])"),
}
CFG = CONFIGS[2]
METRIC = "forecast-steps/sec (268x238 grid, hidden=64)"


def _peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.isfile(p):
        with open(p) as f:
            d = json.load(f)
        return float(d["hbm_gbs"]), "measured (MEASURED_PEAKS.json)"
    return 3350.0, "fallback (H100 SXM data sheet HBM3 bandwidth, not a measurement)"


def bind_to_gpu_numa(local_rank):
    """Pin this process (and therefore its first-touch pinned host buffers) to the CPUs of the NUMA node the GPU hangs
    off: at 8 ranks the host<->device staging of `e2e` otherwise crosses the socket interconnect.  Best effort."""
    try:
        bus = torch.cuda.get_device_properties(local_rank).pci_bus_id
        dom = torch.cuda.get_device_properties(local_rank).pci_domain_id
        dev = torch.cuda.get_device_properties(local_rank).pci_device_id
        path = f"/sys/bus/pci/devices/{dom:04x}:{bus:02x}:{dev:02x}.0/numa_node"
        node = int(open(path).read().strip())
        if node < 0:
            return None
        cpus = set()
        for part in open(f"/sys/devices/system/node/node{node}/cpulist").read().strip().split(","):
            a, _, z = part.partition("-")
            cpus.update(range(int(a), int(z or a) + 1))
        cpus &= os.sched_getaffinity(0)
        if cpus:
            os.sched_setaffinity(0, cpus)
            return node
    except Exception:
        return None
    return None


def _bf16_peak():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.isfile(p):
        with open(p) as f:
            return float(json.load(f).get("bf16_tflops_sustained", 989.0))
    return 989.0


class ClockSampler:
    """nvidia-smi sampler for SM clocks / throttle reasons during the timed region."""

    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, index=0):
        self.index = index
        self.samples = []
        self._stop = threading.Event()
        self._t = None

    def _run(self):
        while not self._stop.is_set():
            try:
                out = subprocess.run(["nvidia-smi", f"--id={self.index}", f"--query-gpu={self.Q}",
                                      "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=5).stdout
                parts = [x.strip() for x in out.strip().split(",")]
                if len(parts) >= 7:
                    self.samples.append(parts)
            except Exception:
                pass
            self._stop.wait(0.1)

    def __enter__(self):
        self._t = threading.Thread(target=self._run, daemon=True)
        self._t.start()
        return self

    def __exit__(self, *a):
        self._stop.set()
        self._t.join(timeout=6)

    def summary(self):
        if not self.samples:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["no samples"]}
        sm = sorted(float(s[0]) for s in self.samples)
        reasons = set()
        for s in self.samples:
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), s[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": sm[len(sm) // 2], "sm_max_mhz": float(self.samples[0][1]), "reasons": sorted(reasons),
                "samples": len(sm)}


def build_model(device, math="auto"):
    from neural_lam_b200 import models, synthetic

    spec = synthetic.make_graph_spec(*CFG["grid"], hierarchical=CFG["hierarchical"], n_levels=CFG["n_levels"])
    ds = synthetic.SyntheticDatastore(spec, d_state=D_STATE, d_forcing=D_FORCING, d_static=D_STATIC, boundary_width=10)
    torch.manual_seed(42)
    model = models.MODELS[CFG["model"]](ds, spec, hidden_dim=CFG["hidden"], processor_layers=CFG["layers"], math=math)
    fc = models.ARForecaster(model, ds)
    if device is not None:
        fc = fc.to(device)
    fc.eval()
    return spec, ds, model, fc


def synth_inputs(B, T, G, seed=123, pin=False):
    g = torch.Generator().manual_seed(seed)
    init = torch.randn(B, 2, G, D_STATE, generator=g)
    forc = torch.randn(B, T, G, D_FORCING, generator=g)
    bnd = torch.randn(B, T, G, D_STATE, generator=g)
    if pin:
        init, forc, bnd = init.pin_memory(), forc.pin_memory(), bnd.pin_memory()
    return init, forc, bnd


def oracle_setup(model, fc):
    from oracle import reference_port as rp  # noqa: F401  (CPU baseline leg only)

    from neural_lam_b200 import models

    g = {}
    for k in ("grid_static_features", "g2m_features", "m2g_features", "g2m_edge_index", "m2g_edge_index",
              "diff_std", "diff_mean", "m2m_features", "m2m_edge_index", "mesh_static_features", "mesh_up_features",
              "mesh_up_edge_index", "mesh_down_features", "mesh_down_edge_index"):
        if hasattr(model, k):
            v = getattr(model, k)
            g[k] = [t.detach().cpu() for t in v] if isinstance(v, models.BufferList) else v.detach().cpu()
    g["boundary_mask"] = fc.boundary_mask.detach().cpu()
    params = {f"predictor.{k}": v.detach().cpu() for k, v in model.state_dict().items()}
    cfg = dict(model=CFG["model"], hidden_layers=1, processor_layers=CFG["layers"], mesh_aggr="sum")
    return params, g, cfg


def time_cpu_reference(params, g, cfg, G, steps, warmup, B=1):
    """The reference op sequence (CPU oracle port: index_select + cat + Linear/SiLU/LayerNorm +
    index_add_) on all host cores.  Returns (steps/sec, seconds per step, cores)."""
    from oracle import reference_port as rp

    ncpu = os.cpu_count() or 1
    init, forc, bnd = synth_inputs(B, max(1, steps + warmup), G)
    # "all the host threads it can use": torch's intra-op pool does not scale to 100+ threads on
    # these small ops, so probe a few pool sizes with one B=1 step each and keep the fastest
    best = (None, 1e30)
    with torch.no_grad():
        for nt in sorted({ncpu, min(ncpu, 64), min(ncpu, 32), min(ncpu, 16), min(ncpu, 8)}, reverse=True):
            torch.set_num_threads(nt)
            t0 = time.perf_counter()
            rp.ar_rollout(params, g, cfg, init[:1], forc[:1, :1], bnd[:1, :1])
            dt = time.perf_counter() - t0
            if dt < best[1]:
                best = (nt, dt)
            if dt > 20:  # keep the probe bounded
                continue
    cores = best[0]
    torch.set_num_threads(cores)
    with torch.no_grad():
        if warmup:
            rp.ar_rollout(params, g, cfg, init, forc[:, :warmup], bnd[:, :warmup])
        t0 = time.perf_counter()
        rp.ar_rollout(params, g, cfg, init, forc[:, warmup:warmup + steps], bnd[:, warmup:warmup + steps])
        dt = time.perf_counter() - t0
    return B * steps / dt, dt / steps, cores


def algorithmic_bytes_inet(B, Ns, Nr, E, H, update_edges, same_nodes):
    """SURVEY.md 8(d): fp32 forward bytes of one InteractionNet call."""
    nodes_read = Nr if same_nodes else (Ns + Nr)
    return (4 * H * B * (nodes_read + E) + 4 * H * B * (Nr + (E if update_edges else 0))
            + 4 * E + 4 * (Nr + 1) + 4 * (7 * H * H + 8 * H))


def roofline_m2m(model, B, device, iters=20):
    """Time one m2m processor layer (all launches of nlam_inet_fwd) with L2 flushed between
    iterations; achieved = algorithmic bytes / mean CUDA-event time."""
    # GraphLAM: a processor layer over the multiscale mesh; HiLAM: the level-0 same-level layer of the first sweep
    layer = model.processor[0] if hasattr(model, "processor") else model.mesh_down_same_gnns[0][0]
    Nm, E, H = layer.num_rec, layer.num_edges, CFG["hidden"]
    g = torch.Generator(device="cpu").manual_seed(7)
    mesh = torch.randn(B, Nm, H, generator=g).to(device)
    edge = torch.randn(B, E, H, generator=g).to(device)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=device)
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    # as the forecast step runs the middle layers of the processor stack: e' written over e (same bytes moved as the
    # out-of-place call: E rows read, E rows written); the stand-alone out-of-place call is timed next to it
    stacked = hasattr(layer, "forward_stacked")

    def call(inplace):
        if inplace and stacked:
            layer.forward_stacked(mesh, edge, first=False, last=False)
        else:
            layer(mesh, mesh, edge)

    res = {}
    with torch.no_grad():
        for inplace in (False, True):
            for _ in range(3):
                call(inplace)
            torch.cuda.synchronize(device)
            for s, e in ev:
                flush.zero_()
                s.record()
                call(inplace)
                e.record()
            torch.cuda.synchronize(device)
            ms = sorted(s.elapsed_time(e) for s, e in ev)
            res[inplace] = (sum(ms) / len(ms), ms[len(ms) // 2])
    nbytes = algorithmic_bytes_inet(B, Nm, Nm, E, H, True, True)
    return nbytes, res[True][0], res[True][1], res[False][0]



def kernel_table(fc, bufs, peak):
    """One EAGER forecast step with the library's per-launch profile on: [{kernel, us, bytes, gbs, frac}] in launch
    order.  The step's tensors (hundreds of MB at the bench batch) stream through the 50 MB L2 exactly as in the
    replayed step; the launches are the same ones the CUDA graph holds."""
    import ctypes

    from neural_lam_b200 import _lib

    L = _lib.lib()
    with torch.no_grad():
        fc._one_step(bufs, 0)
        torch.cuda.synchronize()
        L.nlam_profile_enable(1)
        fc._one_step(bufs, 0)
        torch.cuda.synchronize()
        n = L.nlam_profile_count()
        rows = []
        name = ctypes.create_string_buffer(96)
        ms, nb = ctypes.c_float(), ctypes.c_double()
        for i in range(n):
            _lib.check(L.nlam_profile_get(i, name, 96, ctypes.byref(ms), ctypes.byref(nb)))
            us = ms.value * 1e3
            gbs = nb.value / (us * 1e-6) / 1e9 if us > 0 else 0.0
            rows.append({"kernel": name.value.decode(), "us": round(us, 1), "bytes": int(nb.value),
                         "gbs": round(gbs, 1), "frac": round(gbs / peak, 3)})
        L.nlam_profile_enable(0)
    return rows


def time_ref_cuda(model, fc, device, B, steps, warmup):
    """The reference op sequence on the GPU (the reference's "PyG/CUDA path"): oracle/reference_port.ar_rollout —
    index_select gathers, cat, nn.Linear-equivalent matmuls, SiLU, LayerNorm, index_add_ scatter — on CUDA tensors
    with TF32 matmuls enabled as the reference does (train_model.py:484-488).  Returns (steps/s, ms per step)."""
    from oracle import reference_port as rp

    params, g, cfg = oracle_setup(model, fc)
    params = {k: v.to(device) for k, v in params.items()}
    g = {k: ([t.to(device) for t in v] if isinstance(v, list) else v.to(device)) for k, v in g.items()}
    G = model.num_grid_nodes
    init, forc, bnd = (t.to(device) for t in synth_inputs(B, steps + warmup, G, seed=321))
    old = torch.get_float32_matmul_precision()
    torch.set_float32_matmul_precision("high")
    try:
        with torch.no_grad():
            rp.ar_rollout(params, g, cfg, init, forc[:, :warmup], bnd[:, :warmup])
            torch.cuda.synchronize(device)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            rp.ar_rollout(params, g, cfg, init, forc[:, warmup:], bnd[:, warmup:])
            e1.record()
            torch.cuda.synchronize(device)
    finally:
        torch.set_float32_matmul_precision(old)
    ms = e0.elapsed_time(e1) / steps
    return B / (ms * 1e-3), ms


def parity_check(model, fc, device, B=2):
    """Our step vs the fp64 CPU oracle at the workload's real size: max abs / max rel error of one forecast step,
    next to the error of the reference's own GPU configuration (fp32 oracle with TF32-rounded matmul operands)."""
    from oracle import reference_port as rp

    params, g, cfg = oracle_setup(model, fc)
    G = model.num_grid_nodes
    init, forc, bnd = synth_inputs(B, 1, G, seed=777)
    with torch.no_grad():
        want = rp.ar_rollout({k: v.double() for k, v in params.items()}, g, cfg, init.double(), forc.double(), bnd.double())
        with rp.tf32_matmul():
            ref = rp.ar_rollout(params, g, cfg, init, forc, bnd)
        got = fc.rollout_graphed(init.to(device), forc.to(device), bnd.to(device)).cpu().double()
    err = (got - want).abs()
    return {"max_abs": err.max().item(), "max_rel": (err / want.abs().clamp(min=1.0)).max().item(),
            "reference_tf32_max_abs": (ref.double() - want).abs().max().item(),
            "what": f"1 forecast step, B={B}, real-size workload, vs fp64 oracle (rel = |err|/max(|x|,1))"}


def step_algorithmic(model, B):
    """Algorithmic fp32 bytes and FLOPs of one forecast step of B forecasts (SURVEY.md 8d formulas: every InteractionNet
    call + the grid-side MLPs; input-independent embedders excluded, they are cached)."""
    from neural_lam_b200.gnn_layers import InteractionNet

    H = CFG["hidden"]
    G = model.num_grid_nodes
    nbytes = flops = 0.0
    for name, mod in model.named_modules():
        if isinstance(mod, InteractionNet):
            E, Nr = mod.num_edges, mod.num_rec
            Ns = mod.num_send_min
            same = name.startswith(("processor", "mesh_down_same", "mesh_up_same"))
            nbytes += algorithmic_bytes_inet(B, Ns, Nr, E, H, mod.update_edges, same)
            flops += B * (8.0 * H * H * E + 6.0 * H * H * Nr)
    d_in = D_STATE * 2 + D_FORCING + D_STATIC
    rows = float(B) * G
    nbytes += 4 * rows * (d_in + H) + 4 * rows * 2 * H + 4 * rows * (H + 3 * D_STATE)   # embedder, encoding, output_map+epilogue
    flops += 2 * rows * (d_in * H + H * H) + 2 * rows * 2 * H * H + 2 * rows * (H * H + H * D_STATE)
    return nbytes, flops




def measure_train_step(model, device, B=4, iters=5):
    """One TRAINING step of the step predictor (forward + backward of a weighted-MSE-like loss; the optimiser step is
    plain torch AdamW as in the reference, models/module.py:303) at the reference's default batch size 4
    (train_model.py:261-263): our kernels (tensor-core forward, hand-written backward) next to the reference op sequence
    under autograd on the same GPU with TF32 matmuls.  Returns a dict (ms per step, samples/s, both arms)."""
    from oracle import reference_port as rp

    G = model.num_grid_nodes
    g = torch.Generator().manual_seed(17)
    prev, pprev = torch.randn(B, G, D_STATE, generator=g).to(device), torch.randn(B, G, D_STATE, generator=g).to(device)
    forc, tgt = torch.randn(B, G, D_FORCING, generator=g).to(device), torch.randn(B, G, D_STATE, generator=g).to(device)
    opt = torch.optim.AdamW(model.parameters(), lr=1e-4, betas=(0.9, 0.95))

    def ours():
        opt.zero_grad(set_to_none=True)
        pred, _ = model(prev, pprev, forc)
        ((pred - tgt) ** 2).mean().backward()
        opt.step()

    def timed(fn):
        for _ in range(2):
            fn()
        torch.cuda.synchronize(device)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize(device)
        return e0.elapsed_time(e1) / iters

    model.train()
    ms_ours = timed(ours)
    model.eval()
    # reference arm: the oracle op sequence with autograd, parameters as leaf tensors, same optimiser
    sd = {k: v.detach().clone().to(device) for k, v in model.state_dict().items()}
    params = {k: (v.requires_grad_(True) if v.is_floating_point() else v) for k, v in sd.items()}
    graph = {}
    from neural_lam_b200 import models as _m

    for k in ("grid_static_features", "g2m_features", "m2g_features", "g2m_edge_index", "m2g_edge_index", "diff_std", "diff_mean",
              "m2m_features", "m2m_edge_index", "mesh_static_features", "mesh_up_features", "mesh_up_edge_index",
              "mesh_down_features", "mesh_down_edge_index"):
        if hasattr(model, k):
            v = getattr(model, k)
            graph[k] = [t.detach() for t in v] if isinstance(v, _m.BufferList) else v.detach()
    cfg = dict(model=CFG["model"], hidden_layers=1, processor_layers=CFG["layers"], mesh_aggr="sum")
    ropt = torch.optim.AdamW([p for p in params.values() if p.is_floating_point()], lr=1e-4, betas=(0.9, 0.95))
    old = torch.get_float32_matmul_precision()
    torch.set_float32_matmul_precision("high")

    def ref():
        ropt.zero_grad(set_to_none=True)
        pred = rp.graph_model_forward(params, graph, cfg, prev, pprev, forc)
        ((pred - tgt) ** 2).mean().backward()
        ropt.step()

    try:
        ms_ref = timed(ref)
    finally:
        torch.set_float32_matmul_precision(old)
    return {"batch": B, "ms_per_step": ms_ours, "value": B / (ms_ours * 1e-3), "unit": "training samples/s",
            "ref_cuda_ms_per_step": ms_ref, "ref_cuda_value": B / (ms_ref * 1e-3), "speedup": ms_ref / ms_ours,
            "what": "forward + backward + AdamW step of one forecast step; ours = wgmma forward kernels + hand-written "
                    "backward (backward.py), reference arm = the reference op sequence under torch autograd with TF32 matmuls"}


def measure_partition(cfg_id, device, rank, world, steps, warmup, math="auto", batch=None):
    """STRONG-scaling measurement of the node-partitioned rollout (SURVEY.md 8e; BASELINE.json configs[3] shape by
    default): ONE batch of forecasts on the whole graph, grid and every mesh level split into `world` contiguous strips,
    one halo exchange per InteractionNet call — ``halo_push_kernel`` stores boundary rows straight into the peers'
    symmetric-memory buffers over NVLink, one device barrier, all of it inside the captured CUDA graph.  world == 1 runs
    the plain model on the same workload (the strong-scaling reference).  Every rank returns the dict (rank 0 prints)."""
    import torch.distributed as dist

    from neural_lam_b200 import dist as nd
    from neural_lam_b200 import models, synthetic

    c = CONFIGS[cfg_id]
    B = batch or c["batch"]
    spec = synthetic.make_graph_spec(*c["grid"], hierarchical=c["hierarchical"], n_levels=c["n_levels"])
    ds = synthetic.SyntheticDatastore(spec, d_state=D_STATE, d_forcing=D_FORCING, d_static=D_STATIC, boundary_width=10)
    cls = models.MODELS[c["model"]]
    torch.manual_seed(42)
    if world > 1:
        model = nd.partition_model(cls, ds, spec, rank, world, hidden_dim=c["hidden"], processor_layers=c["layers"], math=math)
        lds, sl = model.local_datastore, model.own_grid_slice()
    else:
        model = cls(ds, spec, hidden_dim=c["hidden"], processor_layers=c["layers"], math=math)
        lds, sl = ds, slice(0, ds.num_grid_nodes)
    fc = models.ARForecaster(model, lds).to(device).eval()
    G_own = sl.stop - sl.start
    T = steps + warmup
    g = torch.Generator().manual_seed(99)
    init = torch.randn(B, 2, G_own, D_STATE, generator=g).pin_memory()
    forc = torch.randn(B, T, G_own, D_FORCING, generator=g).pin_memory()
    bnd = torch.randn(B, T, G_own, D_STATE, generator=g).pin_memory()
    d_init, d_forc, d_bnd = init.to(device), forc.to(device), bnd.to(device)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize(device)

    with torch.no_grad():
        bufs = fc.capture(B)
        fc.set_state(d_init[:, 0], d_init[:, 1])

        def run(t0, n):
            for i in range(t0, t0 + n):
                bufs["forcing"].copy_(d_forc[:, i])
                bufs["boundary"].copy_(d_bnd[:, i])
                fc.replay_step()

        run(0, warmup)
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run(warmup, steps)
        e1.record()
        barrier()
        dev_ms = e0.elapsed_time(e1)
        h_out = torch.empty(B, steps, G_own, D_STATE).pin_memory()
        fc.rollout_from_host(init, forc[:, :warmup], bnd[:, :warmup])
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fc.rollout_from_host(init, forc[:, warmup:], bnd[:, warmup:], out=h_out)
        e1.record()
        barrier()
        e2e_ms = e0.elapsed_time(e1)
    t = torch.tensor([dev_ms, e2e_ms], device=device, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    dev_ms, e2e_ms = t.tolist()
    out = {"workload": c["workload"], "batch": B, "n_gpus": world, "scaling": "strong",
           "value": B * steps / (dev_ms * 1e-3), "unit": "forecast-steps/s", "ms_per_step": dev_ms / steps,
           "e2e": {"value": B * steps / (e2e_ms * 1e-3), "unit": "forecast-steps/s",
                   "h2d_bytes_per_step": fc.host_io_bytes_per_step(B)[0],
                   "d2h_bytes_per_step": fc.host_io_bytes_per_step(B)[1]},
           "parallelism": ("single GPU, whole graph" if world == 1 else
                           f"node partition x{world}: grid + every mesh level in {world} strips, halo rows pushed into the "
                           "peers' symmetric-memory buffers by halo_push_kernel over NVLink, one device barrier per "
                           "InteractionNet call, captured in the CUDA graph")}
    if world > 1:
        sent, recv = model.halo_bytes_per_step(B)
        out["comm"] = {"halo_exchanges_per_step": len(nd._gnn_edge_sets(model)), "halo_bytes_sent_per_step_rank0": sent,
                       "halo_bytes_received_per_step_rank0": recv, "transport": type(model.exchanger).__name__}
    del fc, model, bufs
    torch.cuda.empty_cache()
    return out


def dump_outputs(out_dir, new_state, max_nodes=16384):
    """Write what the timed path returned in its last step: the new state (B, G, d_state), float32.  At the default
    batch it exceeds 64 MB, so a fixed sample of grid nodes (seeded, sorted; every batch element and variable) is
    written: new_state.npy (B, min(G, max_nodes), d_state)."""
    import numpy as np

    G = new_state.shape[1]
    gen = torch.Generator().manual_seed(0)
    nodes = torch.arange(G) if G <= max_nodes else torch.randperm(G, generator=gen)[:max_nodes].sort().values
    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, "new_state.npy"),
            new_state[:, nodes.to(new_state.device)].float().cpu().numpy())


def run_ours(args):
    import torch.distributed as dist

    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    assert torch.cuda.is_available(), "bench.py needs a CUDA device (no CPU fallback)"
    device = torch.device("cuda", local_rank)
    torch.cuda.set_device(device)
    numa_node = bind_to_gpu_numa(local_rank) if world > 1 else None
    import __graft_entry__

    __graft_entry__.build()
    from neural_lam_b200 import _lib

    B, K, W = args.batch, args.steps, max(args.warmup, 3)
    if args.parallelism == "partition":
        res = measure_partition(args.config, device, rank, world, K, W, args.math, batch=args.batch)
        if rank == 0:
            line = {"metric": METRIC, "value": res["value"], "unit": res["unit"], "n_gpus": world, "steps": K, "warmup": W,
                    "ms_per_step": res["ms_per_step"], "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
                    "dtype": "f32 I/O; tf32 tensor-core MLPs, f32 accumulate", "data": "synthetic",
                    "config": {"workload": res["workload"], "global_batch": res["batch"], "parallelism": res["parallelism"],
                               "cuda_graph": True}, "e2e": res["e2e"], "comm": res.get("comm")}
            print(json.dumps(line))
        if world > 1:
            dist.barrier()
            dist.destroy_process_group()
        return
    spec, ds, model, fc = build_model(device, math=args.math)
    G = model.num_grid_nodes
    T = K + W
    init, forc, bnd = synth_inputs(B, T, G, seed=123 + rank, pin=True)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize(device)

    # ------------------------------------------------------------------ device-resident value
    d_init, d_forc, d_bnd = init.to(device), forc.to(device), bnd.to(device)
    with torch.no_grad():
        n0 = _lib.lib().nlam_launch_count()
        bufs = fc.capture(B)
        # launches of OUR kernels per captured step = those issued during the capture pass
        n1 = _lib.lib().nlam_launch_count()
        fc._one_step(bufs, 0)  # eager step to count launches per step exactly
        launches_per_step = _lib.lib().nlam_launch_count() - n1
        del n0

        def graphed_steps(t0, n):
            # one AR step = stage this step's forcing / boundary (already in HBM) + replay the captured step; the
            # state feedback is a rotation of the captured graphs' three state buffers (no copies).  Returns the buffer
            # holding the last step's new state.
            new_state = None
            for i in range(t0, t0 + n):
                bufs["forcing"].copy_(d_forc[:, i])
                bufs["boundary"].copy_(d_bnd[:, i])
                new_state = fc.replay_step()
            return new_state

        fc.set_state(d_init[:, 0], d_init[:, 1])
        graphed_steps(0, W)
        barrier()
        with ClockSampler(local_rank) as clk:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            last_state = graphed_steps(W, K)
            e1.record()
            barrier()
            dev_ms = e0.elapsed_time(e1)
            if args.dump_outputs and rank == 0:
                dump_outputs(args.dump_outputs, last_state)
            # keep the sampler alive for at least ~0.5 s of load for short runs
            if dev_ms < 500:
                t_end = time.time() + 0.6
                while time.time() < t_end:
                    graphed_steps(W, 1)
                torch.cuda.synchronize(device)
        clocks = clk.summary()

        # ------------------------------------------------------------------ end-to-end (host buffers)
        # public API: ARForecaster.rollout_from_host — pinned host tensors in, pinned host tensor
        # out; per step H2D(forcing, boundary) + graph replay + D2H(prediction) in the timed region
        h_out = torch.empty(B, K, G, D_STATE).pin_memory()
        h_warm = torch.empty(B, W, G, D_STATE).pin_memory()
        fc.rollout_from_host(init, forc[:, :W], bnd[:, :W], out=h_warm)
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fc.rollout_from_host(init, forc[:, W:], bnd[:, W:], out=h_out)
        e1.record()
        barrier()
        e2e_ms = e0.elapsed_time(e1)

    t = torch.tensor([dev_ms, e2e_ms], device=device, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    dev_ms, e2e_ms = t.tolist()

    partition = None
    if not args.no_partition and args.config == 2:
        # second measurement of the same run: the node-partitioned rollout (strong scaling) on BASELINE config 4's
        # shape; at N = 1 this is the unpartitioned reference the N > 1 lines are compared with
        partition = measure_partition(4, device, rank, world, steps=min(K, 10), warmup=3, math=args.math)

    if rank == 0:
        peak, peak_src = _peaks()
        with torch.no_grad():
            nbytes, mean_ms, med_ms, oop_ms = roofline_m2m(model, B, device)
        achieved = nbytes / (mean_ms * 1e-3) / 1e9
        # DRAM traffic of the roofline kernel from an `ncu --set full` capture AT THIS BATCH (profiles/traffic.json:
        # {"m2m_layer_dram_bytes": {"<B>": bytes}}); null when no capture exists for the batch that was run
        traffic = None
        tp = os.path.join(ROOT, "profiles", "traffic.json")
        if os.path.isfile(tp):
            try:
                traffic = json.load(open(tp)).get("m2m_layer_inplace_dram_bytes", {}).get(str(B))
            except Exception:
                traffic = None
        sb, sf = step_algorithmic(model, B)
        t_step = dev_ms / K * 1e-3
        tf32_peak = 0.5 * _bf16_peak()
        step_roof = {"algorithmic_bytes": sb, "flops": sf, "hbm_gbs": sb / t_step / 1e9, "hbm_frac": sb / t_step / 1e9 / peak,
                     "tflops": sf / t_step / 1e12, "tensor_frac": sf / t_step / 1e12 / tf32_peak,
                     "tensor_peak": tf32_peak, "tensor_peak_source": "0.5 x dense bf16 (MEASURED_PEAKS.json if present, else the H100 "
                     "SXM data sheet's 989 TFLOP/s); a TF32 peak was not measured", "binding": "tensor" if sf / tf32_peak / 1e12 > sb / peak / 1e9 else "hbm"}
        kernels = kernel_table(fc, bufs, peak)
        train = None
        if not args.no_train:
            # reference default batch 4 (train_model.py:261-263); the 1024^2 H=256 workload trains one sample per GPU
            tb = 1 if args.config == 4 else 4
            try:
                with torch.enable_grad():
                    train = measure_train_step(model, device, B=tb)
            except torch.OutOfMemoryError as e:  # recompute-in-backward workspaces of the largest layer
                train = {"batch": tb, "unavailable": "out of device memory: " + str(e).split(".")[0]}
                for p_ in model.parameters():
                    p_.grad = None
                torch.cuda.empty_cache()
        parity = None if args.no_parity else parity_check(model, fc, device)
        ref_cuda = None
        if not args.no_ref_cuda:
            v, ms = time_ref_cuda(model, fc, device, B, steps=min(K, 10), warmup=2)
            ref_cuda = {"value": v, "unit": "forecast-steps/s", "ms_per_step": ms, "batch_per_gpu": B,
                        "what": "reference op sequence (oracle port of gnn_layers.py + PyG 2.3.1 gather/scatter_add + "
                                "graph/base.py) on this GPU, torch fp32 with TF32 matmuls (train_model.py:484-488), eager"}
        cpu = None
        if world >= 1 and not args.no_cpu_baseline:
            params, g, cfg = oracle_setup(model, fc)
            n_cpu = max(1, min(args.cpu_steps, 2))
            v, sec, cores = time_cpu_reference(params, g, cfg, G, steps=n_cpu, warmup=1, B=B)
            cpu = {"value": v, "unit": "forecast-steps/s", "cores": cores, "kind": "port",
                   "sample": f"B={B} (same batch as the GPU arm), {n_cpu} AR steps of the same GraphLAM config after 1 "
                             f"warm-up ({sec:.3f} s per step of {B} forecasts, torch CPU {torch.get_num_threads()} threads)"}
        h2d, d2h = fc.host_io_bytes_per_step(B)  # forcing + the boundary-mask rows of the boundary state in, prediction out
        line = {
            "metric": METRIC,
            "value": world * B * K / (dev_ms * 1e-3),
            "unit": "forecast-steps/s",
            "n_gpus": world, "steps": K, "warmup": W,
            "ms_per_step": dev_ms / K,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "f32 I/O; " + ("tf32 tensor-core MLPs, f32 accumulate" if args.math != "fp32" else "f32 FFMA"),
            "data": "synthetic",
            "config": {"workload": CFG["workload"],
                       "batch_per_gpu": B, "global_batch": world * B, "math": args.math,
                       "parallelism": f"replicas x{world} (independent forecasts per GPU, no collective)",
                       "l2": "per-step working set (~0.36 GB x B algorithmic) exceeds the 50 MB L2; "
                             "roofline kernel timed with an explicit 256 MB L2 flush between iterations",
                       "cuda_graph": True, "numa_node_rank0": numa_node},
            "e2e": {"value": world * B * K / (e2e_ms * 1e-3), "unit": "forecast-steps/s",
                    "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": d2h},
            "gpu_launches": int(launches_per_step) * K,
            "gpu_launches_per_step": int(launches_per_step),
            "clocks": clocks,
            "roofline": {"bound": "hbm", "kernel": "m2m InteractionNet layer as the step runs its middle layers (nlam_inet_fwd, "
                                                   "edge tensor updated in place; all 3 launches)",
                         "out_of_place_ms": oop_ms,
                         "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
                         "traffic": traffic, "algorithmic_bytes": nbytes, "ms_mean": mean_ms, "ms_median": med_ms,
                         "peak_source": peak_src, "l2_flushed": True},
            "step_roofline": step_roof,
            "partition": partition,
            "train": train,
            "cpu_baseline": cpu,
            "ref_cuda": ref_cuda,
            "parity": parity,
            "kernels": kernels,
        }
        if ref_cuda:
            line["ref_cuda"]["speedup_device_resident"] = line["value"] / world / ref_cuda["value"]
        print(json.dumps(line))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def run_reference(args):
    """Reference arm: the reference's own CPU implementation of the path.  torch_geometric /
    pytorch_lightning are not installable here (no network, not in /opt/wheelhouse), so
    `baseline/_ref` cannot exist; per the tier rules the arm times the CPU oracle port of the
    reference op sequence (kind "port") on all host cores."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    spec, ds, model, fc = build_model(None)
    params, g, cfg = oracle_setup(model, fc)
    K, W = args.steps, args.warmup
    B = args.batch
    # each step = one forecast step of the SAME batch as our arm (B forecasts); bounded sample of the K steps
    k = max(1, min(K, args.cpu_steps, 3))
    v, sec, cores = time_cpu_reference(params, g, cfg, model.num_grid_nodes, steps=k, warmup=min(W, 1), B=B)
    line = {
        "impl": "reference",
        "metric": METRIC,
        "value": v, "unit": "forecast-steps/s", "n_gpus": int(os.environ.get("WORLD_SIZE", "1")),
        "steps": K, "warmup": W, "ms_per_step": sec * 1e3, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": CFG["workload"], "batch_per_gpu": B, "global_batch": B,
                   "math": "f32 (torch CPU)", "parallelism": "host cores of one box"},
        "cpu_baseline": {"value": v, "unit": "forecast-steps/s", "cores": cores, "kind": "port",
                         "sample": f"each step = one forecast step of B={B} forecasts on the host cores; {k} timed steps "
                                   f"(bounded from --steps {K})"},
        "e2e": {"value": v, "unit": "forecast-steps/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }
    print(json.dumps(line))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--config", type=int, default=2, choices=sorted(CONFIGS),
                    help="BASELINE.json config (1-based): 2 = the metric's workload (default), 3 = HiLAM H=128, 4 = 1024^2 H=256")
    ap.add_argument("--batch", type=int, default=0, help="independent forecasts (ensemble members) per GPU per step "
                                                          "(default: 32 / 8 / 1 for configs 2 / 3 / 4)")
    ap.add_argument("--math", default="auto", choices=["auto", "tf32", "fp32"])
    ap.add_argument("--cpu-steps", type=int, default=5)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-ref-cuda", action="store_true")
    ap.add_argument("--no-parity", action="store_true")
    ap.add_argument("--no-train", action="store_true", help="skip the training-step (forward + backward) measurement")
    ap.add_argument("--no-partition", action="store_true", help="skip the node-partition (strong scaling) sub-measurement")
    ap.add_argument("--parallelism", default="replicas", choices=["replicas", "partition"],
                    help="replicas: independent forecasts per GPU (weak scaling, the headline line); partition: ONE batch "
                         "on the node-partitioned graph (strong scaling; --config selects the workload, default 4)")
    ap.add_argument("--cpu-at-scale", action="store_true", help="time the CPU port even for config 4 (minutes)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write the last step's new state (a fixed sample of grid nodes) as "
                         "DIR/new_state.npy (float32); inputs and weights are seeded, so runs with the same arguments "
                         "are comparable output for output")
    args = ap.parse_args()
    if args.dump_outputs and (args.parallelism == "partition" or args.impl == "reference"):
        ap.error("--dump-outputs writes the replicated device-resident step's outputs: not available with "
                 "--parallelism partition or --impl reference")
    global CFG, METRIC
    CFG = CONFIGS[args.config]
    METRIC = ("forecast-steps/sec (268x238 grid, hidden=64)" if args.config == 2 else
              f"forecast-steps/sec ({CFG['grid'][0]}x{CFG['grid'][1]} grid, hidden={CFG['hidden']}, BASELINE config {args.config})")
    if args.parallelism == "partition" and args.config == 2 and "--config" not in sys.argv:
        args.config = 4
        CFG = CONFIGS[4]
        METRIC = f"forecast-steps/sec ({CFG['grid'][0]}x{CFG['grid'][1]} grid, hidden={CFG['hidden']}, BASELINE config 4)"
    if not args.batch:
        args.batch = CFG["batch"]
    if args.config == 4:  # the fp64 / fp32 CPU oracle takes minutes per step at 1 M grid nodes
        args.no_parity = True
        args.no_cpu_baseline = args.no_cpu_baseline or not args.cpu_at_scale
    if args.impl == "reference":
        run_reference(args)
    else:
        run_ours(args)


if __name__ == "__main__":
    main()
