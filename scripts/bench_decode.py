"""Time the mesh -> grid decoder of one forecast step at bench.py config 2 size (MEPS 268x238 grid, GraphLAM H = 64), two ways
on the same inputs, alternating:

  old:   edge-only InteractionNet (tc_rowlinear_kernel for P_s / P_r, tc_ell_window_kernel) + tc_node_out_kernel
         (``aggregate_only`` + ``ops.node_update_step``)
  fused: tc_rowlinear_kernel for P_s / P_e + tc_decode_kernel (``decode_step``)

Each round times ITERS calls of one variant with CUDA events; rounds alternate old / fused.  Prints one JSON line: median,
min and max ms per call of each, the speed-up of the medians, and the maximum absolute difference of the two outputs.

    python scripts/bench_decode.py [--batch 32] [--rounds 7] [--iters 50]

With --base-lib PATH the fused decoder of two builds of libnlam_b200.so is compared instead (PATH: another build, for
example the parent commit's, in a directory git ignores).  Each round runs one subprocess per library
(`_lib.LIB_PATH` set before the library loads), in alternating order, on the same seeded inputs; a worker times ITERS
calls of the decoder's two launches (tc_rowlinear_kernel, tc_decode_kernel) from the library's per-launch profile and
takes their medians.  Prints one JSON line: per batch size, the median, min and max over the rounds in ms of both launches
together and of tc_decode_kernel alone, the algorithmic GB/s of tc_decode_kernel's median and its share of the data sheet's
3.35 TB/s, and the maximum |difference| of the outputs of the two libraries; plus the card's name, power limit and SM clock.

    python scripts/bench_decode.py --base-lib PATH [--rounds 7] [--iters 30] [--batch 32 8]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HBM_TBS = 3.35  # H100 SXM data sheet
LAUNCHES = ("tc_rowlinear_kernel", "tc_decode_kernel")


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def setup(B):
    """config 2's model and seeded decoder inputs at batch size B"""
    import torch
    from neural_lam_b200 import models, synthetic

    assert torch.cuda.is_available(), "bench_decode.py needs a CUDA device"
    dev = torch.device("cuda")
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
    return m, net, out_map, mesh, grid, m2g, prev, bnd, mask


def worker(lib_path, batches, iters, out_path):
    sys.path.insert(0, ROOT)
    from neural_lam_b200 import _lib
    _lib.LIB_PATH = lib_path
    import torch
    from neural_lam_b200 import ops

    res, outs = {}, {}
    for B in batches:
        m, net, _, mesh, grid, m2g, prev, bnd, mask = setup(B)
        out = torch.empty_like(prev)

        @torch.no_grad()
        def fused():
            r = net.decode_step(mesh, grid, m2g, m.output_map, prev, bnd, mask, m.diff_std, m.diff_mean, out=out)
            assert r is not None, "decode_step does not cover this shape"

        for _ in range(3):
            fused()
        torch.cuda.synchronize()
        outs[str(B)] = out.cpu()
        per = {k: [] for k in LAUNCHES}
        nbytes = 0.0
        with ops.profile_launches() as prof:
            for _ in range(iters):
                fused()
        for row in prof.rows:
            assert row[0] in per, row[0]
            per[row[0]].append(row[1])
            if row[0] == "tc_decode_kernel":
                nbytes = row[2]
        assert all(len(v) == iters for v in per.values()), {k: len(v) for k, v in per.items()}
        res[str(B)] = {"both_ms": statistics.median([a + b for a, b in zip(*per.values())]) / 1e3,
                       "decode_ms": statistics.median(per["tc_decode_kernel"]) / 1e3, "bytes": nbytes}
    torch.save(outs, out_path + ".pt")
    with open(out_path, "w") as f:
        json.dump(res, f)


def compare_libs(args):
    new_lib = os.path.join(ROOT, "neural_lam_b200", "lib", "libnlam_b200.so")
    assert os.path.isfile(args.base_lib), "--base-lib: path of the library to compare against"
    libs = {"base": os.path.abspath(args.base_lib), "new": new_lib}
    runs = {k: [] for k in libs}
    with tempfile.TemporaryDirectory() as tmp:
        for r in range(args.rounds):
            for tag in (("base", "new") if r % 2 == 0 else ("new", "base")):
                out = os.path.join(tmp, f"{tag}_{r}.json")
                subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", libs[tag], "--out", out, "--iters",
                                str(args.iters), "--batch", *map(str, args.batch)], check=True)
                with open(out) as f:
                    runs[tag].append(json.load(f))
        import torch
        base_out, new_out = torch.load(os.path.join(tmp, "base_0.json.pt")), torch.load(os.path.join(tmp, "new_0.json.pt"))
    res = {"gpu": gpu_info(), "rounds": args.rounds, "iters": args.iters}
    for B in map(str, args.batch):
        entry = {}
        for tag in libs:
            entry[tag] = {}
            for what in ("both_ms", "decode_ms"):
                t = [run[B][what] for run in runs[tag]]
                entry[tag][what] = {"median": round(statistics.median(t), 4), "min": round(min(t), 4), "max": round(max(t), 4)}
            gbs = runs[tag][0][B]["bytes"] / (entry[tag]["decode_ms"]["median"] * 1e6)
            entry[tag]["decode_gb_s"] = round(gbs, 1)
            entry[tag]["decode_hbm_share"] = round(gbs / (HBM_TBS * 1e3), 3)
        entry["speedup_both"] = round(entry["base"]["both_ms"]["median"] / entry["new"]["both_ms"]["median"], 3)
        entry["speedup_decode"] = round(entry["base"]["decode_ms"]["median"] / entry["new"]["decode_ms"]["median"], 3)
        entry["max_abs_diff"] = (base_out[B] - new_out[B]).abs().max().item()
        res[f"B{B}"] = entry
    print(json.dumps(res))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=None, help="old vs fused: one size (default 32); "
                    "--base-lib: one or more (default 32 8)")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=None, help="calls per round (default 50; --base-lib: 30)")
    ap.add_argument("--base-lib", help="compare the fused decoder of this build of libnlam_b200.so against the tree's")
    ap.add_argument("--worker", help=argparse.SUPPRESS)
    ap.add_argument("--out", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        worker(args.worker, args.batch, args.iters, args.out)
        return
    if args.base_lib:
        args.batch = args.batch or [32, 8]
        args.iters = args.iters or 30
        compare_libs(args)
        return
    assert args.batch is None or len(args.batch) == 1, "old vs fused: one batch size"
    B = args.batch[0] if args.batch else 32
    args.iters = args.iters or 50
    sys.path.insert(0, ROOT)
    import torch
    from neural_lam_b200 import ops

    m, net, out_map, mesh, grid, m2g, prev, bnd, mask = setup(B)
    G = m.num_grid_nodes
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
