"""Time the H = 64 node-update launches of a forecast step at bench.py config 2 size (MEPS 268x238 grid, GraphLAM H = 64,
four processor layers) with two builds of the library, alternating them, and check that their outputs agree.

Launches (each timed from the library's per-launch profile, CUDA events around the kernel):
  g2m_node    grid -> mesh node update, rec = the static mesh embedding shared by the batch   (tc_rowmlp_kernel)
  m2m_proj    m2m layers 1-3: node update + the next layer's node projections                  (tc_node_proj_kernel)
  m2m_last    m2m layer 4: node update                                                         (tc_rowmlp_kernel)
  node_out    mesh -> grid node update + output_map + step epilogue (the decoder's second rung,
              not part of config 2's step)                                                     (tc_node_out_kernel)
The step runs g2m_node once, m2m_proj three times and m2m_last once: `step_sum_*` adds them up that way.

Each round runs one subprocess per library (`_lib.LIB_PATH` set before the library loads), in alternating order, on the
same seeded inputs; a worker times ITERS calls of each launch and takes their median.  Prints one JSON line: per batch
size and launch, the median, min and max over the rounds in µs, the algorithmic GB/s of the median and its share of the
data sheet's 3.35 TB/s, and the maximum |difference| of every output between the two libraries; plus the card's name,
power limit and SM clock.

    python scripts/bench_node.py --base-lib PATH [--rounds 7] [--iters 30] [--batch 32 8]

PATH is another build of libnlam_b200.so (for example the parent commit's, built into a directory git ignores).
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
LAUNCHES = {"g2m_node": "tc_rowmlp_kernel", "m2m_proj": "tc_node_proj_kernel", "m2m_last": "tc_rowmlp_kernel",
            "node_out": "tc_node_out_kernel"}
PER_STEP = {"g2m_node": 1, "m2m_proj": 3, "m2m_last": 1}


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def worker(lib_path, batches, iters, out_path, dump):
    sys.path.insert(0, ROOT)
    from neural_lam_b200 import _lib
    _lib.LIB_PATH = lib_path
    import torch
    from neural_lam_b200 import models, ops, synthetic

    assert torch.cuda.is_available(), "bench_node.py needs a CUDA device"
    dev = torch.device("cuda")
    spec = synthetic.make_graph_spec(268, 238, hierarchical=False)
    ds = synthetic.SyntheticDatastore(spec, d_state=17, d_forcing=18, d_static=4, boundary_width=10)
    torch.manual_seed(0)
    m = models.GraphLAM(ds, spec, hidden_dim=64, processor_layers=4).to(dev).eval()
    with torch.no_grad():
        st = m.static_embeddings()
    G = m.num_grid_nodes
    g2m, m2g, layers = m.g2m_gnn, m.m2g_gnn, [m.processor[i] for i in range(len(m.processor))]
    gg, gm = g2m._graph(dev), layers[0]._graph(dev)
    res, outs = {}, {}
    for B in batches:
        gen = torch.Generator(device=dev).manual_seed(1)
        grid = torch.randn(B, G, 64, device=dev, generator=gen)
        x = torch.randn(B, gm.n_rec, 64, device=dev, generator=gen)
        aggr_g = torch.randn(B, G, 64, device=dev, generator=gen)
        prev = torch.randn(B, G, m.diff_std.numel(), device=dev, generator=gen)
        mesh, g2m_e = m.expand_to_batch(st["mesh_emb"], B), m.expand_to_batch(st["g2m_emb"], B)
        m2m_e = m.expand_to_batch(st["m2m_emb"], B)
        with torch.no_grad():
            e_dense = ops.inet_fwd(gm, layers[0].edge_mlp, layers[0].aggr_mlp, x, x, m2m_e, True, layers[0]._flags())[1]
        calls = {
            "g2m_node": lambda: ops.inet_fwd(gg, g2m.edge_mlp, g2m.aggr_mlp, grid, mesh, g2m_e, False, g2m._flags()),
            "m2m_proj": lambda: ops.inet_fwd(gm, layers[0].edge_mlp, layers[0].aggr_mlp, x, x, m2m_e, True, layers[0]._flags(),
                                             next_edge_seq=layers[1].edge_mlp),
            "m2m_last": lambda: ops.inet_fwd(gm, layers[3].edge_mlp, layers[3].aggr_mlp, x, x, e_dense, False, layers[3]._flags()),
            "node_out": lambda: (ops.node_update_step(m2g.aggr_mlp, m.output_map, grid, aggr_g, prev, None, None, m.diff_std,
                                                      m.diff_mean, flags=m.output_map.nlam_flags),),
        }
        with torch.no_grad():
            for name, fn in calls.items():
                if dump:  # outputs of one call on fresh inputs
                    got = fn()
                    assert got[0] is not None, name
                    outs[f"{B}/{name}/out"] = got[0].cpu()
                    if len(got) == 4:
                        outs[f"{B}/{name}/proj"] = got[3].cpu()
                for _ in range(3):
                    fn()
                us, nbytes, labels = [], 0.0, set()
                with ops.profile_launches() as prof:
                    for _ in range(iters):
                        fn()
                for row in prof.rows:
                    if row[0] == LAUNCHES[name]:
                        us.append(row[1])
                        nbytes = row[2]
                    labels.add(row[0])
                assert len(us) == iters, (name, sorted(labels))
                res[f"{B}/{name}"] = {"us": statistics.median(us), "bytes": nbytes}
    if dump:
        torch.save(outs, out_path + ".pt")
    with open(out_path, "w") as f:
        json.dump(res, f)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base-lib", required=False, help="the library to compare against")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--batch", type=int, nargs="+", default=[32, 8])
    ap.add_argument("--worker", help=argparse.SUPPRESS)
    ap.add_argument("--out", help=argparse.SUPPRESS)
    ap.add_argument("--dump", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        worker(args.worker, args.batch, args.iters, args.out, args.dump)
        return
    new_lib = os.path.join(ROOT, "neural_lam_b200", "lib", "libnlam_b200.so")
    assert args.base_lib and os.path.isfile(args.base_lib), "--base-lib: path of the library to compare against"
    libs = {"base": os.path.abspath(args.base_lib), "new": new_lib}
    times = {k: {} for k in libs}
    with tempfile.TemporaryDirectory() as tmp:
        for r in range(args.rounds):
            for tag in (("base", "new") if r % 2 == 0 else ("new", "base")):
                out = os.path.join(tmp, f"{tag}_{r}.json")
                cmd = [sys.executable, os.path.abspath(__file__), "--worker", libs[tag], "--out", out, "--iters", str(args.iters),
                       "--batch", *map(str, args.batch)] + (["--dump"] if r == 0 else [])
                subprocess.run(cmd, check=True)
                with open(out) as f:
                    for key, v in json.load(f).items():
                        times[tag].setdefault(key, []).append(v)
        import torch
        base_out, new_out = torch.load(os.path.join(tmp, "base_0.json.pt")), torch.load(os.path.join(tmp, "new_0.json.pt"))
    res = {"gpu": gpu_info(), "rounds": args.rounds, "iters": args.iters, "launches": {}}
    for B in args.batch:
        tot = {t: {"median": 0.0, "min": 0.0, "max": 0.0} for t in libs}
        for name in LAUNCHES:
            key = f"{B}/{name}"
            entry = {"label": LAUNCHES[name]}
            for tag in libs:
                us = [v["us"] for v in times[tag][key]]
                med = statistics.median(us)
                gbs = times[tag][key][0]["bytes"] / (med * 1e3)
                k = PER_STEP.get(name, 0)
                tot[tag]["median"] += k * med
                tot[tag]["min"] += k * min(us)
                tot[tag]["max"] += k * max(us)
                entry[tag] = {"median_us": round(med, 1), "min_us": round(min(us), 1), "max_us": round(max(us), 1),
                              "gb_s": round(gbs, 1), "hbm_share": round(gbs / (HBM_TBS * 1e3), 3)}
            entry["speedup"] = round(entry["base"]["median_us"] / entry["new"]["median_us"], 3)
            for what in ("out", "proj"):
                k = f"{key}/{what}"
                if k in base_out:
                    entry[f"max_abs_diff_{what}"] = (base_out[k] - new_out[k]).abs().max().item()
            res["launches"][key] = entry
        # the step's five node launches; min / max: sums of the per-launch extremes (a bound on the range of the sum)
        res[f"step_sum_us_B{B}"] = {t: {k: round(v, 1) for k, v in d.items()} for t, d in tot.items()}
        res[f"step_sum_speedup_B{B}"] = round(tot["base"]["median"] / tot["new"]["median"], 3)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
