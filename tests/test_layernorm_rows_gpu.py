"""LayerNorm on rows whose mean is large against their spread, in every kernel that normalises rows (`-m gpu`).

Every make_mlp in the model ends in Linear -> LayerNorm.  A last Linear whose bias has a common offset across its columns
gives LayerNorm rows with |mu| >> sigma; statistics taken in one pass (E[x²] − mu²) cancel there and x̂ goes wrong by up
to 1 / sqrt(eps).  These cases build that regime on purpose and hold every kernel to the bounds of DESIGN.md §2.

The regime: the call runs once through the fp64 oracle, which records the LayerNorm input rows of each MLP; the MLP under
test then gets c = ratio x sigma_hat − median(mu) added to its last bias, sigma_hat and mu the median row std and the row
means of those rows.  The offset sits in the bias, which both this code and the reference add in fp32 after the GEMM, so
the reference's TF32 configuration stays accurate and its error stays a fair yardstick.  The ratio reached is printed
(run with -s) and must be at least half the target.  Ratios 1 (control), 100, 1 000 and 10 000; near-constant rows
(mu ≈ 1, sigma ≈ 1e-3, sigma² well below eps); exactly constant rows (W2 = 0, b2 = c), whose output must be beta.

Bounds (DESIGN.md §2): max |got − fp64 oracle| <= 1e-2 and <= max(3 x the error of the reference's TF32 configuration,
4e-3) per call; gradients as test_backward_coverage_gpu._check; whole rollouts 2e-2 (test_decode_gpu).
"""
import contextlib

import pytest
import torch
import torch.nn.functional as F

import neural_lam_b200 as nlb
from neural_lam_b200 import _lib, backward, models, ops, synthetic
from neural_lam_b200.networks import make_mlp
from oracle import reference_port as rp
from test_backward_coverage_gpu import _check as _check_grad
from test_backward_coverage_gpu import _graph as _bwd_graph
from test_backward_coverage_gpu import _report, _run_checked
import test_decode_gpu as dec
import test_edge_path_gpu as edg
from test_efm_gpu import _latent_modules
from test_efm_gpu import _oracle as _latent_oracle
from test_models import _oracle_graph

pytestmark = pytest.mark.gpu
DEV = "cuda"
ABS_TOL = 1e-2
RATIOS = [1, 100, 1000, 10000]
KINDS = [f"ratio{r}" for r in RATIOS] + ["near_constant"]


# ------------------------------------------------------------------------------------------------ the regime
@contextlib.contextmanager
def _recording():
    """while active, rp.mlp records the fp64 LayerNorm input rows of every MLP it runs, by parameter prefix"""
    rec, orig = {}, rp.mlp

    def mlp(x, params, prefix, hidden_layers=1, layer_norm=True, eps=1e-5):
        if layer_norm:
            pre = orig(x, params, prefix, hidden_layers, layer_norm=False)
            rec.setdefault(prefix, []).append(pre.detach().reshape(-1, pre.shape[-1]).double().cpu())
        return orig(x, params, prefix, hidden_layers, layer_norm, eps)

    rp.mlp = mlp
    try:
        yield rec
    finally:
        rp.mlp = orig


def _rows(ref64, prefixes):
    """-> {prefix: the LayerNorm input rows of that MLP in one run of ``ref64``}"""
    with torch.no_grad(), _recording() as rec:
        ref64()
    missing = [p for p in prefixes if p not in rec]
    assert not missing, f"the oracle runs no LayerNorm MLP {missing} ({sorted(rec)})"
    return {p: torch.cat(rec[p]) for p in prefixes}


def _stats(rows):
    mu, sd = rows.mean(-1), rows.std(-1, unbiased=False)
    return mu, sd


def _make_regime(ref64, mods, kind):
    """offset the last Linear of every MLP in ``mods`` (oracle prefix -> make_mlp) for ``kind``; the rows are those of
    ``ref64`` (the call's fp64 oracle).  The LayerNorm output does not depend on the offset, so one MLP's offset leaves the
    rows of the others as they were."""
    rows = _rows(ref64, mods)
    with torch.no_grad():
        for p, m in mods.items():
            lin = m[-2]
            mu, sd = _stats(rows[p])
            s_hat = sd.median().item()
            if kind == "near_constant":  # sigma -> 1e-3, mu -> 1
                scale = 1e-3 / s_hat
                lin.weight.mul_(scale)
                lin.bias.mul_(scale)
                lin.bias.add_(1.0 - mu.median().item() * scale)
            elif kind.startswith("constant"):
                lin.weight.zero_()
                lin.bias.fill_(float(kind[len("constant"):]))
            else:
                ratio = float(kind[len("ratio"):])
                lin.bias.add_(ratio * s_hat - mu.median().item())
    rows = _rows(ref64, mods)
    for p in mods:
        mu, sd = _stats(rows[p])
        if kind.startswith("ratio"):
            ratio = float(kind[len("ratio"):])
            reached = (mu.abs() / sd).median().item()
            print(f"\n  {p}: median |mu| / sigma {reached:.4g} (target {ratio:g})", end="")
            assert reached >= ratio / 2, (p, reached, ratio)
        elif kind == "near_constant":
            print(f"\n  {p}: median mu {mu.median().item():.4g}, median sigma {sd.median().item():.3g}", end="")
            assert abs(mu.median().item() - 1) < 0.1 and sd.median().item() < 2e-3, (p, mu.median(), sd.median())
        else:
            assert sd.max().item() == 0, (p, sd.max().item())


def _params(dtype, dev, **roots):
    """oracle parameters of modules under their prefixes ("_" : no prefix)"""
    out = {}
    for root, mod in roots.items():
        for k, v in mod.state_dict().items():
            out[k if root == "_" else f"{root}.{k}"] = v.detach().to(dev, dtype)
    return out


def _tuple(x):
    return x if isinstance(x, (tuple, list)) else (x,)


def _check_call(name, run, ref, labels):
    """run -> (outputs, launch names); ref(dtype, device) -> outputs of the oracle.  -> max |err|"""
    with torch.no_grad():
        got, names = run()
    for lab in labels:  # a label, or the prefix of templated ones (tc_linear_kernel<N>)
        assert any(n == lab or n.startswith(lab + "<") for n in names), f"{name}: {lab} did not run ({names})"
    got = [g.detach().double().cpu() for g in _tuple(got)]
    with torch.no_grad():
        want = [w.double().cpu() for w in _tuple(ref(torch.float64, "cpu"))]
        with rp.tf32_matmul(mode="rna"):
            ref32 = [w.double().cpu() for w in _tuple(ref(torch.float32, DEV))]
    assert len(got) == len(want)
    for g in got:
        assert torch.isfinite(g).all(), f"{name}: non-finite output"
    err = max((g.reshape(w.shape) - w).abs().max().item() for g, w in zip(got, want))
    ref_err = max((r - w).abs().max().item() for r, w in zip(ref32, want))
    print(f"\n{name} ({', '.join(labels)}): max |err| vs fp64 oracle {err:.3e} "
          f"(reference TF32 configuration {ref_err:.3e})")
    assert err <= ABS_TOL, f"{name}: max |err| {err:.3e} > {ABS_TOL}"
    assert err <= max(3 * ref_err, 4e-3), f"{name}: max |err| {err:.3e} > max(3 x {ref_err:.3e}, 4e-3)"
    return err


def _bias_noise(module, seed):
    gen = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p in module.parameters():
            if p.dim() == 1:
                p.add_(0.1 * torch.randn(p.shape, generator=gen).to(p.device))
    return module


# ------------------------------------------------------------------------------------------------ row MLPs
ROW_MLPS = {
    # name: (source widths, B, rows); a width w < 0: a (rows, -w) source shared by the batch
    "mlp_64": ([64], 2, 3000),
    "grid_embedder_17_17_18_4": ([17, 17, 18, -4], 2, 3000),  # the grid embedder's sources: state, state, forcing, static
}
ROW_PATHS = {"tc": (_lib.MATH_TF32, "tc_rowmlp_kernel"), "simt": (_lib.MATH_FP32, "rowmlp_simt_kernel")}


def _rowmlp_case(widths, B, n, flags, seed=0):
    torch.manual_seed(seed)
    m = _bias_noise(make_mlp([sum(abs(w) for w in widths), 64, 64]), seed + 1).to(DEV)
    gen = torch.Generator().manual_seed(seed + 2)
    xs = [torch.randn(B, n, w, generator=gen) if w > 0 else torch.randn(n, -w, generator=gen) for w in widths]

    def run():
        with ops.profile_launches() as prof:
            out = ops.rowmlp(m, [x.to(DEV) for x in xs], flags=flags)
        return out, prof.names()

    def ref(dtype, dev):
        x = torch.cat([(x if x.dim() == 3 else x.expand(B, -1, -1)).to(dev, dtype) for x in xs], -1)
        return rp.mlp(x, _params(dtype, dev, m=m), "m")

    return m, run, ref


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("path", list(ROW_PATHS))
@pytest.mark.parametrize("mlp", list(ROW_MLPS))
def test_rowmlp(mlp, path, kind):
    """ops.rowmlp on the H = 64 row kernel (fused_mlp_kernel) and on the exact fp32 kernel (two-pass statistics: the
    control)"""
    widths, B, n = ROW_MLPS[mlp]
    flags, label = ROW_PATHS[path]
    m, run, ref = _rowmlp_case(widths, B, n, flags)
    _make_regime(lambda: ref(torch.float64, "cpu"), {"m": m}, kind)
    _check_call(f"{mlp} {path} {kind}", run, ref, [label])


CONSTANT_PATHS = {
    "tc_rowmlp": ([64, 64, 64], _lib.MATH_TF32, "tc_rowmlp_kernel"),
    "simt": ([64, 64, 64], _lib.MATH_FP32, "rowmlp_simt_kernel"),
    "tc_linear_128": ([128, 128, 128], None, "tc_linear_kernel<128>"),
    "tc_linear_256": ([256, 256, 256], None, "tc_linear_kernel<256>"),
}


@pytest.mark.parametrize("c", [0.1, 3.7])
@pytest.mark.parametrize("path", list(CONSTANT_PATHS))
def test_constant_rows_give_beta(path, c):
    """W2 = 0, b2 = c: every LayerNorm row is exactly constant; the output is beta (finite, within 1e-4)"""
    bp, flags, label = CONSTANT_PATHS[path]
    torch.manual_seed(5)
    m = _bias_noise(make_mlp(bp), 6)
    with torch.no_grad():
        m[-2].weight.zero_()
        m[-2].bias.fill_(c)
    m = m.to(DEV)
    x = torch.randn(2, 1000, bp[0], device=DEV)
    with torch.no_grad(), ops.profile_launches() as prof:
        if flags is None:
            m.nlam_flags = _lib.MATH_TF32
            out = m.apply_rows([x])
        else:
            out = ops.rowmlp(m, [x], flags=flags)
    assert label in prof.names(), prof.names()
    assert torch.isfinite(out).all()
    err = (out.double() - m[-1].bias.double()).abs().max().item()
    print(f"\n{path} c={c}: max |out - beta| {err:.3e}")
    assert err <= 1e-4, err


# ------------------------------------------------------------------------------------------------ H = 64 edge paths
EDGE_CASES = {  # test_edge_path_gpu.CASES row -> the split-form / K = 192 label it selects
    "below_threshold_b1": "tc_edge_kernel",
    "mesh_out_of_place_b3": "tc_edge3_kernel",
    "mesh_inplace_b3": "tc_edge_rmw_kernel",
    "g2m_b3": "tc_edge_bcast_kernel",
    "ell_b2": "tc_ell_window_kernel",
}


def _edge_case(row):
    case = next(c for c in edg.CASES if c[0] == row)
    name, (kind, ns, nr, m_), B, same, shared, upd, inplace = case[:7]
    g = edg._graph(case)
    ei = edg._uniform_graph(ns, nr, m_, 1) if kind == "uniform" else edg._random_graph(ns, nr, m_, 1)
    edge_mlp, aggr_mlp = edg._mlps(0)
    _bias_noise(edge_mlp, 1)
    _bias_noise(aggr_mlp, 2)
    send, rec, edge = edg._tensors(case)

    def run():
        e = edge.clone() if inplace else edge  # the in-place call overwrites its edge input
        with ops.profile_launches() as prof:
            out = ops.inet_fwd(g, edge_mlp, aggr_mlp, send, rec, e, upd, 0, edge_inplace=inplace)
        return (out[0], out[1]) if upd else out[0], prof.names()

    def ref(dtype, dev):
        t = [x.to(dev, dtype) for x in (send, rec, edge)]
        return rp.interaction_net(_params(dtype, dev, edge_mlp=edge_mlp, aggr_mlp=aggr_mlp), ei.to(dev), *t,
                                  update_edges=upd)

    return {"edge_mlp": edge_mlp, "aggr_mlp": aggr_mlp}, run, ref


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("which", ["edge_mlp", "aggr_mlp"])
@pytest.mark.parametrize("row", list(EDGE_CASES))
def test_edge_paths(row, which, kind):
    """the edge MLP (fused_mlp_kernel at K = 192, tc_edge_split_kernel otherwise) and the node update (tc_node_kernel)
    of one InteractionNet call, one of the two offset at a time; in place (tc_edge_rmw_kernel) and out of place"""
    mods, run, ref = _edge_case(row)
    _make_regime(lambda: ref(torch.float64, "cpu"), {which: mods[which]}, kind)
    _check_call(f"{row} {which} {kind}", run, ref, [EDGE_CASES[row], "tc_rowmlp_kernel"])


# ------------------------------------------------------------------------------------------------ H = 64 node kernel
def _node_tensors(N, B, D=17, seed=11):
    gen = torch.Generator().manual_seed(seed)
    rec, aggr, prev, bnd = (torch.randn(B, N, d, generator=gen) for d in (64, 64, D, D))
    std, mean = torch.rand(D, generator=gen) + 0.5, torch.randn(D, generator=gen)
    mask = (torch.rand(N, 1, generator=gen) < 0.3).float()
    return rec, aggr, prev, bnd, std, mean, mask


def _node_out_case():
    N, B = 64 * 50 + 33, 3
    torch.manual_seed(9)
    node = _bias_noise(make_mlp([128, 64, 64]), 9).to(DEV)
    out_map = _bias_noise(make_mlp([64, 64, 17], layer_norm=False), 10).to(DEV)
    t = _node_tensors(N, B)

    def run():
        d = [x.to(DEV) for x in t]
        with ops.profile_launches() as prof:
            out = ops.node_update_step(node, out_map, d[0], d[1], d[2], d[3], d[6], d[4], d[5])
        return out, prof.names()

    def ref(dtype, dev):
        rec, aggr, prev, bnd, std, mean, mask = (x.to(dev, dtype) for x in t)
        p = _params(dtype, dev, n=node, o=out_map)
        grid = rec + rp.mlp(torch.cat([rec, aggr], -1), p, "n")
        step = prev + rp.mlp(grid, p, "o", layer_norm=False) * std + mean
        return mask * bnd + (1 - mask) * step

    return {"n": node}, run, ref, ["tc_node_out_kernel"]


def _node_rowmlp_case():
    N, B = 64 * 50 + 33, 3
    torch.manual_seed(12)
    node = _bias_noise(make_mlp([128, 64, 64]), 12).to(DEV)
    rec, aggr = _node_tensors(N, B)[:2]

    def run():
        r, a = rec.to(DEV), aggr.to(DEV)
        with ops.profile_launches() as prof:
            out = ops.rowmlp(node, [r, a], res=r, flags=_lib.MATH_TF32)
        return out, prof.names()

    def ref(dtype, dev):
        r, a = rec.to(dev, dtype), aggr.to(dev, dtype)
        return r + rp.mlp(torch.cat([r, a], -1), _params(dtype, dev, n=node), "n")

    return {"n": node}, run, ref, ["tc_rowmlp_kernel"]


def _node_proj_case():
    N, B = 64 * 20 + 17, 3
    gen = torch.Generator().manual_seed(5)
    ei = torch.stack([torch.randint(0, N, (6 * N,), generator=gen), torch.randint(0, N, (6 * N,), generator=gen)])
    ei[1, -1] = N - 1
    ei = ei[:, torch.sort(ei[1], stable=True).indices]
    torch.manual_seed(6)
    l1 = _bias_noise(nlb.InteractionNet(ei, 64, math="tf32"), 6).to(DEV)
    l2 = _bias_noise(nlb.InteractionNet(ei, 64, math="tf32"), 7).to(DEV)
    x, e = torch.randn(B, N, 64, generator=gen), torch.randn(B, 6 * N, 64, generator=gen)
    g = l1._graph(torch.device(DEV, torch.cuda.current_device()))

    def run():
        xd = x.to(DEV)
        with ops.profile_launches() as prof:
            rec, e1, _, proj = ops.inet_fwd(g, l1.edge_mlp, l1.aggr_mlp, xd, xd, e.to(DEV), True, l1._flags(),
                                            next_edge_seq=l2.edge_mlp)
        return (rec, e1, proj[0], proj[1]), prof.names()

    def ref(dtype, dev):
        p = _params(dtype, dev, l1=l1)
        x_ = x.to(dev, dtype)
        r1, e1 = rp.interaction_net(p, ei.to(dev), x_, x_, e.to(dev, dtype), prefix="l1")
        w, b1 = l2.edge_mlp[0].weight.detach().to(dev, dtype), l2.edge_mlp[0].bias.detach().to(dev, dtype)
        return r1, e1, r1 @ w[:, 64:128].T, r1 @ w[:, 128:].T + b1

    return {"l1.aggr_mlp": l1.aggr_mlp}, run, ref, ["tc_node_proj_kernel"]


NODE_CASES = {"node_update": _node_rowmlp_case, "node_proj": _node_proj_case, "node_out": _node_out_case}


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("case", list(NODE_CASES))
def test_node_kernel(case, kind):
    mods, run, ref, labels = NODE_CASES[case]()
    _make_regime(lambda: ref(torch.float64, "cpu"), mods, kind)
    _check_call(f"{case} {kind}", run, ref, labels)


# ------------------------------------------------------------------------------------------------ decoder
def _decode_case(std_out):
    d = dec.D
    c = dec._setup(dec._ell_graph(200, 1000, 4, 2), 200, 1000, 3, d_out=2 * d if std_out else d)
    if std_out:  # the state takes the first d outputs; prev, boundary keep d columns
        c["prev"], c["bnd"] = torch.randn(3, 1000, d), torch.randn(3, 1000, d)
        c["std"], c["mean"] = c["std"][:d], c["mean"][:d]

    def run():
        net, out_map, g = dec._on_gpu(c)
        so = torch.empty(3, 1000, d, device=DEV) if std_out else None
        with ops.profile_launches() as prof:
            got = net.decode_step(g["send"], g["rec"], g["edge"], out_map, g["prev"], g["bnd"], g["mask"], g["std"], g["mean"],
                                  std_out=so)
        return ((got, so) if std_out else got), prof.names()

    def ref(dtype, dev):
        if not std_out:
            return dec._oracle(c, dev, dtype)
        pn = _params(dtype, dev, _=c["net"])
        po = _params(dtype, dev, m=c["out_map"])
        t = {k: c[k].to(dev, dtype) for k in ("send", "rec", "edge", "prev", "std", "mean", "bnd")}
        grid = rp.interaction_net(pn, c["ei"].to(dev), t["send"], t["rec"], t["edge"].expand(3, -1, -1), update_edges=False)
        y = rp.mlp(grid, po, "m", layer_norm=False)
        new = t["prev"] + y[..., :d] * t["std"] + t["mean"]
        mk = c["mask"].to(dev, dtype)[None, :, None]
        return mk * t["bnd"] + (1 - mk) * new, F.softplus(y[..., d:])

    return {"edge_mlp": c["net"].edge_mlp, "aggr_mlp": c["net"].aggr_mlp}, run, ref


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("which", ["edge_mlp", "aggr_mlp"])
@pytest.mark.parametrize("std_out", [False, True], ids=["state", "state_and_std"])
def test_decode(std_out, which, kind):
    """tc_decode_kernel's edge LayerNorm and node LayerNorm, one offset at a time"""
    mods, run, ref = _decode_case(std_out)
    _make_regime(lambda: ref(torch.float64, "cpu"), {which: mods[which]}, kind)
    _check_call(f"decode {'std ' if std_out else ''}{which} {kind}", run, ref, dec.DECODER)


# ------------------------------------------------------------------------------------------------ encoder
def _encode_case():
    spec = synthetic.make_graph_spec(31, 26, hierarchical=False)
    ds = synthetic.SyntheticDatastore(spec, d_state=17, d_forcing=18, d_static=4, boundary_width=2)
    torch.manual_seed(3)
    m = models.GraphLAM(ds, spec, hidden_dim=64, processor_layers=1)
    for mod in (m.grid_embedder, m.encoding_grid_mlp):
        _bias_noise(mod, 4)
    m = m.to(DEV).eval()
    G, B = m.num_grid_nodes, 2
    f = m.grid_input_dim - 2 * 17 - 4
    gen = torch.Generator().manual_seed(8)
    prev, pprev, forc = (torch.randn(B, G, d, generator=gen) for d in (17, 17, f))
    static = m.grid_static_features.detach().cpu()

    def run():
        with torch.no_grad():
            st = m.static_embeddings()
            mesh, g2m = m.expand_to_batch(st["mesh_emb"], B), m.expand_to_batch(st["g2m_emb"], B)
            srcs = [prev.to(DEV), pprev.to(DEV), forc.to(DEV), m.expand_to_batch(m.grid_static_features, B)]
            with ops.profile_launches() as prof:
                grid_rep, _, _ = m.g2m_gnn.encode_step(m.grid_embedder, m.encoding_grid_mlp, srcs, mesh, g2m)
        return grid_rep, prof.names()

    def ref(dtype, dev):
        p = _params(dtype, dev, grid_embedder=m.grid_embedder, encoding_grid_mlp=m.encoding_grid_mlp)
        x = torch.cat([prev.to(dev, dtype), pprev.to(dev, dtype), forc.to(dev, dtype),
                       static.to(dev, dtype).expand(B, -1, -1)], -1)
        emb = rp.mlp(x, p, "grid_embedder")
        return emb + rp.mlp(emb, p, "encoding_grid_mlp")

    return {"grid_embedder": m.grid_embedder, "encoding_grid_mlp": m.encoding_grid_mlp}, run, ref


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("which", ["grid_embedder", "encoding_grid_mlp"])
def test_encode(which, kind):
    """tc_encode_kernel's two LayerNorms (grid embedder, encoding grid MLP), one offset at a time"""
    mods, run, ref = _encode_case()
    _make_regime(lambda: ref(torch.float64, "cpu"), {which: mods[which]}, kind)
    _check_call(f"encode {which} {kind}", run, ref, ["tc_encode_kernel"])


# ------------------------------------------------------------------------------------------------ latent step
@pytest.mark.parametrize("kind", KINDS)
def test_latent(kind):
    """tc_latent_kernel's latent_embedder LayerNorm (diagonal Gaussian)"""
    pm, em = _latent_modules(True, seed=4)
    gen = torch.Generator().manual_seed(4)
    x, eps = torch.randn(3, 64 * 30 + 9, 64, generator=gen), torch.randn(3, 64 * 30 + 9, 64, generator=gen)

    def run():
        with ops.profile_launches() as prof:
            out = ops.latent_sample(pm, em, x.to(DEV), eps.to(DEV))
        return out, prof.names()

    def ref(dtype, dev):
        return _latent_oracle(pm, em, x.to(DEV), eps.to(DEV), True, dtype=dtype, tf32=rp._TF32 is not None)

    _make_regime(lambda: ref(torch.float64, "cpu"), {"e": em}, kind)
    _check_call(f"latent {kind}", run, ref, ["tc_latent_kernel"])


# ------------------------------------------------------------------------------------------------ generic Linear
LINEAR_LAYERS = {
    # name: (class, H)
    "inet_h128": ("InteractionNet", 128),
    "inet_h256": ("InteractionNet", 256),
    "prop_h64": ("PropagationNet", 64),
}


def _layer_case(cls, H, B=2, math="tf32"):
    gen = torch.Generator().manual_seed(H)
    ns, nr, ne = 300, 200, 1500
    ei = torch.stack([torch.randint(0, ns, (ne,), generator=gen), torch.randint(0, nr, (ne,), generator=gen)])
    ei[1, -1] = nr - 1
    torch.manual_seed(H + 1)
    net = _bias_noise(getattr(nlb, cls)(ei, H, math=math), H + 2)
    send, rec, edge = (torch.randn(B, n, H, generator=gen) for n in (ns, nr, ne))
    prop = cls == "PropagationNet"

    def ref(dtype, dev, s=send, r=rec, e=edge):
        return rp.interaction_net(_params(dtype, dev, _=net), ei.to(dev), s.to(dev, dtype), r.to(dev, dtype),
                                  e.to(dev, dtype), propagation=prop)

    return net, (send, rec, edge), ref


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("which", ["edge_mlp", "aggr_mlp"])
@pytest.mark.parametrize("layer", list(LINEAR_LAYERS))
def test_generic_linear(layer, which, kind):
    """the LayerNorm epilogue of tc_linear_kernel<N> (H = 128, 256; PropagationNet at H = 64)"""
    net, xs, ref = _layer_case(*LINEAR_LAYERS[layer])
    _make_regime(lambda: ref(torch.float64, "cpu"), {which: getattr(net, which)}, kind)
    net = net.to(DEV)

    def run():
        with ops.profile_launches() as prof:
            out = net(*(x.to(DEV) for x in xs))
        return out, prof.names()

    _check_call(f"{layer} {which} {kind}", run, ref, ["tc_linear_kernel"])


# ------------------------------------------------------------------------------------------------ ln_fwd / ln_bwd
@pytest.mark.parametrize("ratio", [1, 1000, "near_constant"])
@pytest.mark.parametrize("H", [64, 128, 256])
def test_layernorm_fwd_bwd_direct(H, ratio):
    """backward.layernorm_fwd / layernorm_bwd (ln_fwd_kernel, ln_bwd_kernel) on rows with a large mean: forward within
    1e-2 of fp64, gradients within test_backward_coverage_gpu._check's bound of fp64 autograd"""
    gen = torch.Generator(device=DEV).manual_seed(H)
    eps, rows = 1e-5, 5000
    if ratio == "near_constant":
        y = 1 + 1e-3 * torch.randn(rows, H, device=DEV, generator=gen)
    else:
        y = ratio * (1 + 0.2 * torch.rand(rows, 1, device=DEV, generator=gen)) + torch.randn(rows, H, device=DEV, generator=gen)
    gamma = 1 + 0.1 * torch.randn(H, device=DEV, generator=gen)
    beta = 0.1 * torch.randn(H, device=DEV, generator=gen)
    g = torch.randn(rows, H, device=DEV, generator=gen)
    y64, gm64, b64 = (t.double().requires_grad_(True) for t in (y, gamma, beta))
    want = F.layer_norm(y64, (H,), gm64, b64, eps)
    want.backward(g.double())
    with ops.profile_launches() as prof:
        out = backward.layernorm_fwd(y, gamma, beta, eps)
        gy, dg, db = backward.layernorm_bwd(g, y, gamma, eps)
    assert "ln_fwd_kernel" in prof.names() and "ln_bwd_kernel" in prof.names(), prof.names()
    err = (out.double() - want.detach()).abs().max().item()
    print(f"\nln H={H} {ratio}: max |fwd err| {err:.3e}")
    assert torch.isfinite(out).all() and err <= ABS_TOL, err
    errs = {"g_y": _check_grad("g_y", gy, y64.grad), "dgamma": _check_grad("dgamma", dg, gm64.grad),
            "dbeta": _check_grad("dbeta", db, b64.grad)}
    _report(f"ln H={H} {ratio}", errs)


# ------------------------------------------------------------------------------------------------ gradients
@pytest.mark.parametrize("H", [64, 128])
def test_layer_gradients_offset_rows(H):
    """one InteractionNet call with both MLPs offset to ratio 1 000: its forward within the per-call bound, and every
    parameter and input gradient within test_backward_coverage_gpu._check's bound of fp64 autograd through the oracle —
    the backward recomputes the forward with two-pass statistics, so forward and backward must agree on the function"""
    B = 2
    ei, ns, nr = _bwd_graph("random", torch.Generator().manual_seed(11))
    torch.manual_seed(0)
    net = _bias_noise(nlb.InteractionNet(ei, H, math="auto"), 1)
    E = ei.shape[1]
    gen = torch.Generator().manual_seed(12)
    send, rec, edge = (torch.randn(B, n, H, generator=gen) for n in (ns, nr, E))
    w_rec, w_edge = torch.randn(B, nr, H, generator=gen), torch.randn(B, E, H, generator=gen)

    def ref(dtype, dev, s=send, r=rec, e=edge, p=None):
        p = p if p is not None else _params(dtype, dev, _=net)
        return rp.interaction_net(p, ei.to(dev), s.to(dev, dtype), r.to(dev, dtype), e.to(dev, dtype))

    _make_regime(lambda: ref(torch.float64, "cpu"), {"edge_mlp": net.edge_mlp, "aggr_mlp": net.aggr_mlp}, "ratio1000")
    p64 = {k: v.detach().to(DEV).double().requires_grad_(True) for k, v in net.state_dict().items()}
    x64 = [t.to(DEV).double().requires_grad_(True) for t in (send, rec, edge)]
    r64, e64 = ref(torch.float64, DEV, *x64, p=p64)
    ((r64 * w_rec.to(DEV).double()).sum() + (e64 * w_edge.to(DEV).double()).sum()).backward()
    net = net.to(DEV)
    xd = [t.to(DEV).requires_grad_(True) for t in (send, rec, edge)]
    out = {}

    def step():
        r, e = net(*xd)
        out["fwd"] = (r.detach(), e.detach())
        ((r * w_rec.to(DEV)).sum() + (e * w_edge.to(DEV)).sum()).backward()

    _run_checked(step, need=("ln_bwd_kernel", "transpose_pad_kernel"))
    err = max((o.double() - w.detach()).abs().max().item() for o, w in zip(out["fwd"], (r64, e64)))
    print(f"\nH={H} forward with grad: max |err| vs fp64 oracle {err:.3e}")
    assert err <= ABS_TOL, err
    errs = {f"g_{k}": _check_grad(f"g_{k}", t.grad, t64.grad) for k, t, t64 in zip(("send", "rec", "edge"), xd, x64)}
    for k, p in net.named_parameters():
        errs[k] = _check_grad(k, p.grad, p64[k].grad)
    _report(f"InteractionNet H={H} ratio 1000", errs)


# ------------------------------------------------------------------------------------------------ whole models
def _ln_mlps(model):
    """every make_mlp of the model that ends in a LayerNorm, under its oracle prefix"""
    return {f"predictor.{n}": m for n, m in model.named_modules()
            if isinstance(m, torch.nn.Sequential) and len(m) >= 2 and isinstance(m[-1], torch.nn.LayerNorm)}


@pytest.mark.parametrize("kind", ["graph_lam", "hi_lam"])
def test_model_rollout_offset_rows(kind):
    """GraphLAM (multiscale) and a 3-level HiLAM, H = 64, with every LayerNorm MLP offset to ratio 1 000: the eager and the
    CUDA-graph rollout of 2 steps within 2e-2 of the fp64 oracle"""
    spec = synthetic.make_graph_spec(30, 27, hierarchical=kind == "hi_lam")
    ds = synthetic.SyntheticDatastore(spec, d_state=5, d_forcing=6, d_static=1, boundary_width=2)
    torch.manual_seed(1)
    m = (models.HiLAM if kind == "hi_lam" else models.GraphLAM)(ds, spec, hidden_dim=64, processor_layers=2)
    fc = models.ARForecaster(m, ds)
    _bias_noise(m, 2)
    g = _oracle_graph(m, fc)
    cfg = dict(model=kind, hidden_layers=1, processor_layers=2, mesh_aggr="sum")
    G, B, T = m.num_grid_nodes, 2, 2
    gen = torch.Generator().manual_seed(5)
    init, forc, bnd = torch.randn(B, 2, G, 5, generator=gen), torch.randn(B, T, G, 6, generator=gen), torch.randn(B, T, G, 5,
                                                                                                               generator=gen)

    def ref64():
        params = {f"predictor.{k}": v.detach().double() for k, v in m.state_dict().items()}
        return rp.ar_rollout(params, g, cfg, init.double(), forc.double(), bnd.double())

    mods = _ln_mlps(m)
    assert len(mods) >= 8, sorted(mods)
    _make_regime(ref64, mods, "ratio1000")
    want = ref64()
    fc = fc.to(DEV).eval()
    with torch.no_grad(), ops.profile_launches() as prof:
        got, _ = fc(init.to(DEV), forc.to(DEV), bnd.to(DEV))
    with torch.no_grad():
        graphed = fc.rollout_graphed(init.to(DEV), forc.to(DEV), bnd.to(DEV))
    names = prof.names()
    if kind == "graph_lam":
        assert names.count("tc_decode_kernel") == T, names
    for name, out in (("eager", got), ("graphed", graphed)):
        assert torch.isfinite(out).all(), name
        err = (out.double().cpu() - want).abs().max().item()
        print(f"\n{kind} {name}, {len(mods)} LayerNorm MLPs at ratio 1000: max |err| vs fp64 oracle {err:.3e}")
        assert err < 2e-2, (name, err)
