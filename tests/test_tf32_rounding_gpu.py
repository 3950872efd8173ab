"""TF32 operand rounding of every tensor-core path (wgmma ``.tf32``).

Each fp32 operand of a tensor-core GEMM must be rounded to TF32 (10 explicit mantissa bits) to nearest, ties away from
zero, before the MMA reads it: the reference's GPU configuration (``reference_port.tf32_matmul()``) does so, and an MMA
handed the raw fp32 bits truncates them, which biases every product toward zero by about 7e-4 relative.  Bounds of
4e-3 to 1e-2 on O(1) outputs do not see a scale error of that size, so these tests pin the rounding mode itself.

"Tailed" operands x = s (t - 0.375 ulp(t)), t in {3/8, 5/8, 3/4, 7/8}, ulp = the TF32 ulp of t: round-to-nearest gives
exactly s t, truncation s (t - ulp).

A. Bit-exact tests of the generic Linear (csrc/tc7.cu) through ``backward.linear`` / ``grad_input`` / ``grad_weight``.
   Every product of two t's is a multiple of 1/64 below 1, so every partial sum (up to 160 993 terms, plus biases and
   residuals that are multiples of 1/64) is exact in fp32 in any order: a kernel that rounds to nearest equals the fp64
   product of the s t BIT FOR BIT; a truncating one differs almost everywhere.
B. Every tensor-core forward path on tailed inputs and weights (weights scaled by 1/8, which keeps the tail) against two
   fp64 references, operands rounded to nearest (ref_rna) and truncated (ref_rz):
   ||got - ref_rna|| <= 0.6 ||got - ref_rz||, plus the absolute bound of test_tc_kernels.py.  The ratio is printed
   (run with -s); it also carries the error of the approximate SiLU.
C. Gaussian operands at production-like sizes: the least-squares slope s of got = (1 + s) ref (ref = the exact fp64
   product of the fp32 operands) is |s| <= 1e-4; truncation gives about -7e-4.
D. One GraphLAM training step (H = 64): the slope of every parameter gradient against fp64 autograd.
"""
import pytest
import torch

import neural_lam_b200 as nlb
from neural_lam_b200 import _lib, backward, models, ops, synthetic
from neural_lam_b200.networks import make_mlp
from oracle import reference_port as rp
from test_backward_coverage_gpu import GW_CASES, _run_checked, _split
from test_models import _oracle_graph

pytestmark = pytest.mark.gpu
DEV = "cuda"
ABS_TOL = 1e-2   # test_tc_kernels.py
RATIO = 0.6


# ------------------------------------------------------------------------------------------------ helpers
def _tailed(shape, gen, scale=1.0):
    """-> (x fp32, its TF32 round-to-nearest value s t scale in fp64), on the generator's device"""
    dev = gen.device
    t = torch.tensor([0.375, 0.625, 0.75, 0.875], dtype=torch.float64, device=dev)[
        torch.randint(0, 4, shape, generator=gen, device=dev)]
    ulp = torch.where(t < 0.5, 2.0 ** -12, 2.0 ** -11)
    s = torch.randint(0, 2, shape, generator=gen, device=dev).double() * 2 - 1
    return (s * (t - 0.375 * ulp) * scale).float(), s * t * scale


def _sixty_fourths(shape, gen, m):
    """exact multiples of 1/64 in [-m, m]"""
    return torch.randint(-64 * m, 64 * m + 1, shape, generator=gen, device=gen.device).float() / 64


def _assert_bit_exact(name, got, want):
    got = got.double()
    assert got.shape == want.shape, (name, got.shape, want.shape)
    bad = got != want
    if bad.any():
        err = (got - want).abs().nan_to_num(float("inf")).max().item()
        raise AssertionError(f"{name}: {int(bad.sum())} of {got.numel()} elements differ from the product of the "
                             f"TF32-rounded-to-nearest operands (max |err| {err:.3e})")


def _slope(got, ref):
    """least-squares s in got = (1 + s) ref"""
    got, ref = got.double().flatten(), ref.double().flatten()
    return ((got - ref) @ ref / (ref @ ref)).item()


# ------------------------------------------------------------------------------------------------ A. bit-exact
LIN_CASES = [
    # N, k0, k1, bias, residual
    (17, 32, 0, True, False),
    (17, 96, 64, True, False),
    (64, 64, 0, True, True),
    (64, 160, 96, False, True),
    (128, 4096, 0, True, True),
    (128, 128, 128, True, False),
    (256, 256, 32, True, True),
    (256, 1024, 0, False, False),
]


@pytest.mark.parametrize("N,k0,k1,bias,res", LIN_CASES,
                         ids=[f"N{n}_K{a}+{b}{'_bias' if c else ''}{'_res' if d else ''}" for n, a, b, c, d in LIN_CASES])
def test_linear_rounds_operands_to_nearest(N, k0, k1, bias, res):
    B, n = 2, 1000
    g = torch.Generator(device=DEV).manual_seed(N * 7919 + k0 + k1)
    x0, x0r = _tailed((B, n, k0), g)
    x1, x1r = _tailed((B, n, k1), g) if k1 else (None, None)
    w, wr = _tailed((N, k0 + k1), g)
    b = _sixty_fourths((N,), g, 1) if bias else None
    r = _sixty_fourths((B, n, N), g, 2) if res else None
    got = backward.linear(x0, w, N, x1=x1, bias=b, res=r)
    want = x0r @ wr[:, :k0].t()
    if k1:
        want = want + x1r @ wr[:, k0:].t()
    if bias:
        want = want + b.double()
    if res:
        want = want + r.double()
    _assert_bit_exact(f"Linear N={N} K={k0}+{k1}", got, want)


@pytest.mark.parametrize("N", (17, 64))
def test_grad_input_two_column_blocks_rounds_to_nearest(N):
    B, n, n_in, w_off = 2, 1500, 512, 8
    g = torch.Generator(device=DEV).manual_seed(N)
    gy, gyr = _tailed((B, n, N), g)
    w, wr = _tailed((N, n_in + 24), g)
    got = backward.grad_input(gy, w, n_in, w_off=w_off, ldw=w.shape[1])
    _assert_bit_exact(f"dX N={N} n_in={n_in}", got, gyr @ wr[:, w_off:w_off + n_in])


# S = 1 (two), S >= 32 with the tall reduction (two), the cap S = 296 (two)
GW_ROUNDING = [c for c in GW_CASES if c in {(1, 64, 64), (511, 17, 17), (40000, 64, 64), (40000, 17, 512),
                                              (160001, 128, 64), (160993, 64, 512)}]


@pytest.mark.parametrize("R,N,K", GW_ROUNDING, ids=[f"R{r}_N{n}_K{k}" for r, n, k in GW_ROUNDING])
def test_grad_weight_rounds_to_nearest(R, N, K):
    S, _ = _split(R, N)
    g = torch.Generator(device=DEV).manual_seed(R + N + K)
    gy, gyr = _tailed((R, N), g)
    x, xr = _tailed((R, K), g)
    out = torch.full((N, K), float("nan"), device=DEV)
    backward.grad_weight(gy, x, out)
    _assert_bit_exact(f"dW R={R} N={N} K={K} (S={S})", out, gyr.t() @ xr)


def test_tailed_operands_tell_the_rounding_modes_apart():
    """the premise of A and B, on the oracle: tailed values round to s t to nearest and to s (t - ulp) toward zero"""
    x, xr = _tailed((4096,), torch.Generator(device=DEV).manual_seed(0))
    x, xr = x.cpu(), xr.cpu()
    assert torch.equal(rp.round_tf32(x).double(), xr)
    assert torch.equal(rp.round_tf32(x.double()), xr)
    ulp = torch.where(xr.abs() < 0.5, 2.0 ** -12, 2.0 ** -11)
    assert torch.equal(rp.round_tf32(x.double(), "rz"), xr - xr.sign() * ulp)
    assert torch.equal(rp.round_tf32(x, "rz").double(), xr - xr.sign() * ulp)


# ------------------------------------------------------------------------------------------------ B. every forward path
def _tail_params(module, seed):
    """weights: tailed / 8; 1-D parameters (biases, LayerNorm): + 0.1 N(0, 1)"""
    gen = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p in module.parameters():
            if p.dim() == 2:
                p.copy_(_tailed(p.shape, gen, 0.125)[0])
            else:
                p.add_(0.1 * torch.randn(p.shape, generator=gen))
    return module


def _p64(module, prefix=None):
    return {(f"{prefix}.{k}" if prefix else k): v.detach().cpu().double() for k, v in module.state_dict().items()}


def _inputs(shapes, seed):
    gen = torch.Generator().manual_seed(seed)
    return [_tailed(sh, gen)[0] for sh in shapes]


def _graph(ns, nr, ne, seed, sort=True):
    g = torch.Generator().manual_seed(seed)
    ei = torch.stack([torch.randint(0, ns, (ne,), generator=g), torch.randint(0, nr, (ne,), generator=g)])
    ei[1, -1] = nr - 1
    return ei[:, torch.sort(ei[1], stable=True).indices] if sort else ei


def _ell_graph(ns, nr, d, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.stack([torch.randint(0, ns, (nr * d,), generator=g), torch.arange(nr).repeat_interleave(d)])


def _rows_case(blueprint, shapes, res_i, ln, flags_path):
    """make_mlp on row sources: flags_path "fused" = ops.rowmlp (H = 64 row kernel), "generic" = apply_rows with the
    TF32 flag (H = 128 / 256: tc_linear_kernel)"""
    m = _tail_params(make_mlp(blueprint, layer_norm=ln), len(blueprint) + len(shapes))
    srcs = _inputs(shapes, 3)
    B = max((t.shape[0] for t in srcs if t.dim() == 3), default=1)
    cat64 = torch.cat([(t if t.dim() == 3 else t.unsqueeze(0).expand(B, -1, -1)).double() for t in srcs], dim=-1)
    p64 = _p64(m, "m")

    def ref():
        y = rp.mlp(cat64, p64, "m", layer_norm=ln)
        return y if res_i is None else y + srcs[res_i].double()

    m = m.to(DEV)
    ds = [t.to(DEV) for t in srcs]
    res = None if res_i is None else ds[res_i]
    with torch.no_grad(), ops.profile_launches() as prof:
        if flags_path == "fused":
            got = ops.rowmlp(m, ds, res=res, flags=_lib.MATH_TF32)
        else:
            m.nlam_flags = _lib.MATH_TF32
            got = m.apply_rows(ds, res=res)
    return got, ref, prof.names()


def _case_output_map_step():
    m = _tail_params(make_mlp([64, 64, 17], layer_norm=False), 4)
    x, prev = _inputs([(3, 900, 64), (3, 900, 17)], 5)
    gen = torch.Generator().manual_seed(6)
    std, mean = torch.rand(17, generator=gen) + 0.5, torch.randn(17, generator=gen)
    p64 = _p64(m, "m")

    def ref():
        return prev.double() + rp.mlp(x.double(), p64, "m", layer_norm=False) * std.double() + mean.double()

    m = m.to(DEV)
    with torch.no_grad(), ops.profile_launches() as prof:
        got = ops.rowmlp_step(m, x.to(DEV), prev.to(DEV), None, None, std.to(DEV), mean.to(DEV))
    return got, ref, prof.names()


def _inet_case(cls, H, ei, ns, nr, B, upd=True, aggr="sum", bcast=(), chunks=None):
    """one InteractionNet / PropagationNet call (module forward, math="tf32"); bcast: inputs given as stride-0 batch
    expansions ("rec", "edge")"""
    kw = dict(edge_chunk_sizes=chunks[0], aggr_chunk_sizes=chunks[1]) if chunks else {}
    net = _tail_params(getattr(nlb, cls)(ei, H, update_edges=upd, aggr=aggr, math="tf32", **kw), H + ei.shape[1])
    ne = ei.shape[1]
    send, rec, edge = _inputs([(B, ns, H), (1 if "rec" in bcast else B, nr, H), (1 if "edge" in bcast else B, ne, H)], 7)
    p64 = _p64(net)
    prop = cls == "PropagationNet"

    def ref():
        return rp.interaction_net(p64, ei, send.double(), rec.double().expand(B, -1, -1), edge.double().expand(B, -1, -1),
                                  aggr=aggr, update_edges=upd, propagation=prop,
                                  **({"edge_chunk_sizes": chunks[0], "aggr_chunk_sizes": chunks[1]} if chunks else {}))

    net = net.to(DEV)
    with torch.no_grad(), ops.profile_launches() as prof:
        got = net(send.to(DEV), rec.to(DEV).expand(B, -1, -1), edge.to(DEV).expand(B, -1, -1))
    return got, ref, prof.names()


def _inet_fwd_case(inplace):
    """ops.inet_fwd with the edge tensor written out of place (tc_edge3_kernel) or updated in place (tc_edge_rmw_kernel)"""
    nn_, B = 300, 3
    ei = _graph(nn_, nn_, 2600, 3)
    net = _tail_params(nlb.InteractionNet(ei, 64, update_edges=True, math="tf32"), 8)
    x, edge = _inputs([(B, nn_, 64), (B, 2600, 64)], 9)
    p64 = _p64(net)

    def ref():
        return rp.interaction_net(p64, ei, x.double(), x.double(), edge.double(), update_edges=True)

    net = net.to(DEV)
    g = net._graph(torch.device(DEV, torch.cuda.current_device()))
    xs, e0 = x.to(DEV), edge.to(DEV)
    with torch.no_grad(), ops.profile_launches() as prof:
        rec, e1, _ = ops.inet_fwd(g, net.edge_mlp, net.aggr_mlp, xs, xs, e0.clone() if inplace else e0, True, net._flags(),
                                  edge_inplace=inplace)
    return (rec, e1), ref, prof.names()


def _case_node_proj():
    """layer 1's node kernel also computes layer 2's node projections (tc_node_proj_kernel); layer 2 consumes them"""
    N, B = 500, 3
    ei = _graph(N, N, 9 * N, 7)
    l1 = _tail_params(nlb.InteractionNet(ei, 64, math="tf32"), 10)
    l2 = _tail_params(nlb.InteractionNet(ei, 64, math="tf32"), 11)
    x, e = _inputs([(B, N, 64), (B, 9 * N, 64)], 12)
    p1, p2 = _p64(l1), _p64(l2)

    def ref():
        r1, e1 = rp.interaction_net(p1, ei, x.double(), x.double(), e.double())
        r2, _ = rp.interaction_net(p2, ei, r1, r1, e1)
        return r1, e1, r2

    l1, l2 = l1.to(DEV), l2.to(DEV)
    with torch.no_grad(), ops.profile_launches() as prof:
        y1, f1, proj = l1.forward_stacked(x.to(DEV), e.to(DEV), first=True, last=False, next_layer=l2)
        y2, _, _ = l2.forward_stacked(y1, f1, first=False, last=True, proj_in=proj)
    return (y1, f1, y2), ref, prof.names()


def _case_node_out():
    """node update of the mesh -> grid layer + output_map + forecast-step epilogue in one launch (tc_node_out_kernel)"""
    B, G = 3, 1000
    ei = _graph(50, G, 4 * G, 2)
    net = _tail_params(nlb.InteractionNet(ei, 64, update_edges=False, math="tf32"), 13)
    out_map = _tail_params(make_mlp([64, 64, 17], layer_norm=False), 14)
    rec, aggr, prev = _inputs([(B, G, 64), (B, G, 64), (B, G, 17)], 15)
    gen = torch.Generator().manual_seed(16)
    std, mean = torch.rand(17, generator=gen) + 0.5, torch.randn(17, generator=gen)
    pn, po = _p64(net), _p64(out_map, "m")

    def ref():
        r64 = rec.double()
        grid = r64 + rp.mlp(torch.cat([r64, aggr.double()], -1), pn, "aggr_mlp")
        return prev.double() + rp.mlp(grid, po, "m", layer_norm=False) * std.double() + mean.double()

    net, out_map = net.to(DEV), out_map.to(DEV)
    with torch.no_grad(), ops.profile_launches() as prof:
        got = ops.node_update_step(net.aggr_mlp, out_map, rec.to(DEV), aggr.to(DEV), prev.to(DEV), None, None,
                                   std.to(DEV), mean.to(DEV))
    return got, ref, prof.names()


FWD_CASES = {
    # name: (kernel that must run, case)
    "rowmlp_grid_embedder_56": ("tc_rowmlp_kernel", lambda: _rows_case(
        [56, 64, 64], [(2, 400, 17), (2, 400, 17), (2, 400, 18), (400, 4)], None, True, "fused")),
    "rowmlp_node_update_res": ("tc_rowmlp_kernel", lambda: _rows_case(
        [128, 64, 64], [(2, 777, 64), (2, 777, 64)], 0, True, "fused")),
    "rowmlp_output_map_step": ("tc_rowmlp_kernel", _case_output_map_step),
    "edge_k192": ("tc_edge_kernel", lambda: _inet_case("InteractionNet", 64, _graph(40, 600, 300, 1), 40, 600, 2)),
    "edge3_out_of_place": ("tc_edge3_kernel", lambda: _inet_fwd_case(False)),
    "edge_rmw_in_place": ("tc_edge_rmw_kernel", lambda: _inet_fwd_case(True)),
    "edge_bcast_g2m": ("tc_edge_bcast_kernel", lambda: _inet_case(
        "InteractionNet", 64, _graph(3000, 200, 2500, 1), 3000, 200, 3, upd=False, bcast=("rec", "edge"))),
    "ell_window_d4_mean": ("tc_ell_window_kernel", lambda: _inet_case(
        "InteractionNet", 64, _ell_graph(100, 1000, 4, 1), 100, 1000, 3, upd=False, aggr="mean")),
    "node_proj_chain": ("tc_node_proj_kernel", _case_node_proj),
    "node_out_step": ("tc_node_out_kernel", _case_node_out),
    "linear_mlp_h128": ("tc_linear_kernel", lambda: _rows_case([128, 128, 128], [(2, 700, 128)], None, True, "generic")),
    "linear_mlp_h256_res": ("tc_linear_kernel", lambda: _rows_case(
        [512, 256, 256], [(1, 1000, 256), (1, 1000, 256)], 1, True, "generic")),
    "linear_inet_h128": ("tc_linear_kernel", lambda: _inet_case(
        "InteractionNet", 128, _graph(300, 200, 1500, 3), 300, 200, 2)),
    "linear_prop_h64": ("tc_linear_kernel", lambda: _inet_case(
        "PropagationNet", 64, _graph(120, 80, 700, 3), 120, 80, 2)),
    "linear_split_mlps": ("tc_linear_kernel", lambda: _inet_case(
        "InteractionNet", 64, _graph(70, 50, 600, 4, sort=False), 70, 50, 2, chunks=([250, 350], [20, 30]))),
}


@pytest.mark.parametrize("name", list(FWD_CASES))
def test_forward_path_rounds_operands_to_nearest(name):
    kernel, case = FWD_CASES[name]
    got, ref, names = case()
    assert any(n.startswith(kernel) for n in names), f"{kernel} did not run: {names}"
    got = got if isinstance(got, tuple) else (got,)
    with torch.no_grad():
        with rp.tf32_matmul(mode="rna"):
            rna = ref()
        with rp.tf32_matmul(mode="rz"):
            rz = ref()
    rna = rna if isinstance(rna, tuple) else (rna,)
    rz = rz if isinstance(rz, tuple) else (rz,)
    got = torch.cat([g.detach().double().cpu().reshape(w.shape).flatten() for g, w in zip(got, rna)])
    rna, rz = torch.cat([w.flatten() for w in rna]), torch.cat([w.flatten() for w in rz])
    d_rna, d_rz = (got - rna).norm().item(), (got - rz).norm().item()
    err = (got - rna).abs().max().item()
    print(f"\n{name} ({kernel}): ||got - ref_rna|| / ||got - ref_rz|| = {d_rna / d_rz:.3f}; "
          f"max |got - ref_rna| {err:.3e}, max |ref_rna - ref_rz| {(rna - rz).abs().max().item():.3e}")
    assert err <= ABS_TOL, f"{name}: max err {err:.3e} > {ABS_TOL}"
    assert d_rna <= RATIO * d_rz, (f"{name}: the output is closer to truncated operands than to rounded ones "
                                   f"(||got - ref_rna|| = {d_rna:.3e}, ||got - ref_rz|| = {d_rz:.3e})")


# ------------------------------------------------------------------------------------------------ C. unbiasedness
SLOPE_GEMM = 1e-4


def test_linear_unbiased_at_scale():
    g = torch.Generator(device=DEV).manual_seed(21)
    x, w = torch.randn(1, 100000, 128, device=DEV, generator=g), torch.randn(128, 128, device=DEV, generator=g)
    s = _slope(backward.linear(x, w, 128), x.double() @ w.double().t())
    print(f"\nLinear 100000x128 . 128x128: slope {s:+.2e}")
    assert abs(s) <= SLOPE_GEMM, s


def test_grad_input_unbiased_at_scale():
    g = torch.Generator(device=DEV).manual_seed(22)
    gy, w = torch.randn(2, 50000, 128, device=DEV, generator=g), torch.randn(128, 256, device=DEV, generator=g)
    s = _slope(backward.grad_input(gy, w, 256), gy.double() @ w.double())
    print(f"\ngrad_input 2x50000x128 . 128x256: slope {s:+.2e}")
    assert abs(s) <= SLOPE_GEMM, s


def test_grad_weight_unbiased_at_scale():
    R, N, K = 160993, 128, 64
    assert _split(R, N)[0] == 296
    g = torch.Generator(device=DEV).manual_seed(23)
    gy, x = torch.randn(R, N, device=DEV, generator=g), torch.randn(R, K, device=DEV, generator=g)
    out = torch.empty(N, K, device=DEV)
    backward.grad_weight(gy, x, out)
    s = _slope(out, gy.double().t() @ x.double())
    print(f"\ngrad_weight R={R} N={N} K={K}: slope {s:+.2e}")
    assert abs(s) <= SLOPE_GEMM, s


# ------------------------------------------------------------------------------------------------ D. a training step
# measured on an H100 80GB HBM3 (700 W): worst slope -9.85e-4 with rounded operands; -2.37e-3 when the generic Linear
# truncated its operands, +1.62e-3 with the fused kernel's operands truncated.  Bound: min(3 x -9.85e-4, 1e-3).
SLOPE_STEP = 1e-3


def test_training_step_gradients_unbiased():
    """GraphLAM H = 64 (forward on the fused kernels, backward on the generic Linear), one step: the slope of every
    parameter gradient against fp64 autograd through the oracle"""
    spec = synthetic.make_graph_spec(30, 27, hierarchical=False)
    ds = synthetic.SyntheticDatastore(spec, d_state=17, d_forcing=18, d_static=4, boundary_width=2)
    torch.manual_seed(42)
    m = models.GraphLAM(ds, spec, hidden_dim=64, processor_layers=2, math="auto")
    g = _oracle_graph(m)
    cfg = dict(model="graph_lam", hidden_layers=1, processor_layers=2, mesh_aggr="sum")
    G = m.num_grid_nodes
    gen = torch.Generator().manual_seed(5)
    prev, pprev, forc = (torch.randn(2, G, d, generator=gen) for d in (17, 17, 18))
    w = torch.randn(2, G, 17, generator=gen)
    p64 = {k: (v.detach().double().requires_grad_(True) if v.is_floating_point() else v) for k, v in m.state_dict().items()}
    (rp.graph_model_forward(p64, g, cfg, prev.double(), pprev.double(), forc.double()) * w.double()).sum().backward()
    m = m.to(DEV)

    def step():
        got, _ = m(prev.to(DEV), pprev.to(DEV), forc.to(DEV))
        (got * w.to(DEV)).sum().backward()

    _run_checked(step, need=("ln_bwd_kernel", "transpose_pad_kernel"))
    slopes = {k: _slope(p.grad.cpu(), p64[k].grad) for k, p in m.named_parameters()
              if p64[k].grad is not None and p64[k].grad.abs().max() > 0}  # (a zero gradient has no slope)
    worst = max(slopes, key=lambda k: abs(slopes[k]))
    print(f"\nGraphLAM H=64 training step: gradient slopes vs fp64 autograd, worst {slopes[worst]:+.2e} ({worst})")
    for k, s in sorted(slopes.items(), key=lambda kv: kv[1]):
        print(f"  {s:+.2e}  {k}")
    assert abs(slopes[worst]) <= SLOPE_STEP, f"{worst}: gradient slope {slopes[worst]:+.2e}"
