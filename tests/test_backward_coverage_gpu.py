"""The hand-written backward (neural_lam_b200/backward.py, csrc/bwd.cu) at training-sized and edge-case shapes.

1. Exact-arithmetic unit tests of the building blocks (``grad_weight``, ``grad_input``, ``colsum``, ``layernorm_bwd``).
   Operands are drawn from {±0.25, ±0.5, ±0.75, ±1}: TF32 rounding of such operands is exact, every product is a
   multiple of 1/16 below 1, and every partial and full sum stays far below 2^24 / 16, so each sum is exact in fp32 in
   any order.  The kernels must then equal the fp64 product BIT FOR BIT, at every split-K range count S (up to its cap
   of 296): a dropped, duplicated or shifted row range, a wrong transpose or a wrong column offset is a mismatch.
2. Layer-level gradients of InteractionNet / PropagationNet / make_mlp against fp64 autograd through the oracle
   (oracle/reference_port.py) on the edge cases of the index plumbing, and at sizes where S reaches its cap.
3. Whole training steps (three-level HiLAM at H = 64, GraphLAM at H = 128) against fp64 autograd.

Every layer-level case also checks that the library's backward ran (``ln_bwd_kernel`` / ``transpose_pad_kernel`` among
the launches) and that no library GEMM did.  TF32 tolerances: |g - g_ref| <= 2e-2 * max|g_ref| + 1e-4 per tensor (as in
test_backward_gpu.py) and ||g - g_ref||_F <= FROB * ||g_ref||_F per tensor (layers; measured at most 1.6e-3 on an
H100 80GB HBM3, 700 W); the measured values are printed (run with -s).
"""
import pytest
import torch
import torch.nn.functional as F

import neural_lam_b200 as nlb
from neural_lam_b200 import _lib, backward, models, ops, synthetic
from oracle import reference_port as rp
from test_models import _oracle_graph

pytestmark = pytest.mark.gpu
DEV = "cuda"
FROB = 4e-3
_LIB_GEMM = ("gemm", "cublas", "cutlass", "gemv")


# ------------------------------------------------------------------------------------------------ helpers
def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _exact(shape, gen):
    """values in {±0.25, ±0.5, ±0.75, ±1} (exact in TF32; products exact multiples of 1/16)"""
    mag = (torch.randint(1, 5, shape, device=DEV, generator=gen) * 0.25).float()
    sign = torch.randint(0, 2, shape, device=DEV, generator=gen).float() * 2 - 1
    return mag * sign


def _assert_bit_exact(name, got, want):
    got = got.double()
    assert got.shape == want.shape, (name, got.shape, want.shape)
    bad = got != want
    if bad.any():
        n = int(bad.sum())
        err = (got - want).abs().nan_to_num(float("inf")).max().item()
        raise AssertionError(f"{name}: {n} of {got.numel()} elements differ from the exact product (max |err| {err:.3e})")


def _check(name, got, want, rel=2e-2, abs_=1e-4, frob=FROB):
    """max-normalised bound + relative Frobenius error (a reference of zeros, or None for a parameter the loss does not
    reach, must be matched exactly); -> (relative Frobenius error, max err / max |ref|)"""
    assert got is not None, name
    got = got.detach().double()
    want = torch.zeros_like(got) if want is None else want.detach().double().to(got.device)
    assert got.shape == want.shape, (name, got.shape, want.shape)
    d = got - want
    err, ref_max = d.abs().max().item(), want.abs().max().item()
    fro = d.norm().item() / max(want.norm().item(), 1e-300)
    assert err <= rel * ref_max + abs_, f"{name}: max err {err:.3e} > {rel * ref_max + abs_:.3e} (max |ref| {ref_max:.3e})"
    assert frob is None or fro <= frob, f"{name}: relative Frobenius error {fro:.3e} > {frob:.0e}"
    return fro, err / max(ref_max, 1e-300)


def _report(case, errs):
    fro = max(errs.items(), key=lambda kv: kv[1][0])
    rel = max(errs.items(), key=lambda kv: kv[1][1])
    print(f"\n{case}: worst relative Frobenius error {fro[1][0]:.3e} ({fro[0]}), "
          f"worst max err / max |ref| {rel[1][1]:.3e} ({rel[0]})")


def _run_checked(step, need=("transpose_pad_kernel",)):
    """run ``step`` under both profilers: the library's backward kernels ran, no library GEMM did"""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        with ops.profile_launches() as lp:
            step()
        torch.cuda.synchronize()
    kernels = [e.key for e in prof.key_averages()]
    bad = [k for k in kernels if any(t in k.lower() for t in _LIB_GEMM)]
    assert not bad, f"library GEMMs in the backward: {bad}"
    names = lp.names()
    for n in need:
        assert n in names, f"{n} not launched: the library's backward did not run ({sorted(set(names))})"


# ------------------------------------------------------------------------------------------------ 1. exact unit tests
def _split(R, N):
    """(S, k_per) of grad_weight: the row ranges of the split-K product"""
    n_tiles = (N + 127) // 128
    S = max(1, min(296 // n_tiles, (R + 511) // 512))
    return S, ((R + S - 1) // S + 31) // 32 * 32


GW_CASES = [
    # R, N, K
    (1, 64, 64),          # S = 1, one row
    (511, 17, 17),        # S = 1, narrow N (TMA box padding) and kc < 32
    (4097, 64, 56),       # S = 9
    (4097, 256, 300),     # two column chunks (256 + 44), n_tiles = 2
    (40000, 64, 64),      # S = 79 >= 32, N * K <= 8192: reduce_partials_tall_kernel
    (40000, 17, 512),     # two full chunks, tall reduction
    (160001, 128, 64),    # S = 296 (cap), k_per = 544: range 294 holds 65 rows, range 295 only padding; tall reduction
    (160001, 17, 300),    # cap, chunks 256 + 44
    (160993, 64, 512),    # cap, every range holds rows (the last 513); N * kc > 8192: reduce_partials_kernel
    (80001, 256, 56),     # n_tiles = 2: S = 148, the last range holds 33 rows
    (80001, 256, 17),
]


@pytest.mark.parametrize("R,N,K", GW_CASES, ids=[f"R{r}_N{n}_K{k}" for r, n, k in GW_CASES])
def test_grad_weight_exact(R, N, K):
    S, _ = _split(R, N)
    g = _gen(R + N + K)
    gy, x = _exact((R, N), g), _exact((R, K), g)
    out = torch.full((N, K), float("nan"), device=DEV)
    backward.grad_weight(gy, x, out)
    _assert_bit_exact(f"dW R={R} N={N} K={K} (S={S})", out, gy.double().t() @ x.double())


@pytest.mark.parametrize("R,N,K", [(4097, 64, 64), (160993, 128, 300)])
def test_grad_weight_exact_column_slices(R, N, K):
    """x = columns [x_off, x_off + K) of a wider tensor, written into columns [out_off, out_off + K) of a wider out (the
    dW1 sections of InteractionNet); the columns outside the slice are left untouched"""
    x_off, x_pitch, out_off, out_pitch = 40, K + 72, 37, K + 100
    g = _gen(R + K)
    gy, xw = _exact((R, N), g), _exact((R, x_pitch), g)
    out = torch.full((N, out_pitch), float("nan"), device=DEV)
    backward.grad_weight(gy, xw, out, out_off=out_off, out_pitch=out_pitch, x_off=x_off, x_cols=K, x_pitch=x_pitch)
    _assert_bit_exact("dW slice", out[:, out_off:out_off + K], gy.double().t() @ xw[:, x_off:x_off + K].double())
    outside = torch.cat([out[:, :out_off], out[:, out_off + K:]], dim=1)
    assert outside.isnan().all(), "grad_weight wrote outside its column slice"


GI_CASES = [(N, n_in, res) for N in (17, 64, 256) for n_in in (64, 256, 300, 512) for res in (False, True)
            if not (res and n_in > 256)]


@pytest.mark.parametrize("N,n_in,res", GI_CASES, ids=[f"N{n}_in{k}{'_res' if r else ''}" for n, k, r in GI_CASES])
def test_grad_input_exact(N, n_in, res):
    """gy (B, n, N) · W[:, w_off : w_off + n_in] (+ res); n_in > 256 runs one Linear per 256-column block of W"""
    B, n, w_off = 2, 1500, 8
    g = _gen(N * 1000 + n_in)
    gy = _exact((B, n, N), g)
    w = _exact((N, n_in + 24), g)
    r = _exact((B, n, n_in), g) if res else None
    got = backward.grad_input(gy, w, n_in, w_off=w_off, ldw=w.shape[1], res=r)
    want = gy.double() @ w[:, w_off:w_off + n_in].double()
    if res:
        want = want + r.double()
    _assert_bit_exact(f"dX N={N} n_in={n_in}", got, want)


def test_grad_input_rejects_residual_with_column_blocks():
    gy = torch.zeros(1, 64, 64, device=DEV)
    with pytest.raises(_lib.NlamError, match="residual"):
        backward.grad_input(gy, torch.zeros(64, 300, device=DEV), 300, res=torch.zeros(1, 64, 300, device=DEV))


ROWS = (1, 8447, 8449, 1000003)   # around 2 x the 4224 warps of the column-sum grid


@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("C", (17, 64, 256))
def test_colsum_exact(rows, C):
    g = _exact((rows, C), _gen(rows + C))
    _assert_bit_exact(f"colsum rows={rows} C={C}", backward.colsum(g), g.double().sum(0))


@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("H", (64, 256))
def test_layernorm_bwd_vs_fp64_autograd(rows, H):
    """g_y, dgamma against fp64 autograd of F.layer_norm with fp32 bounds (2^-16 ~ 256 fp32 ulps):
    |g_y - ref| <= 2^-16 (|ref| + s (1 + |x̂|)) with s = max_j |gamma_j g_j| / sigma per row (the terms of
    (gamma g - mean(gamma g) - x̂ mean(gamma g x̂)) / sigma), |dgamma - ref| <= 2^-16 Σ_rows |g x̂|.
    dbeta = Σ_rows g of exact operands: bit-exact."""
    gen = _gen(rows * 7 + H)
    eps = 1e-5
    y = torch.randn(rows, H, device=DEV, generator=gen) * 1.5 + 0.3
    gamma = 1 + 0.1 * torch.randn(H, device=DEV, generator=gen)
    g = _exact((rows, H), gen)
    y64, gm64 = y.double().requires_grad_(True), gamma.double().requires_grad_(True)
    b64 = torch.zeros(H, device=DEV, dtype=torch.float64, requires_grad=True)
    F.layer_norm(y64, (H,), gm64, b64, eps).backward(g.double())
    gy, dg, db = backward.layernorm_bwd(g, y, gamma, eps)
    with torch.no_grad():
        mu = y64.mean(-1, keepdim=True)
        sigma = ((y64 - mu).pow(2).mean(-1, keepdim=True) + eps).sqrt()
        xhat = (y64 - mu) / sigma
        s = (gm64 * g.double()).abs().amax(-1, keepdim=True) / sigma
        bound = 2.0 ** -16 * (y64.grad.abs() + s * (1 + xhat.abs()))
        excess = ((gy.double() - y64.grad).abs() - bound).max().item()
        assert excess <= 0, f"g_y exceeds its bound by {excess:.3e}"
        dg_bound = 2.0 ** -16 * (g.double() * xhat).abs().sum(0)
        dg_excess = ((dg.double() - gm64.grad).abs() - dg_bound).max().item()
        assert dg_excess <= 0, f"dgamma exceeds its bound by {dg_excess:.3e}"
    _assert_bit_exact("dbeta", db, b64.grad)


# ------------------------------------------------------------------------------------------------ 2. layers
def _sorted(ei):
    return ei[:, torch.sort(ei[1], stable=True).indices]


def _graph(kind, gen):
    """-> (edge_index, n_send rows of the sender tensor, n_rec)"""
    if kind == "random":
        ns, nr, ne = 300, 200, 1500
        ei = torch.stack([torch.randint(0, ns, (ne,), generator=gen), torch.randint(0, nr, (ne,), generator=gen)])
        ei[1, -1] = nr - 1
        return ei, ns, nr
    if kind == "unreferenced_senders":        # senders 240..299 are in the tensor but on no edge
        ns, nr, ne = 300, 200, 1500
        ei = torch.stack([torch.randint(0, 240, (ne,), generator=gen), torch.randint(0, nr, (ne,), generator=gen)])
        ei[1, -1] = nr - 1
        return _sorted(ei), ns, nr
    if kind == "zero_in_degree":              # only even receivers (and the last) have edges
        ns, nr, ne = 250, 201, 1200
        ei = torch.stack([torch.randint(0, ns, (ne,), generator=gen), 2 * torch.randint(0, 101, (ne,), generator=gen)])
        ei[1, -1] = nr - 1
        return _sorted(ei), ns, nr
    if kind == "high_in_degree":              # receiver 0 has in-degree 300
        ns, nr, ne = 400, 100, 1300
        ei = torch.stack([torch.randint(0, ns, (ne,), generator=gen), torch.randint(0, nr, (ne,), generator=gen)])
        ei[1, :300] = 0
        ei[1, -1] = nr - 1
        return _sorted(ei), ns, nr
    if kind == "m2g_deg4":                    # every receiver (grid node) reads 4 senders (mesh nodes)
        ns, nr = 120, 1000
        ei = torch.stack([torch.randint(0, ns, (4 * nr,), generator=gen), torch.arange(nr).repeat_interleave(4)])
        return ei, ns, nr
    if kind.startswith("large_"):             # large_<E>_<nodes>
        ne, nn = (int(v) for v in kind.split("_")[1:])
        ei = torch.stack([torch.randint(0, nn, (ne,), generator=gen), torch.randint(0, nn, (ne,), generator=gen)])
        ei[1, -1] = nn - 1
        return _sorted(ei), nn, nn
    raise ValueError(kind)


INET_CASES = [
    # name, class, H, graph, B, update_edges, aggr, stride-0 inputs, loss on
    ("unsorted_update", "InteractionNet", 64, "random", 2, True, "sum", (), "both"),
    ("unreferenced_senders", "InteractionNet", 64, "unreferenced_senders", 2, True, "sum", (), "both"),
    ("mean_zero_in_degree", "InteractionNet", 64, "zero_in_degree", 2, True, "mean", (), "both"),
    ("edge_output_loss_only", "InteractionNet", 64, "random", 2, True, "sum", (), "edge"),
    ("bcast_rec_edge_b3", "InteractionNet", 64, "zero_in_degree", 3, True, "sum", ("rec", "edge"), "both"),
    ("in_degree_300", "InteractionNet", 64, "high_in_degree", 2, True, "sum", (), "both"),
    ("m2g_deg4_noupd", "InteractionNet", 64, "m2g_deg4", 2, False, "sum", (), "rec"),
    ("prop_bcast_send_b3", "PropagationNet", 64, "unreferenced_senders", 3, True, "sum", ("send",), "both"),
    ("prop_h128", "PropagationNet", 128, "random", 2, True, "sum", (), "both"),
    ("h128_bcast_rec_b3", "InteractionNet", 128, "random", 3, False, "mean", ("rec",), "rec"),
]


def _inet_grads(name, cls, H, kind, B, upd, aggr, bcast, loss, seed=0):
    """gradients of one layer call through the library vs fp64 autograd through the oracle -> (net, errors)"""
    gen = torch.Generator().manual_seed(seed + 11)
    ei, ns, nr = _graph(kind, gen)
    torch.manual_seed(seed)
    net = getattr(nlb, cls)(ei, H, update_edges=upd, aggr=aggr, math="auto")
    with torch.no_grad():
        for p in net.parameters():
            if p.dim() == 1:
                p.add_(0.1 * torch.randn_like(p))
    E = ei.shape[1]
    send, rec, edge = (torch.randn(1 if k in bcast else B, n, H, generator=gen) for k, n in (("send", ns), ("rec", nr), ("edge", E)))
    w_rec, w_edge = torch.randn(B, nr, H, generator=gen).to(DEV), torch.randn(B, E, H, generator=gen).to(DEV)

    def loss_of(out):
        if not upd:
            return (out * w_rec.to(out.dtype)).sum()
        if loss == "edge":
            return (out[1] * w_edge.to(out[1].dtype)).sum()
        return (out[0] * w_rec.to(out[0].dtype)).sum() + (out[1] * w_edge.to(out[1].dtype)).sum()

    p64 = {k: v.detach().to(DEV).double().requires_grad_(True) for k, v in net.state_dict().items()}
    x64 = [t.to(DEV).double().requires_grad_(True) for t in (send, rec, edge)]
    s, r, e = (t.expand(B, -1, -1) for t in x64)
    loss_of(rp.interaction_net(p64, ei.to(DEV), s, r, e, aggr=aggr, update_edges=upd, propagation=cls == "PropagationNet")).backward()
    net = net.to(DEV)
    xd = [t.to(DEV).requires_grad_(True) for t in (send, rec, edge)]

    def step():
        loss_of(net(*(t.expand(B, -1, -1) for t in xd))).backward()

    _run_checked(step, need=("ln_bwd_kernel", "transpose_pad_kernel"))
    errs = {f"g_{k}": _check(f"{name} g_{k}", t.grad, t64.grad) for k, t, t64 in zip(("send", "rec", "edge"), xd, x64)}
    for k, p in net.named_parameters():
        errs[k] = _check(f"{name} {k}", p.grad, p64[k].grad)
    _report(name, errs)
    return net, ei


@pytest.mark.parametrize("case", INET_CASES, ids=[c[0] for c in INET_CASES])
def test_layer_backward_edge_cases(case):
    _inet_grads(*case)


@pytest.mark.parametrize("H,E,nodes,S", [(64, 90000, 20000, 296), (256, 40000, 10000, 148)], ids=["h64_cap", "h256_two_tiles"])
def test_layer_backward_at_scale(H, E, nodes, S):
    """B * E rows reach the split-K cap (S = 296 at N <= 128, 148 at N = 256); the one-call ABI backward
    (``nlam_inet_bwd``) equals the host composition (``backward.inet_backward_py``) bit for bit at this size"""
    B = 2
    assert _split(B * E, H)[0] == S
    net, _ = _inet_grads(f"scale_h{H}", "InteractionNet", H, f"large_{E}_{nodes}", B, True, "sum", (), "both")
    g = torch.Generator(device=DEV).manual_seed(3)
    send, rec, edge = (torch.randn(B, n, H, device=DEV, generator=g) for n in (nodes, nodes, E))
    g_rec, g_edge = torch.randn(B, nodes, H, device=DEV, generator=g), torch.randn(B, E, H, device=DEV, generator=g)
    graph = net._graph(send.device)
    a = backward.inet_backward(net, graph, send, rec, edge, g_rec, g_edge)
    b = backward.inet_backward_py(net, graph, send, rec, edge, g_rec, g_edge)
    for x, y in zip(a[:3], b[:3]):
        torch.testing.assert_close(x, y, rtol=0, atol=0)
    assert set(a[3]) == set(b[3])
    for k in a[3]:
        torch.testing.assert_close(a[3][k], b[3][k], rtol=0, atol=0, msg=lambda m: f"{k}: {m}")


MLP_CASES = [
    # name, blueprint, source shapes (None: one stride-0 expanded (1, n, d) source at B = 2), residual, LayerNorm
    ("in300_two_sources_ln", [300, 64, 64], [(2, 500, 150), (2, 500, 150)], False, True),
    ("in257_no_ln", [257, 64, 17], [(2, 500, 250), (500, 7)], False, False),
    ("in512_res", [512, 256, 256], [(2, 400, 256), (2, 400, 256)], True, True),
    ("bcast_source_b2", [64, 64, 64], None, False, True),
]


@pytest.mark.parametrize("case", MLP_CASES, ids=[c[0] for c in MLP_CASES])
def test_mlp_backward_apply_rows(case):
    name, blueprint, shapes, with_res, ln = case
    torch.manual_seed(5)
    mlp = nlb.make_mlp(blueprint, layer_norm=ln)
    gen = torch.Generator().manual_seed(6)
    srcs = [torch.randn(*sh, generator=gen) for sh in shapes] if shapes else [torch.randn(1, 500, blueprint[0], generator=gen)]
    B = 2
    n = srcs[0].shape[-2]
    w = torch.randn(B, n, blueprint[-1], generator=gen).to(DEV)

    def full(t):
        return t.expand(B, -1, -1) if t.dim() == 3 else t.unsqueeze(0).expand(B, -1, -1)

    p64 = {f"m.{k}": v.detach().to(DEV).double().requires_grad_(True) for k, v in mlp.state_dict().items()}
    s64 = [t.to(DEV).double().requires_grad_(True) for t in srcs]
    out = rp.mlp(torch.cat([full(t) for t in s64], dim=-1), p64, "m", 1, layer_norm=ln)
    if with_res:
        out = out + s64[0]
    (out * w.double()).sum().backward()
    mlp = mlp.to(DEV)
    sd = [t.to(DEV).requires_grad_(True) for t in srcs]

    def step():
        xs = sd if shapes else [sd[0].expand(B, -1, -1)]
        (mlp.apply_rows(xs, res=xs[0] if with_res else None) * w).sum().backward()

    _run_checked(step, need=("transpose_pad_kernel",) + (("ln_bwd_kernel",) if ln else ()))
    errs = {f"g_src{i}": _check(f"{name} g_src{i}", t.grad, t64.grad) for i, (t, t64) in enumerate(zip(sd, s64))}
    for k, p in mlp.named_parameters():
        errs[k] = _check(f"{name} {k}", p.grad, p64[f"m.{k}"].grad)
    _report(name, errs)


def test_mlp_backward_abi_equals_host_composition_wide_input():
    """``nlam_mlp_bwd`` and ``backward.mlp_backward_py`` agree bit for bit with column-blocked input gradients"""
    torch.manual_seed(1)
    mlp = nlb.make_mlp([300, 64, 64]).to(DEV)
    g = _gen(9)
    srcs = [torch.randn(2, 700, 150, device=DEV, generator=g), torch.randn(700, 150, device=DEV, generator=g)]
    go = torch.randn(2, 700, 64, device=DEV, generator=g)
    a = backward.mlp_backward(mlp, srcs, None, go)
    b = backward.mlp_backward_py(mlp, srcs, None, go)
    for x, y in zip(a[0], b[0]):
        torch.testing.assert_close(x, y.contiguous(), rtol=0, atol=0)
    for k in a[2]:
        torch.testing.assert_close(a[2][k], b[2][k], rtol=0, atol=0)


# ------------------------------------------------------------------------------------------------ 3. training steps
@pytest.mark.parametrize("kind,hidden", [("hi_lam", 64), ("graph_lam", 128)])
def test_training_step_vs_fp64_autograd(kind, hidden):
    """one model step, loss.backward() through it; every parameter gradient vs autograd through the fp64 oracle
    (bound of test_backward_gpu.py::test_graphlam_training_step_on_kernel_backward)"""
    if kind == "hi_lam":
        spec = synthetic.make_graph_spec(81, 81, hierarchical=True, n_levels=3)
        cls, P = models.HiLAM, 1
    else:
        spec = synthetic.make_graph_spec(30, 27, hierarchical=False)
        cls, P = models.GraphLAM, 2
    ds = synthetic.SyntheticDatastore(spec, d_state=17, d_forcing=18, d_static=4, boundary_width=2)
    torch.manual_seed(42)
    m = cls(ds, spec, hidden_dim=hidden, processor_layers=P, math="auto")
    g = _oracle_graph(m)
    if kind == "hi_lam":
        assert len(g["mesh_static_features"]) == 3
    cfg = dict(model=kind, hidden_layers=1, processor_layers=P, mesh_aggr="sum")
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
    errs = {k: _check(k, p.grad, p64[k].grad, rel=3e-2, abs_=2e-4, frob=None) for k, p in m.named_parameters()}
    _report(f"{kind} H={hidden} training step", errs)
