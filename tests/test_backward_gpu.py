"""The hand-written backward (neural_lam_b200/backward.py: generic wgmma Linear for dX / split-K dW, SiLU / LayerNorm
backward, CSR segment sums) against (1) the gradients of the reference's own source stored in
tests/golden/inet_cases.npz (H = 64 cases), (2) autograd through the fp64 oracle on fresh graphs — all inputs and all
parameters — and (3) a whole GraphLAM training step; plus the proof that no cuBLAS / ATen GEMM runs in it.

Tolerance: TF32 operands in forward and backward (the reference's GPU configuration, train_model.py:484-488):
|g - g_ref| <= 2e-2 * max|g_ref| + 1e-4 per tensor (measured ~3e-3 relative).
"""
import pytest
import torch

import neural_lam_b200 as nlb
from neural_lam_b200 import models, ops, synthetic
from oracle import reference_port as rp

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _close(name, got, want, rel=2e-2, abs_=1e-4):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    assert got.shape == want.shape, (name, got.shape, want.shape)
    err = (got - want).abs().max().item()
    bound = rel * want.abs().max().item() + abs_
    assert err <= bound, f"{name}: max err {err:.3e} > {bound:.3e} (max |ref| {want.abs().max().item():.3e})"
    return err / max(want.abs().max().item(), 1e-30)


def _cuda_kernel_names(fn):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.key for e in prof.key_averages()]


def test_backward_matches_reference_golden_h64(golden_cases):
    """inputs, weights, output weights and ALL gradients were produced by the reference's InteractionNet source"""
    cases = [c for c in golden_cases if c.name in ("inet_m2m_h64", "inet_g2m_h64_highdeg")]
    assert len(cases) == 2
    for case in cases:
        H = case.t["send"].shape[-1]
        net = nlb.InteractionNet(case.t["edge_index"], H, math="auto", **case.kwargs)
        net.load_state_dict(case.params)
        net = net.to(DEV)
        send = case.t["send"].to(DEV).requires_grad_(True)
        edge = case.t["edge"].to(DEV).requires_grad_(True)
        rec = send if case.same else case.t["rec"].to(DEV).requires_grad_(True)
        with ops.profile_launches() as prof:
            out = net(send, rec, edge)
            if net.update_edges:
                loss = (out[0] * case.t["w_rec"].to(DEV)).sum() + (out[1] * case.t["w_edge"].to(DEV)).sum()
            else:
                loss = (out * case.t["w_rec"].to(DEV)).sum()
            loss.backward()
        names = prof.names()
        assert "ln_bwd_kernel" in names and "transpose_pad_kernel" in names, names  # the kernel backward ran
        rels = [_close("g_send", send.grad, case.t["g_send"]), _close("g_edge", edge.grad, case.t["g_edge"])]
        if not case.same:
            rels.append(_close("g_rec", rec.grad, case.t["g_rec"]))
        for k, p in net.named_parameters():
            rels.append(_close(k, p.grad, case.gparams[k]))
        print(f"{case.name}: max relative gradient error {max(rels):.3e}")


CASES = [
    # name, class, H, ns, nr, ne, B, update_edges, aggr, sorted, expanded edge, same nodes
    ("h64_sum_upd", "InteractionNet", 64, 300, 200, 1500, 2, True, "sum", True, False, False),
    ("h64_mean_noupd_unsorted", "InteractionNet", 64, 300, 200, 1500, 3, False, "mean", False, False, False),
    ("h64_m2m_same_bcast_edge", "InteractionNet", 64, 250, 250, 2000, 2, True, "sum", True, True, True),
    ("h64_prop", "PropagationNet", 64, 120, 80, 700, 2, True, "sum", True, False, False),
    ("h128_sum_upd", "InteractionNet", 128, 200, 150, 900, 2, True, "sum", True, False, False),
    ("h256_noupd", "InteractionNet", 256, 150, 100, 600, 1, False, "sum", True, False, False),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_backward_vs_fp64_oracle_autograd(case):
    name, cls, H, ns, nr, ne, B, upd, aggr, srt, expand, same = case
    g = torch.Generator().manual_seed(7)
    ei = torch.stack([torch.randint(0, ns, (ne,), generator=g), torch.randint(0, nr, (ne,), generator=g)])
    ei[1, -1] = nr - 1
    if srt:
        ei = ei[:, torch.sort(ei[1], stable=True).indices]
    torch.manual_seed(3)
    net = getattr(nlb, cls)(ei, H, update_edges=upd, aggr=aggr, math="auto")
    with torch.no_grad():
        for p in net.parameters():
            if p.dim() == 1:
                p.add_(0.1 * torch.randn_like(p))
    send = torch.randn(B, ns, H)
    rec = send if same else torch.randn(B, nr, H)
    edge = torch.randn(1 if expand else B, ne, H)
    w_rec, w_edge = torch.randn(B, nr, H), torch.randn(B, ne, H)
    prop = cls == "PropagationNet"
    # fp64 oracle + autograd
    p64 = {k: v.detach().double().requires_grad_(True) for k, v in net.state_dict().items()}
    s64 = send.double().requires_grad_(True)
    r64 = s64 if same else rec.double().requires_grad_(True)
    e64 = edge.double().requires_grad_(True)
    out = rp.interaction_net(p64, ei, s64, r64, e64.expand(B, -1, -1), aggr=aggr, update_edges=upd, propagation=prop)
    loss = (out[0] * w_rec.double()).sum() + (out[1] * w_edge.double()).sum() if upd else (out * w_rec.double()).sum()
    loss.backward()
    # kernels
    net = net.to(DEV)
    sd = send.to(DEV).requires_grad_(True)
    rd = sd if same else rec.to(DEV).requires_grad_(True)
    ed = edge.to(DEV).requires_grad_(True)

    def step():
        o = net(sd, rd, ed.expand(B, -1, -1))
        l = (o[0] * w_rec.to(DEV)).sum() + (o[1] * w_edge.to(DEV)).sum() if upd else (o * w_rec.to(DEV)).sum()
        l.backward()

    kernels = _cuda_kernel_names(step)
    bad = [k for k in kernels if any(t in k.lower() for t in ("gemm", "cublas", "cutlass", "gemv"))]
    assert not bad, f"library GEMMs in the training step: {bad}"
    rels = [_close("g_send", sd.grad, s64.grad), _close("g_edge", ed.grad, e64.grad)]
    if not same:
        rels.append(_close("g_rec", rd.grad, r64.grad))
    for k, p in net.named_parameters():
        rels.append(_close(k, p.grad, p64[k].grad))
    print(f"{name}: max relative gradient error vs fp64 autograd {max(rels):.3e}")


MLP_CASES = [
    ("embed_64", [64, 64, 64], [(2, 300, 64)], False, True),
    ("node_res", [128, 64, 64], [(2, 300, 64), (2, 300, 64)], True, True),
    ("grid_embedder_56", [56, 64, 64], [(2, 400, 17), (2, 400, 17), (2, 400, 18), (400, 4)], False, True),
    ("output_map_17", [64, 64, 17], [(2, 500, 64)], False, False),
    ("h128_node_res", [256, 128, 128], [(2, 200, 128), (2, 200, 128)], True, True),
    ("edge_embedder_3", [3, 64, 64], [(700, 3)], False, True),
]


@pytest.mark.parametrize("case", MLP_CASES, ids=[c[0] for c in MLP_CASES])
def test_mlp_backward_vs_fp64_autograd(case):
    name, blueprint, shapes, with_res, ln = case
    torch.manual_seed(5)
    mlp = nlb.make_mlp(blueprint, layer_norm=ln)
    srcs = [torch.randn(*sh) for sh in shapes]
    B = max((t.shape[0] for t in srcs if t.dim() == 3), default=1)
    w = torch.randn(B, shapes[0][-2], blueprint[-1])
    p64 = {f"m.{k}": v.detach().double().requires_grad_(True) for k, v in mlp.state_dict().items()}
    s64 = [t.double().requires_grad_(True) for t in srcs]
    cat = torch.cat([t if t.dim() == 3 else t.unsqueeze(0).expand(B, -1, -1) for t in s64], dim=-1)
    out = rp.mlp(cat, p64, "m", 1, layer_norm=ln)
    if with_res:
        out = out + s64[0]
    (out * w.double()).sum().backward()
    mlp = mlp.to(DEV)
    sdev = [t.to(DEV).requires_grad_(True) for t in srcs]

    def step():
        o = mlp.apply_rows(sdev, res=sdev[0] if with_res else None)
        (o * w.to(DEV)).sum().backward()

    kernels = _cuda_kernel_names(step)
    assert not [k for k in kernels if any(t in k.lower() for t in ("gemm", "cublas", "cutlass"))], kernels
    rels = [_close(f"g_src{i}", t.grad, s.grad) for i, (t, s) in enumerate(zip(sdev, s64))]
    for k, p in mlp.named_parameters():
        rels.append(_close(k, p.grad, p64[f"m.{k}"].grad))
    print(f"{name}: max relative gradient error {max(rels):.3e}")


def test_graphlam_training_step_on_kernel_backward():
    """One GraphLAM training step (MEPS-shaped feature widths, H = 64, tensor-core forward): loss.backward() through the
    whole step, every gradient vs autograd on the fp64 oracle, no library GEMM among the launched kernels."""
    spec = synthetic.make_graph_spec(30, 27, hierarchical=False)
    ds = synthetic.SyntheticDatastore(spec, d_state=17, d_forcing=18, d_static=4, boundary_width=2)
    torch.manual_seed(42)
    m = models.GraphLAM(ds, spec, hidden_dim=64, processor_layers=2, math="auto")
    g = {k: getattr(m, k).detach().cpu() for k in ("grid_static_features", "g2m_features", "m2g_features", "g2m_edge_index",
                                                    "m2g_edge_index", "diff_std", "diff_mean", "m2m_features", "m2m_edge_index",
                                                    "mesh_static_features")}
    cfg = dict(model="graph_lam", hidden_layers=1, processor_layers=2, mesh_aggr="sum")
    G = m.num_grid_nodes
    gen = torch.Generator().manual_seed(5)
    prev, pprev, forc = torch.randn(2, G, 17, generator=gen), torch.randn(2, G, 17, generator=gen), torch.randn(2, G, 18, generator=gen)
    w = torch.randn(2, G, 17, generator=gen)
    p64 = {k: (v.detach().double().requires_grad_(True) if v.is_floating_point() else v) for k, v in m.state_dict().items()}
    out = rp.graph_model_forward(p64, g, cfg, prev.double(), pprev.double(), forc.double())
    (out * w.double()).sum().backward()
    m = m.to(DEV)

    def step():
        got, _ = m(prev.to(DEV), pprev.to(DEV), forc.to(DEV))
        (got * w.to(DEV)).sum().backward()

    kernels = _cuda_kernel_names(step)
    bad = [k for k in kernels if any(t in k.lower() for t in ("gemm", "cublas", "cutlass", "gemv"))]
    assert not bad, f"library GEMMs in the training step: {bad}"
    worst = 0.0
    for k, p in m.named_parameters():
        assert p.grad is not None, k
        worst = max(worst, _close(k, p.grad, p64[k].grad, rel=3e-2, abs_=2e-4))
    print(f"GraphLAM training step: max relative gradient error {worst:.3e}")


def test_abi_backward_chain_equals_host_composition():
    """``nlam_inet_bwd`` / ``nlam_mlp_bwd`` (one ABI call per layer, temporaries in a caller-provided workspace) launch
    the same kernels in the same order as the host-side compositions of backward.py: bit-identical gradients."""
    from neural_lam_b200 import backward

    g = torch.Generator().manual_seed(2)
    ns, nr, ne, H, B = 180, 120, 1000, 64, 2
    ei = torch.stack([torch.randint(0, ns, (ne,), generator=g), torch.randint(0, nr, (ne,), generator=g)])
    ei[1, -1] = nr - 1
    ei = ei[:, torch.sort(ei[1], stable=True).indices]
    for cls, aggr, upd in ((nlb.InteractionNet, "mean", True), (nlb.PropagationNet, "sum", False)):
        torch.manual_seed(0)
        net = cls(ei, H, update_edges=upd, aggr=aggr).to(DEV)
        send, rec = torch.randn(B, ns, H, device=DEV), torch.randn(nr, H, device=DEV).unsqueeze(0).expand(B, -1, -1)
        edge = torch.randn(B, ne, H, device=DEV)
        g_rec, g_edge = torch.randn(B, nr, H, device=DEV), (torch.randn(B, ne, H, device=DEV) if upd else None)
        graph = net._graph(send.device)
        a = backward.inet_backward(net, graph, send, rec, edge, g_rec, g_edge)
        b = backward.inet_backward_py(net, graph, send, rec, edge, g_rec, g_edge)
        for x, y in zip(a[:3], b[:3]):
            torch.testing.assert_close(x, y, rtol=0, atol=0)
        assert set(a[3]) == set(b[3])
        for k in a[3]:
            torch.testing.assert_close(a[3][k], b[3][k], rtol=0, atol=0)
    mlp = nlb.make_mlp([56, 64, 17], layer_norm=False).to(DEV)
    srcs = [torch.randn(2, 300, 17, device=DEV), torch.randn(2, 300, 17, device=DEV), torch.randn(2, 300, 18, device=DEV),
            torch.randn(300, 4, device=DEV)]
    go = torch.randn(2, 300, 17, device=DEV)
    a = backward.mlp_backward(mlp, srcs, None, go)
    b = backward.mlp_backward_py(mlp, srcs, None, go)
    for x, y in zip(a[0], b[0]):
        torch.testing.assert_close(x, y.contiguous(), rtol=0, atol=0)
    for k in a[2]:
        torch.testing.assert_close(a[2][k], b[2][k], rtol=0, atol=0)
