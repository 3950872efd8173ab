"""The H = 64 node-update kernel (launch labels tc_rowmlp_kernel for the node-update form of the row MLP,
tc_node_proj_kernel, tc_node_out_kernel) stages the next item's rows while the current item computes.  These cases cover
what only such a pipeline can get wrong, at row counts chosen against the SM count (the launcher runs one CTA per SM, two
items of 64 rows at a time): one item, two, SMs + 1 and 2 SMs + 1 items, many items, a last item shorter than 64 rows,
a receiver input shared by the batch (stride 0) or batched, all three epilogues, and B = 1 against B > 1.

Each case is checked against the fp64 oracle with TF32 operands (1e-2 absolute, DESIGN §2), and each batch row bit for
bit against that sample run alone (the item-to-CTA assignment differs between the two, so a stale staging buffer would
show).  The two epilogues that go past the node update are also checked bit for bit against launches that do the same
arithmetic on the same TF32 operands: tc_node_proj_kernel's node rows against the plain node update and its projections
against tc_rowlinear_kernel's (through the next layer's outputs), tc_node_out_kernel against the node update followed by
the row MLP with the step epilogue.
"""
import pytest
import torch

import neural_lam_b200 as nlb
from neural_lam_b200 import _lib, ops
from neural_lam_b200.networks import make_mlp
from oracle import reference_port as rp

pytestmark = pytest.mark.gpu
DEV = "cuda"
ABS_TOL = 1e-2


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _items(name):
    """(rows, B) of a named item count: items = ceil(rows / 64) * B"""
    s = _sms()
    return {"one_partial": (40, 1), "two": (128, 1), "sms_plus_1_partial": (64 * s + 17, 1),
            "two_sms_plus_1_partial": (64 * (2 * s + 1) - 30, 1), "many_b5": (64 * 50 + 33, 5), "one_each_b3": (64, 3)}[name]


ITEMS = ["one_partial", "two", "sms_plus_1_partial", "two_sms_plus_1_partial", "many_b5", "one_each_b3"]


def _rand_params(module, seed):
    """weights U(-1, 1) / sqrt(fan_in); biases and LayerNorm parameters: their init + 0.1 N(0, 1)"""
    gen = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p in module.parameters():
            if p.dim() == 2:
                p.copy_((torch.rand(p.shape, generator=gen) * 2 - 1) / p.shape[1] ** 0.5)
            else:
                p.add_(0.1 * torch.randn(p.shape, generator=gen))
    return module


def _inputs(shapes, seed):
    gen = torch.Generator().manual_seed(seed)
    return [torch.randn(sh, generator=gen) for sh in shapes]


def _bit_exact(name, got, want):
    assert got.shape == want.shape, (name, got.shape, want.shape)
    bad = got != want
    if bad.any():
        err = (got - want).abs().max().item()
        raise AssertionError(f"{name}: {int(bad.sum())} of {got.numel()} elements differ (max {err:.3e})")


def _close(name, got, want):
    err = (got.detach().double().cpu() - want).abs().max().item()
    assert err <= ABS_TOL, f"{name}: max |got - fp64 oracle| {err:.3e} > {ABS_TOL}"


def _rows_b(b, *ts):
    return [t[b:b + 1] if t.shape[0] > 1 else t for t in ts]


@pytest.mark.parametrize("shared_rec", [False, True], ids=["batched_rec", "shared_rec"])
@pytest.mark.parametrize("items", ITEMS)
def test_node_update_rowmlp(items, shared_rec):
    """POST_NONE: out = rec + node_mlp([rec | aggr]) through ops.rowmlp (the g2m and last m2m node updates)"""
    N, B = _items(items)
    m = _rand_params(make_mlp([128, 64, 64], layer_norm=True), 1)
    rec, aggr = _inputs([(1 if shared_rec else B, N, 64), (B, N, 64)], 2)
    md, rd, ad = m.to(DEV), rec.to(DEV).expand(B, -1, -1), aggr.to(DEV)

    def run(r, a):
        return (ops.rowmlp(md, [r, a], res=r, flags=_lib.MATH_TF32),)

    with torch.no_grad(), ops.profile_launches() as prof:
        out = run(rd, ad)[0]
    assert prof.names() == ["tc_rowmlp_kernel"], prof.names()
    p64 = {f"m.{k}": v.detach().cpu().double() for k, v in m.state_dict().items()}
    r64 = rec.double().expand(B, -1, -1)
    with rp.tf32_matmul(mode="rna"):
        want = r64 + rp.mlp(torch.cat([r64, aggr.double()], -1), p64, "m")
    _close("out", out, want)
    if B > 1:
        for b in (0, B - 1):
            with torch.no_grad():
                one = run(*_rows_b(b, rd, ad))[0]
            _bit_exact(f"batch row {b} vs alone", out[b:b + 1], one)


@pytest.mark.parametrize("items", ["one_partial", "sms_plus_1_partial", "many_b5"])
def test_node_update_residual_second_source(items):
    """the residual is the second source (PropagationNet's form: out = aggr + node_mlp([rec | aggr]))"""
    N, B = _items(items)
    m = _rand_params(make_mlp([128, 64, 64], layer_norm=True), 3)
    rec, aggr = _inputs([(B, N, 64), (B, N, 64)], 4)
    md, rd, ad = m.to(DEV), rec.to(DEV), aggr.to(DEV)

    def run(r, a):
        return ops.rowmlp(md, [r, a], res=a, flags=_lib.MATH_TF32)

    with torch.no_grad(), ops.profile_launches() as prof:
        out = run(rd, ad)
    assert prof.names() == ["tc_rowmlp_kernel"], prof.names()
    p64 = {f"m.{k}": v.detach().cpu().double() for k, v in m.state_dict().items()}
    with rp.tf32_matmul(mode="rna"):
        want = aggr.double() + rp.mlp(torch.cat([rec.double(), aggr.double()], -1), p64, "m")
    _close("out", out, want)
    if B > 1:
        for b in (0, B - 1):
            with torch.no_grad():
                one = run(*_rows_b(b, rd, ad))
            _bit_exact(f"batch row {b} vs alone", out[b:b + 1], one)


def _graph(n, deg, seed):
    g = torch.Generator().manual_seed(seed)
    ei = torch.stack([torch.randint(0, n, (n * deg,), generator=g), torch.randint(0, n, (n * deg,), generator=g)])
    ei[1, -1] = n - 1
    return ei[:, torch.sort(ei[1], stable=True).indices]


@pytest.mark.parametrize("items", ["one_partial", "two", "sms_plus_1_partial", "two_sms_plus_1_partial", "many_b5"])
def test_node_proj(items):
    """POST_PROJ: layer 1's node update + layer 2's node projections P_s, P_r (tc_node_proj_kernel).  The chained path
    takes dense batched node rows and a graph with E >= 2.5 (n_send + n_rec) edges (nlam_inet_chain_supported): in-degree 6.
    Layer 1's node rows equal the unchained call's; layer 2 with edge output reads the chained projections (rule 2 of the
    edge path) and its outputs equal those of layer 2 computing its own projections (tc_rowlinear_kernel)."""
    N, B = _items(items)
    ei = _graph(N, 6, 5)
    l1 = _rand_params(nlb.InteractionNet(ei, 64, math="tf32"), 6)
    l2 = _rand_params(nlb.InteractionNet(ei, 64, math="tf32"), 7)
    x, e = _inputs([(B, N, 64), (B, 6 * N, 64)], 8)
    l1d, l2d = l1.to(DEV), l2.to(DEV)
    g = l1d._graph(torch.device(DEV, torch.cuda.current_device()))
    xd, ed = x.to(DEV), e.to(DEV)

    def run(xx, ee):
        rec, e1, _, proj = ops.inet_fwd(g, l1d.edge_mlp, l1d.aggr_mlp, xx, xx, ee, True, l1d._flags(),
                                        next_edge_seq=l2d.edge_mlp)
        return rec, e1, proj

    with torch.no_grad():
        with ops.profile_launches() as prof:
            rec, e1, proj = run(xd, ed)
        assert prof.names() == ["tc_rowlinear_kernel", "tc_edge3_kernel", "tc_node_proj_kernel"], prof.names()
        plain = ops.inet_fwd(g, l1d.edge_mlp, l1d.aggr_mlp, xd, xd, ed, True, l1d._flags())[0]
        _bit_exact("out vs the unchained node update", rec, plain)
        with ops.profile_launches() as prof:
            chained = ops.inet_fwd(g, l2d.edge_mlp, l2d.aggr_mlp, rec, rec, e1, True, l2d._flags(), proj_in=proj)
        assert prof.names() == ["tc_edge3_kernel", "tc_rowmlp_kernel"], prof.names()
        with ops.profile_launches() as prof:
            own = ops.inet_fwd(g, l2d.edge_mlp, l2d.aggr_mlp, rec, rec, e1, True, l2d._flags())
        assert prof.names() == ["tc_rowlinear_kernel", "tc_edge3_kernel", "tc_rowmlp_kernel"], prof.names()
    _bit_exact("layer 2 out on chained projections vs its own", chained[0], own[0])
    _bit_exact("layer 2 edge out on chained projections vs its own", chained[1], own[1])
    p1 = {k: v.detach().cpu().double() for k, v in l1.state_dict().items()}
    w = l2.edge_mlp[0].weight.detach().cpu().double()
    b1 = l2.edge_mlp[0].bias.detach().cpu().double()
    x64 = x.double()
    with rp.tf32_matmul(mode="rna"):
        r1, _ = rp.interaction_net(p1, ei, x64, x64, e.double())
        ps, pr = r1 @ w[:, 64:128].T, r1 @ w[:, 128:].T + b1
    _close("out", rec, r1)
    _close("P_s", proj[0], ps)
    _close("P_r", proj[1], pr)
    if B > 1:
        for b in (0, B - 1):
            with torch.no_grad():
                one, _, one_proj = run(*_rows_b(b, xd, ed))
            _bit_exact(f"batch row {b} vs alone", rec[b:b + 1], one)
            _bit_exact(f"batch row {b} P_s, P_r vs alone", proj[:, b:b + 1], one_proj)


@pytest.mark.parametrize("shared_rec", [False, True], ids=["batched_rec", "shared_rec"])
@pytest.mark.parametrize("items", ["one_partial", "two", "two_sms_plus_1_partial", "many_b5", "one_each_b3"])
def test_node_out_step(items, shared_rec):
    """POST_OUTMLP: node update + output_map + forecast-step epilogue with a boundary mix (tc_node_out_kernel).  It equals,
    bit for bit, the node update (tc_node_kernel's POST_NONE) followed by output_map with the step epilogue in
    fused_mlp_kernel: both round the updated rows to TF32 to nearest as the operand of the same GEMMs in the same K order,
    with the same bias, SiLU and step-epilogue code."""
    N, B = _items(items)
    D = 17
    node = _rand_params(make_mlp([128, 64, 64], layer_norm=True), 9)
    out_map = _rand_params(make_mlp([64, 64, D], layer_norm=False), 10)
    rec, aggr, prev, bnd = _inputs([(1 if shared_rec else B, N, 64), (B, N, 64), (B, N, D), (B, N, D)], 11)
    gen = torch.Generator().manual_seed(12)
    std, mean = torch.rand(D, generator=gen) + 0.5, torch.randn(D, generator=gen)
    mask = (torch.rand(N, 1, generator=gen) < 0.3).float()
    nd, od = node.to(DEV), out_map.to(DEV)
    rd, ad, pd, bd = rec.to(DEV).expand(B, -1, -1), aggr.to(DEV), prev.to(DEV), bnd.to(DEV)
    sd, md, kd = std.to(DEV), mean.to(DEV), mask.to(DEV)

    def run(r, a, p, bb):
        got = ops.node_update_step(nd, od, r, a, p, bb, kd, sd, md)
        assert got is not None, "ops.node_update_step declined the call"
        return got

    with torch.no_grad():
        with ops.profile_launches() as prof:
            new = run(rd, ad, pd, bd)
        assert prof.names() == ["tc_node_out_kernel"], prof.names()
        with ops.profile_launches() as prof:
            grid = ops.rowmlp(nd, [rd, ad], res=rd, flags=_lib.MATH_TF32)
            two = ops.rowmlp_step(od, grid, pd, bd, kd, sd, md)
        assert two is not None, "ops.rowmlp_step declined the call"
        assert prof.names() == ["tc_rowmlp_kernel", "tc_rowmlp_kernel"], prof.names()
    _bit_exact("new state vs node update + output_map step", new, two)
    pn = {f"m.{k}": v.detach().cpu().double() for k, v in node.state_dict().items()}
    po = {f"m.{k}": v.detach().cpu().double() for k, v in out_map.state_dict().items()}
    r64 = rec.double().expand(B, -1, -1)
    with rp.tf32_matmul(mode="rna"):
        grid = r64 + rp.mlp(torch.cat([r64, aggr.double()], -1), pn, "m")
        step = prev.double() + rp.mlp(grid, po, "m", layer_norm=False) * std.double() + mean.double()
    want = mask.double() * bnd.double() + (1 - mask.double()) * step
    _close("new state", new, want)
    if B > 1:
        for b in (0, B - 1):
            with torch.no_grad():
                one = run(*_rows_b(b, rd, ad, pd, bd))
            _bit_exact(f"batch row {b} vs alone", new[b:b + 1], one)
