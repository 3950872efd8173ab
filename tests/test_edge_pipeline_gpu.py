"""The split-form edge kernel (launch labels tc_edge3_kernel, tc_edge_rmw_kernel, tc_edge_bcast_kernel) stages the next
CSR tile's edge rows, rowptr entries and gathered node projections while the current tile computes.  These cases cover
what only such a pipeline can get wrong, on synthetic graphs whose tile count is chosen against the SM count (the
launcher runs one CTA per SM): a CTA with one, two, an odd number and many tiles, fewer tiles than SMs, receivers of
in-degree 0 and 128, and a last tile shorter than 128 edges.

Each case is checked against the fp64 oracle (1e-2 absolute, DESIGN §2) and bit for bit twice: the in-place call equals
the out-of-place call (a staging buffer read after its rows were overwritten would differ), and each row of a B = 3 call
equals that sample run alone (the tile-to-CTA assignment differs between the two, so stale staging would show).
"""
import pytest
import torch

import neural_lam_b200 as nlb
from neural_lam_b200 import ops
from oracle import reference_port as rp

pytestmark = pytest.mark.gpu
DEV = "cuda"
ABS_TOL = 1e-2
TILE = 128  # edges and receivers per tile at most (graph.cu)

# in-degree runs that each fill exactly one tile (128 edges, first receiver of nonzero degree), so a run always starts a
# new tile: 16 x 8; one receiver of in-degree 128; in-degree 0 receivers between two others; a ragged mix
UNITS = [[8] * 16, [128], [1] + [0] * 100 + [127], [3, 0, 17, 9, 0, 0, 31, 1, 64, 3]]
SHORT = [40, 0, 50, 0, 0, 3]  # the last tile: 93 edges, with receivers of in-degree 0


def _n_tiles(deg):
    """the tile packing of nlam_graph_create: whole receivers, <= 128 edges and <= 128 receivers per tile"""
    ptr = [0]
    for d in deg:
        ptr.append(ptr[-1] + d)
    r, n = 0, 0
    while r < len(deg):
        r0 = r
        while r < len(deg) and r - r0 < TILE and ptr[r + 1] - ptr[r0] <= TILE:
            r += 1
        n += 1
    return n


def _graph(n_tiles, ns, seed):
    """receiver-sorted edge_index with exactly n_tiles tiles (CSR order = given order)"""
    deg = [d for i in range(n_tiles - 1) for d in UNITS[i % len(UNITS)]] + SHORT
    assert _n_tiles(deg) == n_tiles
    dst = torch.repeat_interleave(torch.arange(len(deg)), torch.tensor(deg))
    src = torch.randint(0, ns, (dst.numel(),), generator=torch.Generator().manual_seed(seed))
    src[0] = ns - 1
    return torch.stack([src, dst]), len(deg)


def _net(ei, aggr, seed):
    torch.manual_seed(seed)
    net = nlb.InteractionNet(ei, 64, update_edges=True, aggr=aggr, math="tf32")
    with torch.no_grad():
        for p in net.parameters():
            if p.dim() == 1:
                p.add_(0.1 * torch.randn_like(p))
    return net


def _call(net, g, send, rec, edge, mode):
    """one ops.inet_fwd call; mode: out (out-of-place edge output), inplace, none (no edge output)"""
    e_in = edge.clone() if mode == "inplace" else edge
    with torch.no_grad(), ops.profile_launches() as prof:
        r, e, a = ops.inet_fwd(g, net.edge_mlp, net.aggr_mlp, send, rec, e_in, mode != "none", net._flags(), want_aggr=True,
                               edge_inplace=mode == "inplace")
    torch.cuda.synchronize()
    if mode == "inplace":
        assert e.data_ptr() == e_in.data_ptr()
    return r, e, a, prof.names()


def _n_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


TILE_COUNTS = {
    "one": lambda n: 1,
    "two": lambda n: 2,
    "sms_plus_1": lambda n: n + 1,         # one CTA gets two tiles, the others one
    "odd_2sms_plus_1": lambda n: 2 * n + 1,
    "many": lambda n: 600,
}
CASES = [("one", "sum"), ("two", "mean"), ("sms_plus_1", "sum"), ("odd_2sms_plus_1", "mean"), ("many", "sum"),
         ("many", "mean")]


@pytest.mark.parametrize("tiles,aggr", CASES, ids=[f"{t}_{a}" for t, a in CASES])
def test_split_edge_pipeline(tiles, aggr):
    n_tiles = TILE_COUNTS[tiles](_n_sms())
    ns, B = 16, 3
    ei, nr = _graph(n_tiles, ns, 1)
    ne = ei.shape[1]
    net = _net(ei, aggr, 2)
    gen = torch.Generator().manual_seed(3)
    send, rec, edge = (torch.randn(B, n, 64, generator=gen) for n in (ns, nr, ne))
    want = rp.interaction_net({k: v.double() for k, v in net.state_dict().items()}, ei, send.double(), rec.double(),
                              edge.double(), aggr=aggr, update_edges=True)
    net = net.to(DEV)
    g = net._graph(torch.device(DEV, torch.cuda.current_device()))
    s, r, e = send.to(DEV), rec.to(DEV), edge.to(DEV)

    runs = {}
    for mode, label in (("out", "tc_edge3_kernel"), ("inplace", "tc_edge_rmw_kernel"), ("none", "tc_edge_rmw_kernel")):
        runs[mode] = _call(net, g, s, r, e, mode)
        names = runs[mode][3]
        assert label in names and "tc_edge_kernel" not in names, (mode, names)
    rec_o, edge_o, aggr_o, _ = runs["out"]
    err = max((rec_o.double().cpu() - want[0]).abs().max().item(), (edge_o.double().cpu() - want[1]).abs().max().item())
    assert err <= ABS_TOL, err
    # in place = out of place, bit for bit; no edge output leaves the aggregate as it is
    for mode in ("inplace", "none"):
        rec_m, edge_m, aggr_m, _ = runs[mode]
        assert torch.equal(aggr_m, aggr_o) and torch.equal(rec_m, rec_o), mode
        assert mode == "none" or torch.equal(edge_m, edge_o)
    # receivers of in-degree 0 aggregate exactly 0
    zero = torch.tensor([d == 0 for d in torch.bincount(ei[1], minlength=nr).tolist()], device=DEV)
    assert zero.any() and torch.count_nonzero(aggr_o[:, zero]).item() == 0
    # each batch row equals that sample run alone
    for b in range(B):
        for mode in ("out", "inplace"):
            rec_1, edge_1, aggr_1, names = _call(net, g, s[b:b + 1], r[b:b + 1], e[b:b + 1], mode)
            assert ("tc_edge3_kernel" if mode == "out" else "tc_edge_rmw_kernel") in names, names
            assert torch.equal(aggr_1[0], aggr_o[b]) and torch.equal(edge_1[0], edge_o[b]) and torch.equal(rec_1[0], rec_o[b]), (
                mode, b)


@pytest.mark.parametrize("tiles", ["one", "sms_plus_1"])
def test_split_edge_pipeline_batch_broadcast(tiles):
    """grid -> mesh shape: edge features and receivers shared by the batch (batch stride 0), many senders, no edge
    update -> tc_edge_bcast_kernel at B = 3 and at B = 1"""
    n_tiles = TILE_COUNTS[tiles](_n_sms())
    B = 3
    ei, nr = _graph(n_tiles, 1, 4)
    ne = ei.shape[1]
    ns = ne  # senders outnumber edges / 2.5: the batch-broadcast path
    ei[0] = torch.randint(0, ns, (ne,), generator=torch.Generator().manual_seed(5))
    torch.manual_seed(6)
    net = nlb.InteractionNet(ei, 64, update_edges=False, aggr="sum", math="tf32")
    with torch.no_grad():
        for p in net.parameters():
            if p.dim() == 1:
                p.add_(0.1 * torch.randn_like(p))
    gen = torch.Generator().manual_seed(7)
    send, rec, edge = torch.randn(B, ns, 64, generator=gen), torch.randn(1, nr, 64, generator=gen), torch.randn(1, ne, 64, generator=gen)
    want = rp.interaction_net({k: v.double() for k, v in net.state_dict().items()}, ei, send.double(),
                              rec.double().expand(B, -1, -1), edge.double().expand(B, -1, -1), update_edges=False)
    net = net.to(DEV)
    s, r, e = send.to(DEV), rec.to(DEV), edge.to(DEV)
    with torch.no_grad(), ops.profile_launches() as prof:
        got = net(s, r.expand(B, -1, -1), e.expand(B, -1, -1))
    assert "tc_edge_bcast_kernel" in prof.names(), prof.names()
    assert (got.double().cpu() - want).abs().max().item() <= ABS_TOL
    for b in range(B):
        with torch.no_grad(), ops.profile_launches() as prof:
            one = net(s[b:b + 1], r, e)
        assert "tc_edge_bcast_kernel" in prof.names(), prof.names()
        assert torch.equal(one[0], got[b]), b
