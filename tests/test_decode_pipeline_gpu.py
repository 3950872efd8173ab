"""Scheduling of the warp-specialized mesh -> grid decoder (tc_decode_kernel): a load warp group feeds two compute warp
groups through a ring of shared-memory units (receiver rows, then one unit per 64-edge sub-tile), one item ahead.

Shapes that exercise what the ring adds: fewer items than compute warp groups, item counts that wrap the ring an odd
number of times, a partial last receiver block that is not a warp group's first item, odd B and B = 1, mean and sum, with
and without boundary, receivers batched and batch-broadcast.  In each case every batch element decoded alone equals its row
of the batched call bit for bit, and the output meets test_decode_gpu.py's fp64-oracle bound.
"""
import pytest
import torch

from test_decode_gpu import DECODER, _check_case, _fused, _multi_item_shape, _setup
from test_tc_kernels import _ell_graph

pytestmark = pytest.mark.gpu
NS = 300

CASES = [
    # name, in-degree, B, aggregation, boundary, batch-broadcast inputs, receivers (None: several items per warp group,
    # a partial last round and a partial last block)
    ("d1_one_item_b1", 1, 1, "sum", True, (), 50),
    ("d1_b5_mean_no_bnd", 1, 5, "mean", False, (), None),
    ("d2_b3_sum_bcast_rec", 2, 3, "sum", True, ("rec",), None),
    ("d2_two_items_b2_mean", 2, 2, "mean", True, (), 70),
    ("d4_b1_mean", 4, 1, "mean", True, (), 64 * 7 + 5),
    ("d4_b7_sum_no_bnd_bcast_rec", 4, 7, "sum", False, ("rec",), None),
    ("d8_b5_sum", 8, 5, "sum", True, (), None),
    ("d8_b1_one_item_mean_no_bnd", 8, 1, "mean", False, (), 33),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_decode_pipeline_per_sample_equals_batch(case):
    name, d, B, aggr, boundary, bcast, nr = case
    if nr is None:
        nr, n_items, groups = _multi_item_shape(B)
        assert n_items > groups and nr % 64 != 0
    c = _setup(_ell_graph(NS, nr, d, 6), NS, nr, B, aggr=aggr, boundary=boundary, bcast=bcast)
    _check_case(name, c)
    got, names = _fused(c)
    assert names == DECODER, names
    for b in range(B):
        one = dict(c, B=1, **{k: c[k][b:b + 1] for k in ("send", "rec", "prev") + (("bnd",) if boundary else ())})
        alone, _ = _fused(one)
        assert torch.equal(alone[0], got[b]), f"batch element {b} alone differs: {(alone[0] - got[b]).abs().max().item():.3e}"
