"""Pin the CPU oracle (oracle/reference_port.py) against the golden vectors generated from the reference's own source
(tests/golden/inet_cases.*.npz, tests/golden/reference_checks.*.npz).
"""
import os

import pytest
import torch

from oracle import reference_port as rp
from golden_util import load_golden_cases, load_shards

CASES = load_golden_cases()


def _run_oracle(case, dtype=torch.float32, requires_grad=False):
    t = case.t
    send = t["send"].to(dtype).clone().requires_grad_(requires_grad)
    rec = send if case.same else t["rec"].to(dtype).clone().requires_grad_(requires_grad)
    edge = t["edge"].to(dtype).clone().requires_grad_(requires_grad)
    params = {k: v.to(dtype).clone().requires_grad_(requires_grad) for k, v in case.params.items()}
    kw = dict(case.kwargs)
    ue = kw.pop("update_edges", True)
    rec_out, edge_out, aggr, msg = rp.interaction_net(
        params, t["edge_index"], send, rec, edge, propagation=case.propagation,
        update_edges=ue, return_internals=True, **kw,
    )
    return dict(send=send, rec=rec, edge=edge, params=params, rec_out=rec_out,
                edge_out=edge_out if ue else None)


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_oracle_matches_golden_forward(case):
    out = _run_oracle(case)
    # same op sequence, same dtype, CPU: differences only from summation order
    torch.testing.assert_close(out["rec_out"], case.t["rec_out"], rtol=1e-5, atol=1e-5)
    if out["edge_out"] is not None:
        torch.testing.assert_close(out["edge_out"], case.t["edge_out"], rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_oracle_fp64_close_to_golden(case):
    out = _run_oracle(case, torch.float64)
    torch.testing.assert_close(out["rec_out"].float(), case.t["rec_out"], rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_oracle_matches_golden_backward(case):
    out = _run_oracle(case, requires_grad=True)
    loss = (out["rec_out"] * case.t["w_rec"]).sum()
    if out["edge_out"] is not None:
        loss = loss + (out["edge_out"] * case.t["w_edge"]).sum()
    loss.backward()
    torch.testing.assert_close(out["send"].grad, case.t["g_send"] , rtol=1e-4, atol=1e-4)
    if not case.same:
        torch.testing.assert_close(out["rec"].grad, case.t["g_rec"], rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(out["edge"].grad, case.t["g_edge"], rtol=1e-4, atol=1e-4)
    for k, g in case.gparams.items():
        torch.testing.assert_close(out["params"][k].grad, g, rtol=1e-4, atol=1e-4, msg=lambda m: f"{k}: {m}")


REFCHECKS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_checks")


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_oracle_matches_reference_source_random(seed):
    """Fresh random graphs / weights, reference source vs oracle, fp32 CPU: the reference's outputs on these inputs are
    stored in tests/golden/reference_checks.*.npz (oracle/gen_golden_refchecks.py)."""
    blob = load_shards(REFCHECKS)
    ran = 0
    for cls, prop in (("InteractionNet", False), ("PropagationNet", True)):
        for aggr in ("sum", "mean"):
            pre = f"oracle_random/s{seed}/{cls}_{aggr}/"
            t = {k[len(pre):]: torch.from_numpy(blob[k]) for k in blob.files if k.startswith(pre)}
            params = {k[6:]: v for k, v in t.items() if k.startswith("param/")}
            r_o, e_o = rp.interaction_net(params, t["ei"], t["send"], t["rec"], t["edge"], aggr=aggr, propagation=prop)
            torch.testing.assert_close(r_o, t["rec_out"], rtol=1e-5, atol=1e-5)
            torch.testing.assert_close(e_o, t["edge_out"], rtol=1e-5, atol=1e-5)
            ran += 1
    assert ran == 4
