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


@pytest.mark.parametrize("mode", ["rna", "rz"])
def test_round_tf32_fp64_matches_fp32(mode):
    """fp64 rounding of fp32-representable values equals the fp32 bit rounding, in both modes, at both signs, exact
    ties (rna: away from zero) and carries into the exponent"""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(100000, generator=g) * torch.exp2(torch.randint(-30, 30, (100000,), generator=g).float())
    base = torch.tensor([1.0, 1.5, 0.375, 3.0, 2.0 - 2.0 ** -10])  # TF32 values; the last tie carries to 2
    tie = base + torch.ldexp(torch.ones(5), torch.frexp(base)[1] - 12)  # exactly half a TF32 ulp above base
    x = torch.cat([x, tie, -tie, torch.tensor([0.0, -0.0])])
    got = rp.round_tf32(x.double(), mode)
    torch.testing.assert_close(got, rp.round_tf32(x, mode).double(), rtol=0, atol=0)
    # a TF32 value: at most 11 significant bits
    m, _ = torch.frexp(got)
    assert torch.equal(m * 2048, torch.round(m * 2048))
    err = (got - x.double()).abs() / x.double().abs().clamp_min(1e-300)
    assert err.max().item() <= (2.0 ** -11 if mode == "rna" else 2.0 ** -10)
    if mode == "rna":
        assert torch.equal(rp.round_tf32(tie.double(), mode), (base + 2 * (tie - base)).double())
    else:
        assert (got.abs() <= x.double().abs()).all()


def test_round_tf32_fp64_rounds_its_own_value():
    """fp64 input is rounded directly, not through fp32 first: 1 + 2^-11 + 2^-40 is above the tie, its fp32 value
    (1 + 2^-11) is the tie itself (rounded away from zero either way); 1 + 2^-11 - 2^-40 is below the tie, its fp32 value
    is the tie (rounded up), while the correct result is 1"""
    below = torch.tensor([1 + 2.0 ** -11 - 2.0 ** -40], dtype=torch.float64)
    assert rp.round_tf32(below).item() == 1.0
    assert rp.round_tf32(below.float()).item() == 1 + 2.0 ** -10
    assert rp.round_tf32(-below).item() == -1.0
    assert rp.round_tf32(torch.tensor([1 + 2.0 ** -10 - 2.0 ** -40], dtype=torch.float64), "rz").item() == 1.0


def test_tf32_matmul_modes_in_fp64():
    """tf32_matmul rounds fp64 operands too (previously only fp32); fp32 results are unchanged by the mode argument's
    default"""
    g = torch.Generator().manual_seed(1)
    x = torch.randn(50, 8, generator=g)
    p = {"m.0.weight": torch.randn(8, 8, generator=g), "m.0.bias": torch.randn(8, generator=g),
         "m.2.weight": torch.randn(4, 8, generator=g), "m.2.bias": torch.randn(4, generator=g)}
    p64 = {k: v.double() for k, v in p.items()}
    exact = rp.mlp(x.double(), p64, "m", layer_norm=False)
    with rp.tf32_matmul():
        f32 = rp.mlp(x, p, "m", layer_norm=False)
        rna = rp.mlp(x.double(), p64, "m", layer_norm=False)
    with rp.tf32_matmul(mode="rz"):
        rz = rp.mlp(x.double(), p64, "m", layer_norm=False)
    h = rp.round_tf32(x) @ rp.round_tf32(p["m.0.weight"]).t() + p["m.0.bias"]
    h = h * torch.sigmoid(h)
    torch.testing.assert_close(f32, rp.round_tf32(h) @ rp.round_tf32(p["m.2.weight"]).t() + p["m.2.bias"], rtol=0, atol=0)
    assert not torch.equal(rna, exact) and not torch.equal(rz, rna)
    assert (rna - exact).abs().max() < (rz - exact).abs().max()
    assert torch.equal(rp.mlp(x.double(), p64, "m", layer_norm=False), exact)  # the context is left
