"""The H = 128 / 256 path (generic wgmma Linear ``tc_linear_kernel<N>``, CSR segment sum, packed row MLPs, the
hand-written backward) at the REAL sizes of the benchmark's configs 3 and 4, against an fp64 oracle run on the GPU.

  * config 4: 1024 x 1024 grid (1 048 576 grid nodes, 59 049 mesh nodes, 527 096 m2m / 1 475 712 g2m / 4 194 304 m2g
    edges), GraphLAM H = 256, 4 processor layers, B = 1.  One m2g edge tensor holds 1.07e9 floats; at B = 2 the m2g
    hidden and message workspaces hold exactly 2^31 floats each.
  * config 3: MEPS 268 x 238 grid with a three-level mesh (6 561 / 729 / 81 nodes), HiLAM H = 128, 6 processor layers,
    B = 8 (B = 4 for the training step, as the benchmark's training leg).

Ground truth: ``oracle/reference_port.py`` in fp64 on the device.  Its unchunked InteractionNet does not fit at config 4
(m2g's ``cat([e | x_s | x_r])`` alone is 25.8 GB in fp64), so ``chunked_oracle()`` installs an edge-chunked
``interaction_net`` and a row-chunked ``mlp`` over the module globals that ``graph_model_forward`` looks up at call time;
``test_chunked_oracle_equals_oracle`` (CPU, no GPU needed) pins them to the originals.  The reference's own GPU
configuration is the same oracle in fp32 on the device with ``torch.backends.cuda.matmul.allow_tf32 = True``
(TF32 cuBLAS matmuls, as the reference enables whenever CUDA is available); its error is printed beside ours.

Bounds: layers as tests/test_tc_kernels.py (|err| <= max(3 x reference-TF32 error, 4e-3) and <= 1e-2 for every element
of every output); forecast steps as tests/test_real_size.py (max(3 x reference-TF32 error, 1e-2) per AR step);
gradients as test_backward_coverage_gpu.py::test_training_step_vs_fp64_autograd (3e-2 max|g_ref| + 2e-4 per tensor).
Past 2^31 elements the generic Linear, the segment sum and the row gather are checked bit for bit on exact operands.

Each GPU test checks the free device memory it needs first and skips (with both numbers) below it; the peak
``torch.cuda.max_memory_allocated`` and the wall time of each test are printed (run with -s).  Peaks of the memory
allocated through torch (the library's graph tables and row-MLP workspaces come on top), measured on one H100 80GB HBM3
(700 W power limit); the errors are in DESIGN.md section 2:

    layer c4_g2m 9.6 GB, c4_m2m 5.0 GB, c4_m2g_b1 20.5 GB, c4_m2g_b2 30.4 GB, c3_g2m 7.1 GB, c3_m2m_l0 3.8 GB,
          c3_m2g 9.7 GB, the other config 3 layers <= 0.6 GB
    generic Linear past 2^31 12.8 GB, segment sum past 2^31 15.3 GB, row gather past 2^31 11.2 GB
    config 3 rollout 11.3 GB, config 4 step 23.6 GB, config 3 training step 24.4 GB
"""
import contextlib
import ctypes
import functools
import time

import pytest
import torch

import neural_lam_b200 as nlb
from neural_lam_b200 import _lib, models, ops, synthetic
from oracle import reference_port as rp
from test_models import _oracle_graph

DEV = "cuda"
GB = 1 << 30
ABS_TOL = 1e-2

# ------------------------------------------------------------------------------------------------ 0. chunked oracle
_ORIG_INET = rp.interaction_net
_ORIG_MLP = rp.mlp
EDGE_CHUNK = 1 << 17   # edges per chunk of the chunked InteractionNet
ROW_CHUNK = 1 << 17    # rows per chunk of the chunked MLP and node update


def chunked_mlp(x, params, prefix, hidden_layers=1, layer_norm=True, eps=1e-5, row_chunk=ROW_CHUNK):
    """``rp.mlp`` over row chunks of ``x`` (dim -2), written into one preallocated output."""
    n = x.shape[-2]
    if n <= row_chunk:
        return _ORIG_MLP(x, params, prefix, hidden_layers, layer_norm, eps)
    n_out = params[f"{prefix}.{2 * hidden_layers}.weight"].shape[0]
    out = x.new_empty(x.shape[:-1] + (n_out,))
    for a in range(0, n, row_chunk):
        out[..., a:a + row_chunk, :] = _ORIG_MLP(x[..., a:a + row_chunk, :], params, prefix, hidden_layers, layer_norm, eps)
    return out


def chunked_interaction_net(params, edge_index, send_rep, rec_rep, edge_rep, prefix="", aggr="sum", update_edges=True,
                            propagation=False, hidden_layers=1, edge_chunk_sizes=None, aggr_chunk_sizes=None,
                            return_internals=False, edge_chunk=EDGE_CHUNK, row_chunk=ROW_CHUNK):
    """``rp.interaction_net`` with the edges in chunks: each chunk's messages are summed into one receiver accumulator
    (``index_add_``, in the messages' dtype: fp64 for the ground truth, fp32 for the reference's TF32 configuration), the
    node update runs over row chunks.  Same operations otherwise.  SplitMLPs layers and ``return_internals`` go to the
    original."""
    if edge_chunk_sizes is not None or aggr_chunk_sizes is not None or return_internals:
        return _ORIG_INET(params, edge_index, send_rep, rec_rep, edge_rep, prefix=prefix, aggr=aggr,
                          update_edges=update_edges, propagation=propagation, hidden_layers=hidden_layers,
                          edge_chunk_sizes=edge_chunk_sizes, aggr_chunk_sizes=aggr_chunk_sizes,
                          return_internals=return_internals)
    p = (prefix + ".") if prefix else ""
    if propagation:
        aggr = "mean"
    senders = edge_index[0].long()
    receivers = edge_index[1].long()
    num_rec = int(receivers.max()) + 1
    assert rec_rep.shape[-2] == num_rec
    E = senders.numel()
    H = params[f"{p}edge_mlp.{2 * hidden_layers}.weight"].shape[0]
    lead = torch.broadcast_shapes(send_rep.shape[:-2], rec_rep.shape[:-2], edge_rep.shape[:-2])
    acc = send_rep.new_zeros(lead + (num_rec, H))
    edge_out = send_rep.new_empty(lead + (E, H)) if update_edges else None
    for a in range(0, E, edge_chunk):
        s, r = senders[a:a + edge_chunk], receivers[a:a + edge_chunk]
        x_j = send_rep.index_select(send_rep.dim() - 2, s)
        x_i = rec_rep.index_select(rec_rep.dim() - 2, r)
        e = edge_rep[..., a:a + edge_chunk, :]
        msg = _ORIG_MLP(torch.cat((e, x_j, x_i), dim=-1), params, p + "edge_mlp", hidden_layers)
        if propagation:
            msg = x_j + msg
        acc.index_add_(acc.dim() - 2, r, msg)
        if update_edges:
            edge_out[..., a:a + edge_chunk, :] = e + msg
        del x_j, x_i, msg
    if aggr == "mean":
        cnt = torch.bincount(receivers, minlength=num_rec).to(acc.dtype)
        acc = acc / cnt.clamp(min=1).unsqueeze(-1)
    new_rec = acc.new_empty(lead + (num_rec, H))
    base = acc if propagation else rec_rep
    for a in range(0, num_rec, row_chunk):
        node_in = torch.cat((rec_rep[..., a:a + row_chunk, :], acc[..., a:a + row_chunk, :]), dim=-1)
        new_rec[..., a:a + row_chunk, :] = base[..., a:a + row_chunk, :] + _ORIG_MLP(node_in, params, p + "aggr_mlp",
                                                                                     hidden_layers)
    if update_edges:
        return new_rec, edge_out
    return new_rec


@contextlib.contextmanager
def chunked_oracle(edge_chunk=EDGE_CHUNK, row_chunk=ROW_CHUNK):
    """``rp.interaction_net`` / ``rp.mlp`` replaced by the chunked versions for the duration of the block."""
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(rp, "interaction_net", functools.partial(chunked_interaction_net, edge_chunk=edge_chunk, row_chunk=row_chunk))
        mp.setattr(rp, "mlp", functools.partial(chunked_mlp, row_chunk=row_chunk))
        yield


def _assert_rel(name, got, want, rel=1e-12):
    got = got if isinstance(got, tuple) else (got,)
    want = want if isinstance(want, tuple) else (want,)
    assert len(got) == len(want), name
    for g, w in zip(got, want):
        assert g.shape == w.shape and g.dtype == w.dtype == torch.float64, (name, g.shape, w.shape)
        err = (g - w).abs().max().item()
        assert err <= rel * w.abs().max().item(), f"{name}: {err:.3e} vs max |ref| {w.abs().max().item():.3e}"


PIN_CASES = [(cls, aggr, upd, B) for cls in ("InteractionNet", "PropagationNet") for aggr in ("sum", "mean")
             for upd in (True, False) for B in (1, 3)]


@pytest.mark.parametrize("cls,aggr,upd,B", PIN_CASES,
                         ids=[f"{c}-{a}-{'upd' if u else 'noupd'}-B{b}" for c, a, u, b in PIN_CASES])
def test_chunked_oracle_equals_oracle(cls, aggr, upd, B):
    """CPU, fp64: the chunked InteractionNet / PropagationNet equals the original within 1e-12 relative; chunk 64 does not
    divide E = 301, and receiver-sorted edges put one receiver's edges on both sides of a chunk boundary."""
    ns, nr, E, H, chunk = 37, 23, 301, 16, 64
    g = torch.Generator().manual_seed(7)
    ei = torch.stack([torch.randint(0, ns, (E,), generator=g), torch.randint(0, nr, (E,), generator=g)])
    ei[1, -1] = nr - 1
    ei = ei[:, torch.sort(ei[1], stable=True).indices]
    assert E % chunk != 0 and ei[1, chunk - 1] == ei[1, chunk]
    torch.manual_seed(0)
    net = getattr(nlb, cls)(ei, H, update_edges=upd, aggr=aggr)
    params = {k: v.double() for k, v in net.state_dict().items()}
    for k, v in params.items():
        if v.dim() == 1:
            v.add_(0.1 * torch.randn(v.shape, generator=g, dtype=torch.float64))
    send = torch.randn(1, ns, H, generator=g, dtype=torch.float64).expand(B, -1, -1)   # stride-0 batch
    rec = torch.randn(B, nr, H, generator=g, dtype=torch.float64)
    edge = torch.randn(1, E, H, generator=g, dtype=torch.float64).expand(B, -1, -1)
    kw = dict(aggr=aggr, update_edges=upd, propagation=cls == "PropagationNet")
    want = _ORIG_INET(params, ei, send, rec, edge, **kw)
    got = chunked_interaction_net(params, ei, send, rec, edge, edge_chunk=chunk, row_chunk=10, **kw)
    _assert_rel(f"{cls} {aggr} upd={upd} B={B}", got, want)


def test_chunked_oracle_graph_model_forward():
    """CPU, fp64: one small three-level HiLAM step through graph_model_forward, with and without the patch (chunks of
    100 edges / 64 rows: every edge set and row block of the model is cut, none evenly)."""
    spec = synthetic.make_graph_spec(30, 27, hierarchical=True, n_levels=3)
    ds = synthetic.SyntheticDatastore(spec, d_state=5, d_forcing=6, d_static=1, boundary_width=2)
    torch.manual_seed(42)
    m = models.HiLAM(ds, spec, hidden_dim=16, processor_layers=1, math="fp32")
    g = _oracle_graph(m)
    cfg = dict(model="hi_lam", hidden_layers=1, processor_layers=1, mesh_aggr="sum")
    G = m.num_grid_nodes
    gen = torch.Generator().manual_seed(3)
    prev, pprev, forc = (torch.randn(2, G, d, generator=gen, dtype=torch.float64) for d in (5, 5, 6))
    params = {k: v.double() for k, v in m.state_dict().items()}
    want = rp.graph_model_forward(params, g, cfg, prev, pprev, forc)
    with chunked_oracle(edge_chunk=100, row_chunk=64):
        assert rp.interaction_net is not _ORIG_INET and rp.mlp is not _ORIG_MLP
        got = rp.graph_model_forward(params, g, cfg, prev, pprev, forc)
    assert rp.interaction_net is _ORIG_INET and rp.mlp is _ORIG_MLP
    _assert_rel("HiLAM step", got, want)


# ------------------------------------------------------------------------------------------------ GPU helpers
@pytest.fixture(autouse=True)
def _peak_and_wall(request):
    if "gpu" not in request.keywords or not torch.cuda.is_available():
        yield
        return
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    yield
    torch.cuda.synchronize()
    print(f"\n[{request.node.name}] peak {torch.cuda.max_memory_allocated() / GB:.1f} GB allocated, "
          f"wall {time.time() - t0:.0f} s")
    torch.cuda.empty_cache()


def _need(gb):
    free, total = torch.cuda.mem_get_info()
    if free < gb * GB:
        pytest.skip(f"needs {gb} GB of free device memory; the card has {free / GB:.1f} GB free of {total / GB:.1f} GB")


@contextlib.contextmanager
def _tf32_matmuls():
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old


def _free():
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


@functools.lru_cache(maxsize=None)
def _spec(cfg_id):
    """the graph ``bench.build_model`` builds for a config, with the edge counts of its workload"""
    if cfg_id == 4:
        spec = synthetic.make_graph_spec(1024, 1024, hierarchical=False)
        assert spec["m2m_edge_index"].shape[1] == 527096 and spec["mesh_static_features"].shape[0] == 59049
        assert spec["g2m_edge_index"].shape[1] == 1475712 and spec["m2g_edge_index"].shape[1] == 4194304
    else:
        spec = synthetic.make_graph_spec(268, 238, hierarchical=True, n_levels=3)
        assert [m.shape[0] for m in spec["mesh_static_features"]] == [6561, 729, 81]
        assert [e.shape[1] for e in spec["m2m_edge_index"]] == [51520, 5512, 544]
        assert [e.shape[1] for e in spec["mesh_up_edge_index"]] == [6561, 729]
        assert [e.shape[1] for e in spec["mesh_down_edge_index"]] == [6561, 729]
        assert spec["g2m_edge_index"].shape[1] == 100656 and spec["m2g_edge_index"].shape[1] == 255136
    return spec


def _bench_model(cfg_id):
    """the model and forecaster exactly as ``bench.build_model`` builds them for --config 3 / 4 (same spec, datastore
    widths 17 / 18 / 4, boundary width 10, seed 42), on the CPU"""
    kind, H, P = ("graph_lam", 256, 4) if cfg_id == 4 else ("hi_lam", 128, 6)
    spec = _spec(cfg_id)
    ds = synthetic.SyntheticDatastore(spec, d_state=17, d_forcing=18, d_static=4, boundary_width=10)
    torch.manual_seed(42)
    m = models.MODELS[kind](ds, spec, hidden_dim=H, processor_layers=P, math="auto")
    return m, models.ARForecaster(m, ds), kind, P


def _to_dev(g, dtype=None):
    def cv(t):
        t = t.to(DEV)
        return t.to(dtype) if (dtype is not None and t.is_floating_point()) else t
    return {k: ([cv(t) for t in v] if isinstance(v, list) else cv(v)) for k, v in g.items()}


_GENERIC = ("tc_linear_kernel", "pack_rows_kernel", "segment_sum_kernel", "gather_rows_kernel", "step_epilogue_kernel")


def _assert_generic_path(names):
    assert any(n.startswith("tc_linear_kernel") for n in names), sorted(set(names))
    other = sorted({n for n in names if not n.startswith(_GENERIC)})
    assert not other, f"kernels outside the generic tensor-core path and the index kernels: {other}"


# ------------------------------------------------------------------------------------------------ 1. layers
# name, config, edge set, level, B, update_edges, free GB needed
LAYER_CASES = [
    ("c4_g2m", 4, "g2m", 0, 1, False, 14),
    ("c4_m2m", 4, "m2m", 0, 1, True, 8),
    ("c4_m2g_b1", 4, "m2g", 0, 1, False, 28),
    ("c4_m2g_b2", 4, "m2g", 0, 2, False, 40),
    ("c3_g2m", 3, "g2m", 0, 8, False, 10),
    ("c3_m2m_l0", 3, "m2m", 0, 8, True, 6),
    ("c3_m2m_l1", 3, "m2m", 1, 8, True, 4),
    ("c3_m2m_l2", 3, "m2m", 2, 8, True, 4),
    ("c3_up_l0", 3, "up", 0, 8, True, 4),
    ("c3_up_l1", 3, "up", 1, 8, True, 4),
    ("c3_down_l0", 3, "down", 0, 8, True, 4),
    ("c3_down_l1", 3, "down", 1, 8, True, 4),
    ("c3_read_down_l0", 3, "down", 0, 8, False, 4),
    ("c3_m2g", 3, "m2g", 0, 8, False, 14),
]


def _layer_graph(spec, kind, level):
    """-> (edge_index, sender rows, receiver rows, receivers batch-broadcast as in the model)"""
    mesh = spec["mesh_static_features"]
    n_mesh = [t.shape[0] for t in mesh] if isinstance(mesh, list) else [mesh.shape[0]]
    sel = (lambda v: v[level] if isinstance(v, list) else v)
    n_grid = int(spec["m2g_edge_index"][1].max()) + 1
    if kind == "g2m":
        return spec["g2m_edge_index"], n_grid, n_mesh[0], True
    if kind == "m2g":
        return spec["m2g_edge_index"], n_mesh[0], n_grid, False
    if kind == "m2m":
        return sel(spec["m2m_edge_index"]), n_mesh[level], n_mesh[level], False
    if kind == "up":
        return spec["mesh_up_edge_index"][level], n_mesh[level], n_mesh[level + 1], False
    return spec["mesh_down_edge_index"][level], n_mesh[level + 1], n_mesh[level], False


@pytest.mark.gpu
@pytest.mark.parametrize("case", LAYER_CASES, ids=[c[0] for c in LAYER_CASES])
def test_layer_at_real_call_shape(case):
    """One InteractionNet call of config 3 / 4 at its real graph, width and batch: every element of every output within
    the bound of tests/test_tc_kernels.py; the generic tensor-core Linear ran, the SIMT row MLP did not."""
    name, cfg_id, kind, level, B, upd, need = case
    _need(need)
    H = 256 if cfg_id == 4 else 128
    ei, ns, nr, bcast_rec = _layer_graph(_spec(cfg_id), kind, level)
    E = ei.shape[1]
    torch.manual_seed(0)
    net = nlb.InteractionNet(ei, H, update_edges=upd, aggr="sum", math="tf32")
    with torch.no_grad():
        for p in net.parameters():
            if p.dim() == 1:
                p.add_(0.1 * torch.randn_like(p))
    sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
    gen = torch.Generator(device=DEV).manual_seed(1)
    send = torch.randn(B, ns, H, device=DEV, generator=gen)
    rec = send if kind == "m2m" else torch.randn(1 if bcast_rec else B, nr, H, device=DEV, generator=gen)
    edge = torch.randn(1, E, H, device=DEV, generator=gen)             # static edge embedding, stride-0 batch

    def inputs(dtype):
        return [t.to(dtype).expand(B, -1, -1) for t in (send, rec, edge)]

    net = net.to(DEV)
    with torch.no_grad(), ops.profile_launches() as prof:
        got = net(*inputs(torch.float32))
    names = prof.names()
    assert any(n.startswith("tc_linear_kernel") for n in names) and not any("rowmlp_simt" in n for n in names), names
    got = [t.cpu() for t in (got if isinstance(got, tuple) else (got,))]
    del net
    _free()

    ei_d = ei.to(DEV)
    with torch.no_grad(), chunked_oracle():
        want = rp.interaction_net({k: v.to(DEV).double() for k, v in sd.items()}, ei_d, *inputs(torch.float64),
                                  update_edges=upd)
        want = want if isinstance(want, tuple) else (want,)
        errs = [(g.to(DEV).double() - w).abs().max().item() for g, w in zip(got, want)]
        with _tf32_matmuls():
            ref = rp.interaction_net({k: v.to(DEV) for k, v in sd.items()}, ei_d, *inputs(torch.float32), update_edges=upd)
        ref = ref if isinstance(ref, tuple) else (ref,)
        ref_errs = [(r.double() - w).abs().max().item() for r, w in zip(ref, want)]
    del want, ref
    for out_name, err, ref_err in zip(("rec_out", "edge_out"), errs, ref_errs):
        bound = min(max(3 * ref_err, 4e-3), ABS_TOL)
        print(f"\n{name} {out_name} (E={E}, B={B}, H={H}): err {err:.3e}, reference TF32 {ref_err:.3e}, bound {bound:.3e}")
        assert err <= ABS_TOL, (name, out_name, err)
        assert err <= max(3 * ref_err, 4e-3), (name, out_name, err, ref_err)


# ------------------------------------------------------------------------------------------------ 2. past 2^31 elements
def _fill_exact(t, gen, chunk=1 << 26):
    """fill t in place with values in {±0.25, ±0.5, ±0.75, ±1} (exact in TF32; products exact multiples of 1/16)"""
    flat = t.view(-1)
    for a in range(0, flat.numel(), chunk):
        n = min(chunk, flat.numel() - a)
        mag = torch.randint(1, 5, (n,), device=DEV, generator=gen, dtype=torch.int32).float() * 0.25
        sign = torch.randint(0, 2, (n,), device=DEV, generator=gen, dtype=torch.int32).float() * 2 - 1
        flat[a:a + n] = mag * sign
    return t


def _exact(shape, gen):
    return _fill_exact(torch.empty(shape, device=DEV), gen)


def _ptr(t):
    return None if t is None else t.data_ptr()


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _assert_equal_rows(name, got, want_fn, n_rows, chunk=1 << 18):
    """got (n_rows, H) equals want_fn(a, b) (fp64, rows a:b) bit for bit, row chunk by row chunk"""
    for a in range(0, n_rows, chunk):
        b = min(n_rows, a + chunk)
        g, w = got[a:b].double(), want_fn(a, b)
        bad = g != w
        if bad.any():
            r = int(bad.any(-1).nonzero()[0]) + a
            raise AssertionError(f"{name}: {int(bad.sum())} elements of rows {a}..{b - 1} differ (first row {r}; "
                                 f"max |err| {(g - w).abs().nan_to_num(float('inf')).max().item():.3e})")


@pytest.mark.gpu
def test_generic_linear_past_2p31_outputs_bit_exact():
    """nlam_linear with an output of 9 x 1 000 000 x 256 = 2.3e9 floats: batch-broadcast x0, a gathered addend with a
    per-batch stride (every batch element's output differs), bias and a batch-broadcast residual.  The output is
    pre-filled with NaN; every element must equal the fp64 result (exact operands: exactly one correct fp32 value)."""
    B, R, N, K, NA = 9, 1_000_000, 256, 32, 4093
    assert B * R * N > 2 ** 31 and R % 128 != 0
    _need(16)
    g = torch.Generator(device=DEV).manual_seed(11)
    x0, w, bias = _exact((R, K), g), _exact((N, K), g), _exact((N,), g)
    add = _exact((B, NA, N), g)
    idx = torch.randint(0, NA, (R,), device=DEV, generator=g, dtype=torch.int32)
    res = _exact((R, N), g)
    out = torch.full((B, R, N), float("nan"), device=DEV)
    L = _lib.lib()
    with ops.profile_launches() as prof:
        _lib.check(L.nlam_linear(_ptr(x0), 0, K, 0, None, 0, 0, _ptr(w), K, 0, 0, _ptr(bias), N, 0, None, None, 0.0,
                                 _ptr(add), _ptr(idx), NA * N, None, None, 0, None, None, 0, _ptr(res), 0, R, B,
                                 _ptr(out), None, _stream()))
    assert prof.names() == ["tc_linear_kernel<256>"], prof.names()
    w64, b64 = w.double(), bias.double()
    for b in range(B):
        _assert_equal_rows(f"batch {b}", out[b], lambda r0, r1: (x0[r0:r1].double() @ w64.t() + b64 + add[b][
            idx[r0:r1].long()].double() + res[r0:r1].double()), R)


@pytest.mark.gpu
def test_segment_sum_past_2p31_inputs_bit_exact():
    """nlam_segment_sum over an input of 3 x 3 000 000 x 256 = 2.3e9 floats (in-degree 4, rows read through a random
    permutation ``order``), sum and mean (÷ 4 is exact); output pre-filled with NaN, bit for bit against fp64."""
    B, S, D, H = 3, 750_000, 4, 256
    assert B * S * D * H > 2 ** 31
    _need(19)
    g = torch.Generator(device=DEV).manual_seed(12)
    x = _exact((B, S * D, H), g)
    order = torch.randperm(S * D, device=DEV, generator=g).to(torch.int32)
    ptr = torch.arange(0, S * D + 1, D, device=DEV, dtype=torch.int32)
    L = _lib.lib()
    for mean in (0, 1):
        out = torch.full((B, S, H), float("nan"), device=DEV)
        _lib.check(L.nlam_segment_sum(_ptr(ptr), _ptr(order), S, _ptr(x), S * D * H, _ptr(out), S * H, B, H, mean,
                                      _stream()))
        for b in range(B):
            def want(s0, s1, b=b):
                rows = order[s0 * D:s1 * D].long()
                v = x[b].index_select(0, rows).double().view(s1 - s0, D, H).sum(1)
                return v / D if mean else v
            _assert_equal_rows(f"{'mean' if mean else 'sum'} batch {b}", out[b], want, S)
        del out


@pytest.mark.gpu
def test_gather_rows_past_2p31_outputs_bit_exact():
    """nlam_gather_rows into an output of 3 x 3 000 000 x 256 = 2.3e9 floats (pre-filled with NaN), batch-dependent
    source rows: every element equals its source element."""
    B, NS, R, H = 3, 100_003, 3_000_000, 256
    assert B * R * H > 2 ** 31
    _need(15)
    g = torch.Generator(device=DEV).manual_seed(13)
    x = torch.randn(B, NS, H, device=DEV, generator=g)
    idx = torch.randint(0, NS, (R,), device=DEV, generator=g, dtype=torch.int32)
    out = torch.full((B, R, H), float("nan"), device=DEV)
    _lib.check(_lib.lib().nlam_gather_rows(_ptr(x), NS * H, _ptr(idx), R, _ptr(out), R * H, B, H, None, _stream()))
    for b in range(B):
        _assert_equal_rows(f"batch {b}", out[b], lambda r0, r1, b=b: x[b].index_select(0, idx[r0:r1].long()).double(), R)


# ------------------------------------------------------------------------------------------------ 3. forecast steps
def _rollout_errors(name, got, want64, ref32):
    ok = True
    for t in range(got.shape[1]):
        e = (got[:, t].to(DEV).double() - want64[:, t]).abs().max().item()
        r = (ref32[:, t].double() - want64[:, t]).abs().max().item()
        bound = max(3 * r, 1e-2)
        print(f"\n{name} AR step {t + 1}: err {e:.3e}, reference TF32 {r:.3e}, bound {bound:.3e}")
        ok &= e <= bound
    assert ok, f"{name}: an AR step exceeds its bound (see the printed table)"
    assert torch.isfinite(got).all()


def _oracle_rollouts(params, g, cfg, init, forc, bnd):
    """(fp64 oracle, the reference's TF32 configuration) on the device, chunked"""
    with torch.no_grad(), chunked_oracle():
        want = rp.ar_rollout({k: v.to(DEV).double() for k, v in params.items()}, _to_dev(g, torch.float64), cfg,
                             init.to(DEV).double(), forc.to(DEV).double(), bnd.to(DEV).double())
        with _tf32_matmuls():
            ref = rp.ar_rollout({k: v.to(DEV) for k, v in params.items()}, _to_dev(g), cfg, init.to(DEV), forc.to(DEV),
                                bnd.to(DEV))
    return want, ref


@pytest.mark.gpu
def test_config3_rollout_real_size():
    """bench --config 3's model (three-level HiLAM H = 128, 6 processor layers) at B = 8: a 2-step rollout_graphed
    against the fp64 oracle; the eager forward equals the replay; only generic-path and index kernels run."""
    _need(16)
    B, T = 8, 2
    m, fc, kind, P = _bench_model(3)
    g = _oracle_graph(m, fc)
    params = {f"predictor.{k}": v.detach().clone() for k, v in m.state_dict().items()}
    G = m.num_grid_nodes
    gen = torch.Generator().manual_seed(123)
    init, forc, bnd = torch.randn(B, 2, G, 17, generator=gen), torch.randn(B, T, G, 18, generator=gen), \
        torch.randn(B, T, G, 17, generator=gen)
    fc = fc.to(DEV).eval()
    with torch.no_grad():
        graphed = fc.rollout_graphed(init.to(DEV), forc.to(DEV), bnd.to(DEV))
        with ops.profile_launches() as prof:
            eager, _ = fc(init.to(DEV), forc.to(DEV), bnd.to(DEV))
    _assert_generic_path(prof.names())
    torch.testing.assert_close(eager, graphed, rtol=1e-6, atol=1e-6)
    got = graphed.cpu()
    del fc, m, graphed, eager
    _free()
    cfg = dict(model=kind, hidden_layers=1, processor_layers=P, mesh_aggr="sum")
    want, ref = _oracle_rollouts(params, g, cfg, init, forc, bnd)
    _rollout_errors("config 3 (HiLAM H=128 P=6, B=8)", got, want, ref)


@pytest.mark.gpu
def test_config4_step_real_size():
    """bench --config 4's model (GraphLAM H = 256, 4 processor layers, 1024 x 1024 grid) at B = 1: one forecast step
    against the chunked fp64 oracle; only generic-path and index kernels run."""
    _need(32)
    m, fc, kind, P = _bench_model(4)
    g = _oracle_graph(m, fc)
    params = {f"predictor.{k}": v.detach().clone() for k, v in m.state_dict().items()}
    G = m.num_grid_nodes
    assert G == 1024 * 1024
    gen = torch.Generator().manual_seed(123)
    init, forc, bnd = torch.randn(1, 2, G, 17, generator=gen), torch.randn(1, 1, G, 18, generator=gen), \
        torch.randn(1, 1, G, 17, generator=gen)
    fc = fc.to(DEV).eval()
    with torch.no_grad():
        fc(init.to(DEV), forc.to(DEV), bnd.to(DEV))  # fills the static-embedding cache
        with ops.profile_launches() as prof:
            got, _ = fc(init.to(DEV), forc.to(DEV), bnd.to(DEV))
    _assert_generic_path(prof.names())
    got = got.cpu()
    del fc, m
    _free()
    cfg = dict(model=kind, hidden_layers=1, processor_layers=P, mesh_aggr="sum")
    want, ref = _oracle_rollouts(params, g, cfg, init, forc, bnd)
    _rollout_errors("config 4 (GraphLAM H=256 P=4, B=1)", got, want, ref)


# ------------------------------------------------------------------------------------------------ 4. training gradients
@pytest.mark.gpu
def test_config3_training_step_gradients_real_size():
    """bench --config 3's model at the training leg's B = 4: one step, weighted loss, every parameter gradient against
    fp64 autograd through the oracle on the device (checkpointed per InteractionNet); the library's backward ran and no
    library GEMM did."""
    from test_backward_coverage_gpu import _check, _report, _run_checked

    _need(32)
    B = 4
    m, _, kind, P = _bench_model(3)
    g = _oracle_graph(m)
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    G = m.num_grid_nodes
    gen = torch.Generator().manual_seed(5)
    prev, pprev, forc = (torch.randn(B, G, d, generator=gen) for d in (17, 17, 18))
    w = torch.randn(B, G, 17, generator=gen)
    m = m.to(DEV)

    def step():
        got, _ = m(prev.to(DEV), pprev.to(DEV), forc.to(DEV))
        (got * w.to(DEV)).sum().backward()

    _run_checked(step, need=("ln_bwd_kernel", "transpose_pad_kernel"))
    grads = {k: p.grad.detach().cpu() for k, p in m.named_parameters()}
    del m
    _free()

    def ckpt_inet(*a, **kw):
        return torch.utils.checkpoint.checkpoint(_ORIG_INET, *a, use_reentrant=False, **kw)

    p64 = {k: (v.to(DEV).double().requires_grad_(True) if v.is_floating_point() else v.to(DEV)) for k, v in sd.items()}
    cfg = dict(model=kind, hidden_layers=1, processor_layers=P, mesh_aggr="sum")
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(rp, "interaction_net", ckpt_inet)
        out = rp.graph_model_forward(p64, _to_dev(g, torch.float64), cfg, prev.to(DEV).double(), pprev.to(DEV).double(),
                                     forc.to(DEV).double())
        (out * w.to(DEV).double()).sum().backward()
    errs = {k: _check(k, grads[k].to(DEV), p64[k].grad, rel=3e-2, abs_=2e-4, frob=None) for k in grads}
    _report(f"config 3 training step (HiLAM H=128 P=6, B={B})", errs)
