"""``--agg-dtype bf16`` through the fused training layers and the training step.

Layer level: ``SageConvFn`` / ``GcnConvFn`` (256 -> 256, the aggregate-first branch every hidden layer takes) with
``PartitionGraph.agg_bf16`` set, forward and backward, against a float64 restatement that rounds exactly the operands the
mode rounds and nothing else: forward, the rows the aggregation gathers (GraphSAGE: ``h_u``; GCN: ``h_u[:n_in] /
out_norm`` -- the f32 product the inner pass gathers -- and the halo rows of ``h_u``, whose column scale stays an f32
per-entry weight); backward, the ``dys`` the transposed passes gather (the f32 result of the layer's own
``(dout W) / norm`` GEMM, recomputed here with the same call).  Output, ``d h_u`` and every parameter gradient agree
within 1e-4 of the sum of the magnitudes of their terms, on the partition of tests/test_fused_layers_gpu.py (long rows,
10 % / 50 % samples through the compaction, the slot-map fallback, 2 source-row blocks, no halo) and on the benchmark's
one-rank Reddit-shape graph (233 K rows, ~115 M entries).

Training step: with ``--agg-dtype bf16``, ``train.GraphedEpoch`` replays are bit-identical to the eager epochs."""
import argparse

import pytest
import torch

from tests import layer_reference as R
from tests.test_fused_layers_gpu import _case, _dev, _inputs, _layer, _leaf, _setup, _step

pytestmark = pytest.mark.gpu

TOL = 1e-4


def _bf(t):
    return t.to(torch.bfloat16).double()


def _sage_reference(case, layer, arena, h_u, dout):
    from bns_gcn_b200.module import dense
    n_in, v, u = case.n_in, case.v, case.u
    rs32 = case.g.recip(case.in_norm)
    rs = rs32.double().unsqueeze(1)
    W1, b1 = arena.padded(layer.linear1.weight).double(), arena.padded(layer.linear1.bias).double()
    W2, b2 = arena.padded(layer.linear2.weight).double(), arena.padded(layer.linear2.bias).double()
    dys = _bf(dense.tc_mm_tn(dout, arena.transposed(layer.linear2.weight), row_scale=rs32))
    h, hb, d = h_u.double(), _bf(h_u), dout.double()
    res = []
    for sgn in (False, True):            # values, then bounds (every operand by magnitude)
        f = torch.abs if sgn else (lambda t: t)
        ah = R.aggregate(f(hb), v, u, n_in) * rs
        out = f(h[:n_in]) @ f(W1).t() + f(b1) + ah @ f(W2).t() + f(b2)
        du = torch.zeros(case.n_u, h.shape[1], dtype=torch.float64, device=h.device).index_add(0, u, f(dys)[v])
        du[:n_in] += f(d) @ f(W1)
        dw1, dw2 = f(d).t() @ f(h[:n_in]), f(d).t() @ ah
        db = f(d).sum(0)
        res.append([out, du, dw1, db, dw2, db])
    return res


def _gcn_reference(case, layer, arena, h_u, dout):
    from bns_gcn_b200 import fused
    from bns_gcn_b200.module import dense
    n_in, v, u, c = case.n_in, case.v, case.u, case.c
    rs32, cs32 = case.g.recip(case.in_norm), case.g.recip(case.out_norm)
    rs = rs32.double().unsqueeze(1)
    W, b = arena.padded(layer.linear.weight).double(), arena.padded(layer.linear.bias).double()
    xb = torch.cat([_bf(fused.scale_rows(h_u[:n_in], cs32[:n_in])), _bf(h_u[n_in:])])
    w_fwd = torch.where(u < n_in, torch.ones_like(c, dtype=torch.float64), cs32.double()[c])
    w_bwd = cs32.double()[c]
    dys = _bf(dense.tc_mm_tn(dout, arena.transposed(layer.linear.weight), row_scale=rs32))
    d = dout.double()
    res = []
    for sgn in (False, True):
        f = torch.abs if sgn else (lambda t: t)
        y = R.aggregate(f(xb), v, u, n_in, w_fwd) * rs
        out = y @ f(W).t() + f(b)
        du = torch.zeros(case.n_u, h_u.shape[1], dtype=torch.float64, device=h_u.device).index_add(
            0, u, f(dys)[v] * w_bwd.unsqueeze(1))
        res.append([out, du, f(d).t() @ y, f(d).sum(0)])
    return res


def _bf16_step(case, layer, arena, h_u, dout):
    case.g.agg_bf16 = True
    try:
        return _step(case, layer, arena, _leaf(h_u), dout)
    finally:
        case.g.agg_bf16 = False


VARIANTS = ["sampled10", "sampled50", "colmap", "sampled50-2blocks", "no-halo-matrix"]


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("kind", ["sage", "gcn"])
def test_layer_bf16_matches_float64(built, monkeypatch, kind, variant):
    case = _case(kind, _setup(monkeypatch, variant, True))
    layer, arena = _layer(kind, 256, 256)
    h_u, dout = _inputs(case, 256, 256, seed=21)
    out, du, grads = _bf16_step(case, layer, arena, h_u, dout)
    want, bound = (_sage_reference if kind == "sage" else _gcn_reference)(case, layer, arena, h_u, dout)
    label = f"{kind} bf16 {variant}"
    R.assert_close(f"{label} out", out, want[0], bound[0], tol=TOL)
    R.assert_close(f"{label} d h_u", du, want[1], bound[1], tol=TOL)
    for (name, _), w, b in zip(layer.named_parameters(), want[2:], bound[2:]):
        R.assert_close(f"{label} d {name}", grads[name], w, b, tol=TOL)
    again = _bf16_step(case, layer, arena, h_u, dout)
    assert torch.equal(out, again[0]) and torch.equal(du, again[1])
    f32 = _step(case, layer, arena, _leaf(h_u), dout)                   # the flag is off again: the f32 result
    assert not torch.equal(out, f32[0])


def _chunked_aggregate(x, ip, ix, n_rows, rows_per_chunk=4096):
    """``A x`` in float64 for a CSR matrix too large for one gather of all its entries."""
    out = torch.empty(n_rows, x.shape[1], dtype=torch.float64, device=x.device)
    for r0 in range(0, n_rows, rows_per_chunk):
        r1 = min(n_rows, r0 + rows_per_chunk)
        e0, e1 = int(ip[r0]), int(ip[r1])
        rows = torch.repeat_interleave(torch.arange(r1 - r0, device=x.device), ip[r0 + 1:r1 + 1] - ip[r0:r1])
        out[r0:r1] = torch.zeros(r1 - r0, x.shape[1], dtype=torch.float64, device=x.device).index_add_(
            0, rows, x[ix[e0:e1].long()])
    return out


def test_sage_layer_bf16_at_bench_shape(built):
    """GraphSAGE 256 -> 256 on the one-rank Reddit-shape partition (every node inner, no halo), forward and backward."""
    from bns_gcn_b200.data import make_graph, partition_graph
    from bns_gcn_b200.graph import PartitionGraph
    from bns_gcn_b200.module import dense
    free, _ = torch.cuda.mem_get_info(0)
    if free < (40 << 30):
        pytest.skip("needs ~40 GB of free device memory")
    from bns_gcn_b200.train import get_in_out_graph
    dev = _dev()
    part = partition_graph(make_graph("reddit", seed=0, device=dev), 1, "random", seed=0, device=dev)[0]
    a_in, _ = get_in_out_graph(part.graph, part.node_dict, dev)
    ip, ix = a_in.csr()
    n = a_in.n_rows
    assert n == part.graph.n_in and a_in.nnz > 100_000_000
    g = PartitionGraph(n, 0, a_in, None, dev)
    g.n_u = n
    deg = (ip[1:] - ip[:-1]).float()
    case = argparse.Namespace(kind="sage", g=g, n_in=n, n_u=n, in_norm=deg.clamp(min=1))
    layer, arena = _layer("sage", 256, 256)
    gen = torch.Generator().manual_seed(31)
    h_u, dout = torch.randn(n, 256, generator=gen).to(dev), torch.randn(n, 256, generator=gen).to(dev)
    out, du, grads = _bf16_step(case, layer, arena, h_u, dout)
    rs32 = g.recip(case.in_norm)
    rs = rs32.double().unsqueeze(1)
    dys = _bf(dense.tc_mm_tn(dout, arena.transposed(layer.linear2.weight), row_scale=rs32))
    ipt, ixt = a_in.transpose().csr()
    W1, b1 = arena.padded(layer.linear1.weight).double(), arena.padded(layer.linear1.bias).double()
    W2, b2 = arena.padded(layer.linear2.weight).double(), arena.padded(layer.linear2.bias).double()
    h, hb, d = h_u.double(), _bf(h_u), dout.double()
    for sgn in (False, True):
        f = torch.abs if sgn else (lambda t: t)
        ah = _chunked_aggregate(f(hb), ip, ix, n) * rs
        o = f(h) @ f(W1).t() + f(b1) + ah @ f(W2).t() + f(b2)
        dh = _chunked_aggregate(f(dys), ipt, ixt, n) + f(d) @ f(W1)
        dw1, dw2, db = f(d).t() @ f(h), f(d).t() @ ah, f(d).sum(0)
        if not sgn:
            want = [o, dh, dw1, db, dw2, db]
        else:
            bound = [o, dh, dw1, db, dw2, db]
        del ah, o, dh
    R.assert_close("bench-shape bf16 out", out, want[0], bound[0], tol=TOL)
    R.assert_close("bench-shape bf16 d h_u", du, want[1], bound[1], tol=TOL)
    for (name, _), w, b in zip(layer.named_parameters(), want[2:], bound[2:]):
        R.assert_close(f"bench-shape bf16 d {name}", grads[name], w, b, tol=TOL)


@pytest.mark.parametrize("model", ["graphsage", "gcn"])
def test_graphed_epoch_bf16_equals_eager(built, model):
    """``--agg-dtype bf16`` on one partition of the ``small`` shape (hidden 256, dropout 0.5): 2 eager epochs, then 3
    replays of the captured epoch, against 5 eager epochs -- losses and weights bit-identical.  (Ranks that live as
    threads of one process cannot capture their exchange -- each waits on events of the other's stream -- so the
    multi-rank replay is the one-process-per-GPU launch's.)"""
    from tests.harness import make_args
    from bns_gcn_b200 import train
    from bns_gcn_b200.data import make_graph, partition_graph
    from bns_gcn_b200.helper import context as ctx
    dev = _dev()
    part = partition_graph(make_graph("small", seed=0), 1, "random", seed=0)[0]

    def fresh():
        ctx.reset()
        a = make_args(dataset="small", model=model, n_hidden=256, dropout=0.5, agg_dtype="bf16")
        a.n_feat, a.n_class, a.n_train = part.meta["n_feat"], part.meta["n_class"], part.meta["n_train"]
        if model == "gcn" and a.n_feat % 4:
            pytest.skip("the fused GCN step needs a feature width that is a multiple of 4")
        st = train.setup(part.graph, part.node_dict, part.gpb, a, dev)
        assert st.arena is not None and st.part.agg_bf16
        return st
    prev = torch.autograd.is_multithreading_enabled()
    torch.autograd.set_multithreading_enabled(False)
    prev_stream = torch.cuda.current_stream(dev)
    torch.cuda.set_stream(torch.cuda.Stream(dev))
    try:
        st = fresh()
        eager = [train.train_epoch(st, e).item() for e in range(5)]
        w_eager = [p.detach().clone() for p in st.model.parameters()]
        st = fresh()
        ge = train.GraphedEpoch(st, warmup=2)
        replay = [ge().item() for _ in range(3)]
        w_graph = [p.detach().clone() for p in st.model.parameters()]
    finally:
        torch.cuda.synchronize(dev)
        torch.cuda.set_stream(prev_stream)
        torch.autograd.set_multithreading_enabled(prev)
        ctx.reset()
    assert replay == eager[2:], (replay, eager)
    for a_, b_ in zip(w_graph, w_eager):
        assert torch.equal(a_, b_)
