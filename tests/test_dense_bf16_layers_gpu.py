"""``--dense-dtype bf16`` through the fused training layers and the training step.

Layer level: ``PPLinearFn``, and ``SageConvFn`` / ``GcnConvFn`` wide (256 -> 256, aggregate first) and narrow (256 -> 41,
transform first), forward and backward, with ``ParamArena.dense_bf16`` set, against a float64 restatement that rounds
exactly the GEMM operands the mode rounds -- every A and B of every forward, input-gradient and weight-gradient product
-- and nothing else.  An operand that is itself a result of the step (``ah``, GCN's ``y``, the narrow layers' ``dt``, the
``dys`` the wide layers' transposed passes gather) is recomputed by the same f32 call the layer makes and then rounded,
as tests/test_agg_bf16_layers_gpu.py does.  Output, ``d h_u`` and every parameter gradient agree within 1e-4 of the sum
of the magnitudes of their terms, on partition variants of tests/test_fused_layers_gpu.py, with ``--agg-dtype bf16``
on as well for the wide layers, and for layer 0 at the benchmark's one-rank Reddit shape.

Training step: graph replays bit-identical to eager epochs; an f32 step after a bf16 one gives the f32 bits; 12 epochs at
4 in-process ranks stay within 2 % of the f32 run's summed loss, alone and with ``--agg-dtype bf16 --comm-dtype bf16``."""
import pytest
import torch

from tests import layer_reference as R
from tests.test_comm_bf16_gpu import _parts
from tests.test_fused_layers_gpu import N_IN, _case, _dev, _inputs, _layer, _leaf, _setup, _step

pytestmark = pytest.mark.gpu

TOL = 1e-4
BENCH_ROWS = 232_965


def _bf(t):
    return t.to(torch.bfloat16).double()


def _bf16_step(case, layer, arena, h_u, dout, agg=False):
    arena.dense_bf16, case.g.agg_bf16 = True, agg
    try:
        return _step(case, layer, arena, _leaf(h_u), dout)
    finally:
        arena.dense_bf16, case.g.agg_bf16 = False, False


def _terms(sgn):
    return torch.abs if sgn else (lambda t: t)


def _sage_reference(case, layer, arena, h_u, dout, narrow, agg):
    from bns_gcn_b200 import fused
    from bns_gcn_b200.module import dense
    g, n_in, v, u = case.g, case.n_in, case.v, case.u
    rs32 = g.recip(case.in_norm)
    rs = rs32.double().unsqueeze(1)
    w1, w2 = layer.linear1.weight, layer.linear2.weight
    W1, b1 = _bf(arena.padded(w1)), arena.padded(layer.linear1.bias).double()
    W2, b2 = _bf(arena.padded(w2)), arena.padded(layer.linear2.bias).double()
    hb, d, db = _bf(h_u), _bf(dout), dout.double()
    if narrow:
        dys32 = fused.scale_rows(dout, rs32, out=fused.gather_friendly(n_in, dout.shape[1], dout.device))
        dt = _bf(fused._aggregate_t(g, dys32, case.n_u))
    else:
        ah = _bf(fused._aggregate(g, h_u, rs32, None, agg))
        dys = dense.tc_mm_tn(dout, arena.transposed(w2), row_scale=rs32, bf16=True).double()
        dys = _bf(dys) if agg else dys
    res = []
    for sgn in (False, True):
        f = _terms(sgn)
        if narrow:
            out = f(hb[:n_in]) @ f(W1).t() + f(b1) + f(b2) + R.aggregate(f(hb) @ f(W2).t(), v, u, n_in) * rs
            du = f(dt) @ f(W2)
            dw2 = f(dt).t() @ f(hb)
        else:
            out = f(hb[:n_in]) @ f(W1).t() + f(b1) + f(ah) @ f(W2).t() + f(b2)
            du = torch.zeros(case.n_u, h_u.shape[1], dtype=torch.float64, device=h_u.device).index_add(0, u, f(dys)[v])
            dw2 = f(d).t() @ f(ah)
        du[:n_in] += f(d) @ f(W1)
        res.append([out, du, f(d).t() @ f(hb[:n_in]), f(db).sum(0), dw2, f(db).sum(0)])
    return res


def _gcn_reference(case, layer, arena, h_u, dout, narrow, agg):
    from bns_gcn_b200 import fused, ops
    from bns_gcn_b200.module import dense
    g, n_in, v, u, c = case.g, case.n_in, case.v, case.u, case.c
    rs32, cs32 = g.recip(case.in_norm), g.recip(case.out_norm)
    rs = rs32.double().unsqueeze(1)
    w = layer.linear.weight
    W, b = _bf(arena.padded(w)), arena.padded(layer.linear.bias).double()
    hb, d, db = _bf(h_u), _bf(dout), dout.double()
    cs_in, cs_halo = cs32[:n_in], cs32[n_in:]
    w_bwd = cs32.double()[c]
    if narrow:
        dys32 = fused.scale_rows(dout, rs32, out=fused.gather_friendly(n_in, dout.shape[1], dout.device))
        dt = _bf(fused._aggregate_t(g, dys32, case.n_u, cs_in, cs_halo))
    else:
        y32 = ops.spmm_auto(g.a_in, fused._gather_table(fused.scale_rows(h_u[:n_in], cs_in), agg), row_scale=rs32)
        if g.a_out is not None and case.n_u > n_in:
            fused.halo_aggregate(g, fused._gather_table(h_u[n_in:], agg), y32, rs32, cs_halo)
        y = _bf(y32)
        dys = dense.tc_mm_tn(dout, arena.transposed(w), row_scale=rs32, bf16=True).double()
        dys = _bf(dys) if agg else dys
    res = []
    for sgn in (False, True):
        f = _terms(sgn)
        if narrow:
            out = R.aggregate(f(hb) @ f(W).t(), v, u, n_in, w_bwd) * rs + f(b)
            res.append([out, f(dt) @ f(W), f(dt).t() @ f(hb), f(db).sum(0)])
        else:
            du = torch.zeros(case.n_u, h_u.shape[1], dtype=torch.float64, device=h_u.device).index_add(
                0, u, f(dys)[v] * w_bwd.unsqueeze(1))
            res.append([f(y) @ f(W).t() + f(b), du, f(d).t() @ f(y), f(db).sum(0)])
    return res


VARIANTS = ["sampled10", "sampled50", "colmap", "sampled50-2blocks", "no-halo-matrix"]


def _check(label, case, layer, arena, h_u, dout, got, want, bound):
    out, du, grads = got
    R.assert_close(f"{label} out", out, want[0], bound[0], tol=TOL)
    R.assert_close(f"{label} d h_u", du, want[1], bound[1], tol=TOL)
    for (name, _), w, b in zip(layer.named_parameters(), want[2:], bound[2:]):
        R.assert_close(f"{label} d {name}", grads[name], w, b, tol=TOL)


@pytest.mark.parametrize("agg", [False, True], ids=["agg-f32", "agg-bf16"])
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("kind", ["sage", "gcn"])
def test_wide_layer_bf16_matches_float64(built, monkeypatch, kind, variant, agg):
    case = _case(kind, _setup(monkeypatch, variant, True))
    layer, arena = _layer(kind, 256, 256)
    h_u, dout = _inputs(case, 256, 256, seed=23)
    f32 = _step(case, layer, arena, _leaf(h_u), dout)
    got = _bf16_step(case, layer, arena, h_u, dout, agg)
    want, bound = (_sage_reference if kind == "sage" else _gcn_reference)(case, layer, arena, h_u, dout, False, agg)
    _check(f"{kind} 256->256 dense bf16 {variant} agg={agg}", case, layer, arena, h_u, dout, got, want, bound)
    again = _bf16_step(case, layer, arena, h_u, dout, agg)
    assert torch.equal(got[0], again[0]) and torch.equal(got[1], again[1])
    assert not torch.equal(got[0], f32[0])
    after = _step(case, layer, arena, _leaf(h_u), dout)          # no state left behind: the f32 bits again
    assert torch.equal(after[0], f32[0]) and torch.equal(after[1], f32[1])
    for name in f32[2]:
        assert torch.equal(after[2][name], f32[2][name]), name


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("kind", ["sage", "gcn"])
def test_narrow_layer_bf16_matches_float64(built, monkeypatch, kind, variant):
    case = _case(kind, _setup(monkeypatch, variant, True))
    layer, arena = _layer(kind, 256, 41)
    h_u, dout = _inputs(case, 256, 41, seed=29)
    got = _bf16_step(case, layer, arena, h_u, dout)
    want, bound = (_sage_reference if kind == "sage" else _gcn_reference)(case, layer, arena, h_u, dout, True, False)
    _check(f"{kind} 256->41 dense bf16 {variant}", case, layer, arena, h_u, dout, got, want, bound)
    fout = 41
    assert torch.all(got[0][:, fout:] == 0), "pad columns of the output are not 0"


@pytest.mark.parametrize("rows", [N_IN, BENCH_ROWS])
@pytest.mark.parametrize("kind,n_feat", [("sage", 602), ("gcn", 604)])
def test_pp_linear_bf16(built, kind, n_feat, rows):
    """Layer 0 (``PPLinearFn``, no dropout): ``bf(x) bf(W)^T + b``, ``dx = bf(dy) bf(W)``, ``dW = bf(dy)^T bf(x)``; at
    the benchmark's one-rank row count too (GraphSAGE: K = 1204, the largest GEMM of the epoch)."""
    dev = _dev()
    layer, arena = _layer(kind, n_feat, 256, pp=True)
    k = layer.linear.in_features
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(rows, k, generator=gen).to(dev)
    dy = torch.randn(rows, 256, generator=gen).to(dev)
    feat = _leaf(x)
    arena.flat_g.fill_(float("nan"))
    arena.dense_bf16 = True
    norms = (None,) if kind == "sage" else (None, None)
    out = layer(None, feat, *norms, fused=(arena, 0.0, 0, None))
    out.backward(dy)
    torch.cuda.synchronize()
    W, b = _bf(arena.padded(layer.linear.weight)), arena.padded(layer.linear.bias).double()
    xb, d = _bf(x), _bf(dy)
    want, bound = [], []
    for sgn, dst in ((False, want), (True, bound)):
        f = _terms(sgn)
        dst += [f(xb) @ f(W).t() + f(b), f(d) @ f(W), f(d).t() @ f(xb), f(dy.double()).sum(0)]
    label = f"{kind} pp {k}->256 rows={rows} dense bf16"
    R.assert_close(f"{label} out", out, want[0], bound[0], tol=TOL)
    R.assert_close(f"{label} dx", feat.grad, want[1], bound[1], tol=TOL)
    R.assert_close(f"{label} d linear.weight", arena.grad_padded(layer.linear.weight), want[2], bound[2], tol=TOL)
    R.assert_close(f"{label} d linear.bias", arena.grad_padded(layer.linear.bias), want[3], bound[3], tol=TOL)


@pytest.mark.parametrize("model", ["graphsage", "gcn"])
def test_graphed_epoch_bf16_equals_eager(built, model):
    """``--dense-dtype bf16`` on one partition of the ``small`` shape (hidden 256, dropout 0.5): 2 eager epochs, then 3
    replays of the captured epoch, against 5 eager epochs -- losses and weights bit-identical."""
    from tests.harness import make_args
    from bns_gcn_b200 import train
    from bns_gcn_b200.data import make_graph, partition_graph
    from bns_gcn_b200.helper import context as ctx
    dev = _dev()
    part = partition_graph(make_graph("small", seed=0), 1, "random", seed=0)[0]

    def fresh():
        ctx.reset()
        a = make_args(dataset="small", model=model, n_hidden=256, dropout=0.5, dense_dtype="bf16")
        a.n_feat, a.n_class, a.n_train = part.meta["n_feat"], part.meta["n_class"], part.meta["n_train"]
        if model == "gcn" and a.n_feat % 4:
            pytest.skip("the fused GCN step needs a feature width that is a multiple of 4")
        st = train.setup(part.graph, part.node_dict, part.gpb, a, dev)
        assert st.arena is not None and st.arena.dense_bf16
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


@pytest.mark.parametrize("flags", [dict(dense_dtype="bf16"),
                                   dict(dense_dtype="bf16", agg_dtype="bf16", comm_dtype="bf16")],
                         ids=["dense", "dense-agg-comm"])
def test_training_converges_like_f32(built, flags):
    """The ``small`` shape at 4 in-process ranks, 3-layer GraphSAGE at hidden 256, 12 epochs: the summed loss stays
    within 2 % of the f32 run's at every epoch."""
    from tests.harness import make_args, run_product
    parts = _parts("small", 4)
    res = {}
    for name, kw in (("f32", {}), ("bf16", flags)):
        a = make_args(dataset="small", n_hidden=256, sampling_rate=0.3, dropout=0.5, backend="p2p", n_partitions=4, **kw)
        res[name] = run_product(parts, a, "cuda:0", 12, capture=False)
    lf = [sum(res["f32"][r]["loss"][e] for r in range(4)) for e in range(12)]
    lb = [sum(res["bf16"][r]["loss"][e] for r in range(4)) for e in range(12)]
    print(f"[loss] f32 {lf}\n[loss] bf16 {lb}")
    for x, y in zip(lf, lb):
        assert abs(x - y) <= 2e-2 * abs(x), (lf, lb)
