"""``--dense-dtype fp8`` through the fused training layers and the training step.

Layer level: ``PPLinearFn``, and ``SageConvFn`` / ``GcnConvFn`` wide (256 -> 256) and narrow (256 -> 41), forward and
backward, with ``ParamArena.dense_fp8`` set, against a float64 restatement that quantizes exactly the TN operands the
mode quantizes by the host rule (``tests/fp8_reference.py``) -- the activations and gradients, ``padded(W)`` for the
forward and ``transposed(W)`` for the input gradients -- and rounds exactly the NT operands (weight gradients) to bf16.
An operand that is itself a result of the step (``ah``, GCN's ``y``, ``dt``, and under ``--agg-dtype fp8`` the ``dys``
table) is recomputed by the same call the layer makes; without it ``dys`` is restated in float64 from its operands.  Output, ``d h_u`` and every parameter gradient agree within 1e-3 of the magnitude sum of their terms
(the fp8 wgmma's own sums keep fewer bits than f32: tests/test_dense_fp8_gpu.py), with ``--agg-dtype fp8`` on as well
for the wide layers.

Training step: graph replays bit-identical to eager epochs; 12 epochs at 4 in-process ranks within 2 % of the f32
run's loss summed over ranks and epochs, alone and with ``--agg-dtype fp8 --comm-dtype fp8``; a resume bit for bit."""
import pytest
import torch

from tests import fp8_reference as Q
from tests import layer_reference as R
from tests.test_comm_bf16_gpu import _parts
from tests.test_fused_layers_gpu import N_IN, _case, _dev, _inputs, _layer, _leaf, _setup, _step

pytestmark = pytest.mark.gpu

TOL = 1e-3
BENCH_ROWS = 232_965


def _q(t):
    """The f64 values of the fp8 rows of the f32 matrix ``t``."""
    return Q.dequantize(*Q.quantize_rows(t))


def _bf(t):
    return t.to(torch.bfloat16).double()


def _terms(sgn):
    return torch.abs if sgn else (lambda t: t)


def _fp8_step(case, layer, arena, h_u, dout, agg=False):
    arena.dense_fp8, case.g.agg_fp8 = True, agg
    try:
        return _step(case, layer, arena, _leaf(h_u), dout)
    finally:
        arena.dense_fp8, case.g.agg_fp8 = False, False


def _dys_table(arena, w, dout, rs32, agg):
    """Under ``--agg-dtype fp8``: the fp8 table of the wide layers' ``(dout W) / deg`` that the transposed passes
    gather, from the layer's own f32 product (its rounding decides the table's codes).  Otherwise ``None``: the
    references restate the product in float64 from its quantized operands."""
    from bns_gcn_b200 import ops
    from bns_gcn_b200.module import dense
    if not agg:
        return None
    return _q(dense.tc_mm_tn_fp8(ops.cvt_rows_fp8_any(dout), arena.fp8_rows(w, True), row_scale=rs32))


def _sage_reference(case, layer, arena, h_u, dout, narrow, agg):
    from bns_gcn_b200 import fused
    g, n_in, v, u = case.g, case.n_in, case.v, case.u
    rs32 = g.recip(case.in_norm)
    rs = rs32.double().unsqueeze(1)
    w1, w2 = layer.linear1.weight, layer.linear2.weight
    W1, W2 = _q(arena.padded(w1)), _q(arena.padded(w2))
    W1t, W2t = _q(arena.transposed(w1)), _q(arena.transposed(w2))
    b1, b2 = arena.padded(layer.linear1.bias).double(), arena.padded(layer.linear2.bias).double()
    hq, dq, db = _q(h_u), _q(dout), dout.double()
    if narrow:
        dys32 = fused.scale_rows(dout, rs32, out=fused.gather_friendly(n_in, dout.shape[1], dout.device))
        dt32 = fused._aggregate_t(g, dys32, case.n_u)
        dtq = _q(dt32)
    else:
        ah32 = fused._aggregate(g, h_u, rs32, None, 'fp8' if agg else False)
        ahq = _q(ah32)
        dys = _dys_table(arena, w2, dout, rs32, agg)
    res = []
    for sgn in (False, True):
        f = _terms(sgn)
        if narrow:
            out = f(hq[:n_in]) @ f(W1).t() + f(b1) + f(b2) + R.aggregate(f(hq) @ f(W2).t(), v, u, n_in) * rs
            du = f(dtq) @ f(W2t).t()
            dw2 = f(_bf(dt32)).t() @ f(_bf(h_u))
        else:
            out = f(hq[:n_in]) @ f(W1).t() + f(b1) + f(ahq) @ f(W2).t() + f(b2)
            d_ys = f(dys) if agg else (f(dq) @ f(W2t).t()) * f(rs)
            du = torch.zeros(case.n_u, h_u.shape[1], dtype=torch.float64, device=h_u.device).index_add(0, u, d_ys[v])
            dw2 = f(_bf(dout)).t() @ f(_bf(ah32))
        du[:n_in] += f(dq) @ f(W1t).t()
        res.append([out, du, f(_bf(dout)).t() @ f(_bf(h_u[:n_in])), f(db).sum(0), dw2, f(db).sum(0)])
    return res


def _gcn_reference(case, layer, arena, h_u, dout, narrow, agg):
    from bns_gcn_b200 import fused, ops
    g, n_in, v, u, c = case.g, case.n_in, case.v, case.u, case.c
    rs32, cs32 = g.recip(case.in_norm), g.recip(case.out_norm)
    rs = rs32.double().unsqueeze(1)
    w = layer.linear.weight
    W, Wt, b = _q(arena.padded(w)), _q(arena.transposed(w)), arena.padded(layer.linear.bias).double()
    hq, dq, db = _q(h_u), _q(dout), dout.double()
    cs_in, cs_halo = cs32[:n_in], cs32[n_in:]
    w_bwd = cs32.double()[c]
    mode = 'fp8' if agg else False
    if narrow:
        dys32 = fused.scale_rows(dout, rs32, out=fused.gather_friendly(n_in, dout.shape[1], dout.device))
        dt32 = fused._aggregate_t(g, dys32, case.n_u, cs_in, cs_halo)
        dtq = _q(dt32)
    else:
        y32 = ops.spmm_auto(g.a_in, fused._gather_table(fused.scale_rows(h_u[:n_in], cs_in), mode), row_scale=rs32)
        if g.a_out is not None and case.n_u > n_in:
            fused.halo_aggregate(g, fused._gather_table(h_u[n_in:], mode), y32, rs32, cs_halo)
        yq = _q(y32)
        dys = _dys_table(arena, w, dout, rs32, agg)
    res = []
    for sgn in (False, True):
        f = _terms(sgn)
        if narrow:
            out = R.aggregate(f(hq) @ f(W).t(), v, u, n_in, w_bwd) * rs + f(b)
            res.append([out, f(dtq) @ f(Wt).t(), f(_bf(dt32)).t() @ f(_bf(h_u)), f(db).sum(0)])
        else:
            d_ys = f(dys) if agg else (f(dq) @ f(Wt).t()) * f(rs)
            du = torch.zeros(case.n_u, h_u.shape[1], dtype=torch.float64, device=h_u.device).index_add(
                0, u, d_ys[v] * w_bwd.unsqueeze(1))
            res.append([f(yq) @ f(W).t() + f(b), du, f(_bf(dout)).t() @ f(_bf(y32)), f(db).sum(0)])
    return res


VARIANTS = ["sampled10", "sampled50", "colmap", "no-halo-matrix"]


def _check(label, layer, got, want, bound):
    out, du, grads = got
    R.assert_close(f"{label} out", out, want[0], bound[0], tol=TOL)
    R.assert_close(f"{label} d h_u", du, want[1], bound[1], tol=TOL)
    for (name, _), w, b in zip(layer.named_parameters(), want[2:], bound[2:]):
        R.assert_close(f"{label} d {name}", grads[name], w, b, tol=TOL)


@pytest.mark.parametrize("agg", [False, True], ids=["agg-f32", "agg-fp8"])
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("kind", ["sage", "gcn"])
def test_wide_layer_fp8_matches_float64(built, monkeypatch, kind, variant, agg):
    case = _case(kind, _setup(monkeypatch, variant, True))
    layer, arena = _layer(kind, 256, 256)
    h_u, dout = _inputs(case, 256, 256, seed=23)
    f32 = _step(case, layer, arena, _leaf(h_u), dout)
    got = _fp8_step(case, layer, arena, h_u, dout, agg)
    want, bound = (_sage_reference if kind == "sage" else _gcn_reference)(case, layer, arena, h_u, dout, False, agg)
    _check(f"{kind} 256->256 dense fp8 {variant} agg={agg}", layer, got, want, bound)
    again = _fp8_step(case, layer, arena, h_u, dout, agg)
    assert torch.equal(got[0], again[0]) and torch.equal(got[1], again[1])
    after = _step(case, layer, arena, _leaf(h_u), dout)          # no state left behind: the f32 bits again
    assert torch.equal(after[0], f32[0]) and torch.equal(after[1], f32[1])


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("kind", ["sage", "gcn"])
def test_narrow_layer_fp8_matches_float64(built, monkeypatch, kind, variant):
    case = _case(kind, _setup(monkeypatch, variant, True))
    layer, arena = _layer(kind, 256, 41)
    h_u, dout = _inputs(case, 256, 41, seed=29)
    got = _fp8_step(case, layer, arena, h_u, dout)
    want, bound = (_sage_reference if kind == "sage" else _gcn_reference)(case, layer, arena, h_u, dout, True, False)
    _check(f"{kind} 256->41 dense fp8 {variant}", layer, got, want, bound)
    assert torch.all(got[0][:, 41:] == 0), "pad columns of the output are not 0"


@pytest.mark.parametrize("rows", [N_IN, BENCH_ROWS])
@pytest.mark.parametrize("kind,n_feat", [("sage", 602), ("gcn", 604)])
def test_pp_linear_fp8(built, kind, n_feat, rows):
    """Layer 0 (``PPLinearFn``, no dropout): ``q(x) q(W)^T + b``, ``dx = q(dy) q(W^T)^T``, ``dW = bf(dy)^T bf(x)``."""
    dev = _dev()
    layer, arena = _layer(kind, n_feat, 256, pp=True)
    k = layer.linear.in_features
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(rows, k, generator=gen).to(dev)
    dy = torch.randn(rows, 256, generator=gen).to(dev)
    feat = _leaf(x)
    arena.flat_g.fill_(float("nan"))
    arena.dense_fp8 = True
    norms = (None,) if kind == "sage" else (None, None)
    out = layer(None, feat, *norms, fused=(arena, 0.0, 0, None))
    out.backward(dy)
    torch.cuda.synchronize()
    w = layer.linear.weight
    W, Wt, b = _q(arena.padded(w)), _q(arena.transposed(w)), arena.padded(layer.linear.bias).double()
    xq, dq = _q(x), _q(dy)
    want, bound = [], []
    for sgn, dst in ((False, want), (True, bound)):
        f = _terms(sgn)
        dst += [f(xq) @ f(W).t() + f(b), f(dq) @ f(Wt).t(), f(_bf(dy)).t() @ f(_bf(x)), f(dy.double()).sum(0)]
    label = f"{kind} pp {k}->256 rows={rows} dense fp8"
    R.assert_close(f"{label} out", out, want[0], bound[0], tol=TOL)
    R.assert_close(f"{label} dx", feat.grad, want[1], bound[1], tol=TOL)
    R.assert_close(f"{label} d linear.weight", arena.grad_padded(w), want[2], bound[2], tol=TOL)
    R.assert_close(f"{label} d linear.bias", arena.grad_padded(layer.linear.bias), want[3], bound[3], tol=TOL)


@pytest.mark.parametrize("model", ["graphsage", "gcn"])
def test_graphed_epoch_fp8_equals_eager(built, model):
    """``--dense-dtype fp8`` on one partition of the ``small`` shape (hidden 256, dropout 0.5): 2 eager epochs, then 3
    replays of the captured epoch, against 5 eager epochs -- losses and weights bit-identical."""
    from tests.harness import make_args
    from bns_gcn_b200 import train
    from bns_gcn_b200.data import make_graph, partition_graph
    from bns_gcn_b200.helper import context as ctx
    dev = _dev()
    part = partition_graph(make_graph("small", seed=0), 1, "random", seed=0)[0]

    def fresh():
        ctx.reset()
        a = make_args(dataset="small", model=model, n_hidden=256, dropout=0.5, dense_dtype="fp8")
        a.n_feat, a.n_class, a.n_train = part.meta["n_feat"], part.meta["n_class"], part.meta["n_train"]
        if model == "gcn" and a.n_feat % 4:
            pytest.skip("the fused GCN step needs a feature width that is a multiple of 4")
        st = train.setup(part.graph, part.node_dict, part.gpb, a, dev)
        assert st.arena is not None and st.arena.dense_fp8 and not st.arena.dense_bf16
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


@pytest.mark.parametrize("flags", [dict(dense_dtype="fp8"),
                                   dict(dense_dtype="fp8", agg_dtype="fp8", comm_dtype="fp8")],
                         ids=["dense", "dense-agg-comm"])
def test_training_converges_like_f32(built, flags):
    """The ``small`` shape at 4 in-process ranks, 3-layer GraphSAGE at hidden 256, 12 epochs: the loss summed over the
    ranks and the 12 epochs stays within 2 % of the f32 run's.  Epoch by epoch it does not always: on an H100 the
    largest gap was 2.2 % (epoch 8, dense fp8 alone) and 3.4 % (epoch 8, with agg / comm fp8); it is printed."""
    from tests.harness import make_args, run_product
    parts = _parts("small", 4)
    res = {}
    for name, kw in (("f32", {}), ("fp8", flags)):
        a = make_args(dataset="small", n_hidden=256, sampling_rate=0.3, dropout=0.5, backend="p2p", n_partitions=4, **kw)
        res[name] = run_product(parts, a, "cuda:0", 12, capture=False)
    lf = [sum(res["f32"][r]["loss"][e] for r in range(4)) for e in range(12)]
    lq = [sum(res["fp8"][r]["loss"][e] for r in range(4)) for e in range(12)]
    gap = max(abs(x - y) / abs(x) for x, y in zip(lf, lq))
    print(f"[loss] f32 {lf}\n[loss] fp8 {lq}\n[loss] largest epoch gap {gap:.4f}, total {sum(lq) / sum(lf) - 1:+.4f}")
    assert abs(sum(lq) - sum(lf)) <= 2e-2 * abs(sum(lf)), (lf, lq)


@pytest.mark.parametrize("model", ["graphsage", "gcn"])
def test_fp8_resumes_bit_for_bit(built, tmp_path, monkeypatch, model):
    """k epochs, a save, a teardown, a resume and k more equal 2k uninterrupted epochs (the derived fp8 weights are
    rebuilt from the loaded weights)."""
    from tests.test_resume_gpu import _args, _check_resume
    _check_resume(_args(4, model=model, backend="p2p", dense_dtype="fp8", agg_dtype="fp8", comm_dtype="fp8"),
                  tmp_path, monkeypatch, fused=True)
