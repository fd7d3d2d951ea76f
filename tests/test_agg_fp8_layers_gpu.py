"""``--agg-dtype fp8`` through the fused training layers and the training step.

Layer level: ``SageConvFn`` / ``GcnConvFn`` (256 -> 256, the aggregate-first branch every hidden layer takes) with
``PartitionGraph.agg_fp8`` set, forward and backward, against a float64 restatement that quantizes exactly the operands
the mode quantizes (tests/fp8_reference.py) and nothing else: forward, the rows the aggregation gathers (GraphSAGE:
``h_u``; GCN: ``h_u[:n_in] / out_norm`` and the halo rows of ``h_u``, whose column scale stays an f32 per-entry
weight); backward, the ``dys`` the transposed passes gather.  Output, ``d h_u`` and every parameter gradient agree within
1e-4 of the sum of the magnitudes of their terms, on the partitions of tests/test_fused_layers_gpu.py.

Training step: graph replays are bit-identical to eager epochs; over 12 epochs at 4 in-process ranks the summed loss
stays within 2 % of f32's, alone and with ``--comm-dtype bf16`` and ``--dense-dtype bf16``; a ``--resume`` run is
bit-exact; with ``--comm-dtype bf16`` the wide layers' halo pass gathers the received bf16 rows as they are."""
import pytest
import torch

from tests import fp8_reference as Q
from tests import layer_reference as R
from tests.test_agg_bf16_layers_gpu import VARIANTS
from tests.test_comm_bf16_gpu import _parts
from tests.test_fused_layers_gpu import _case, _dev, _inputs, _layer, _leaf, _setup, _step

pytestmark = pytest.mark.gpu

TOL = 1e-4


def _q(t):
    """The f64 values of the fp8 table of the f32 rows ``t``."""
    return Q.dequantize(*Q.quantize_rows(t))


def _sage_reference(case, layer, arena, h_u, dout):
    from bns_gcn_b200.module import dense
    n_in, v, u = case.n_in, case.v, case.u
    rs32 = case.g.recip(case.in_norm)
    rs = rs32.double().unsqueeze(1)
    W1, b1 = arena.padded(layer.linear1.weight).double(), arena.padded(layer.linear1.bias).double()
    W2, b2 = arena.padded(layer.linear2.weight).double(), arena.padded(layer.linear2.bias).double()
    dys = _q(dense.tc_mm_tn(dout, arena.transposed(layer.linear2.weight), row_scale=rs32))
    h, d = h_u.double(), dout.double()
    hq = torch.cat([_q(h_u[:n_in]), _q(h_u[n_in:])])        # the inner and the halo pass convert separately
    res = []
    for sgn in (False, True):
        f = torch.abs if sgn else (lambda t: t)
        ah = R.aggregate(f(hq), v, u, n_in) * rs
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
    xq = torch.cat([_q(fused.scale_rows(h_u[:n_in], cs32[:n_in])), _q(h_u[n_in:])])
    w_fwd = torch.where(u < n_in, torch.ones_like(c, dtype=torch.float64), cs32.double()[c])
    w_bwd = cs32.double()[c]
    dys = _q(dense.tc_mm_tn(dout, arena.transposed(layer.linear.weight), row_scale=rs32))
    d = dout.double()
    res = []
    for sgn in (False, True):
        f = torch.abs if sgn else (lambda t: t)
        y = R.aggregate(f(xq), v, u, n_in, w_fwd) * rs
        out = y @ f(W).t() + f(b)
        du = torch.zeros(case.n_u, h_u.shape[1], dtype=torch.float64, device=h_u.device).index_add(
            0, u, f(dys)[v] * w_bwd.unsqueeze(1))
        res.append([out, du, f(d).t() @ y, f(d).sum(0)])
    return res


def _fp8_step(case, layer, arena, h_u, dout):
    case.g.agg_fp8 = True
    try:
        return _step(case, layer, arena, _leaf(h_u), dout)
    finally:
        case.g.agg_fp8 = False


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("kind", ["sage", "gcn"])
def test_layer_fp8_matches_float64(built, monkeypatch, kind, variant):
    case = _case(kind, _setup(monkeypatch, variant, True))
    layer, arena = _layer(kind, 256, 256)
    h_u, dout = _inputs(case, 256, 256, seed=21)
    out, du, grads = _fp8_step(case, layer, arena, h_u, dout)
    want, bound = (_sage_reference if kind == "sage" else _gcn_reference)(case, layer, arena, h_u, dout)
    label = f"{kind} fp8 {variant}"
    R.assert_close(f"{label} out", out, want[0], bound[0], tol=TOL)
    R.assert_close(f"{label} d h_u", du, want[1], bound[1], tol=TOL)
    for (name, _), w, b in zip(layer.named_parameters(), want[2:], bound[2:]):
        R.assert_close(f"{label} d {name}", grads[name], w, b, tol=TOL)
    again = _fp8_step(case, layer, arena, h_u, dout)
    assert torch.equal(out, again[0]) and torch.equal(du, again[1])
    case.g.agg_bf16 = True                                               # fp8 is not bf16
    try:
        bf = _step(case, layer, arena, _leaf(h_u), dout)
    finally:
        case.g.agg_bf16 = False
    assert not torch.equal(out, bf[0])


@pytest.mark.parametrize("model", ["graphsage", "gcn"])
def test_graphed_epoch_fp8_equals_eager(built, model):
    """``--agg-dtype fp8`` on one partition of the ``small`` shape (hidden 256, dropout 0.5): 2 eager epochs, then 3
    replays of the captured epoch, against 5 eager epochs -- losses and weights bit-identical."""
    from tests.harness import make_args
    from bns_gcn_b200 import train
    from bns_gcn_b200.data import make_graph, partition_graph
    from bns_gcn_b200.helper import context as ctx
    dev = _dev()
    part = partition_graph(make_graph("small", seed=0), 1, "random", seed=0)[0]

    def fresh():
        ctx.reset()
        a = make_args(dataset="small", model=model, n_hidden=256, dropout=0.5, agg_dtype="fp8")
        a.n_feat, a.n_class, a.n_train = part.meta["n_feat"], part.meta["n_class"], part.meta["n_train"]
        if model == "gcn" and a.n_feat % 4:
            pytest.skip("the fused GCN step needs a feature width that is a multiple of 4")
        st = train.setup(part.graph, part.node_dict, part.gpb, a, dev)
        assert st.arena is not None and st.part.agg_fp8 and not st.part.agg_bf16
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


@pytest.mark.parametrize("flags", [dict(agg_dtype="fp8"), dict(agg_dtype="fp8", dense_dtype="bf16"),
                                   dict(agg_dtype="fp8", comm_dtype="bf16"),
                                   dict(agg_dtype="fp8", comm_dtype="bf16", dense_dtype="bf16")],
                         ids=["fp8", "fp8-dense", "fp8-comm", "fp8-comm-dense"])
def test_training_converges_like_f32(built, flags):
    """The ``small`` shape at 4 in-process ranks, 3-layer GraphSAGE at hidden 256, 12 epochs: the summed loss stays
    within 2 % of the f32 run's at every epoch."""
    from tests.harness import make_args, run_product
    parts = _parts("small", 4)
    res = {}
    for name, kw in (("f32", {}), ("fp8", flags)):
        a = make_args(dataset="small", n_hidden=256, sampling_rate=0.3, dropout=0.5, backend="p2p", n_partitions=4, **kw)
        res[name] = run_product(parts, a, "cuda:0", 12, capture=False)
    lf = [sum(res["f32"][r]["loss"][e] for r in range(4)) for e in range(12)]
    lq = [sum(res["fp8"][r]["loss"][e] for r in range(4)) for e in range(12)]
    print(f"[loss] f32 {lf}\n[loss] fp8 {lq}")
    for x, y in zip(lf, lq):
        assert abs(x - y) <= 2e-2 * abs(x), (lf, lq)


def test_fp8_with_comm_bf16_halo_pass_gathers_the_received_rows(built, monkeypatch):
    """With ``--comm-dtype bf16`` the wide layers' halo pass takes the received bf16 rows as they are: the forward pass
    gathers no fp8 table of them (only the inner rows and the transposed passes' ``dys`` are converted)."""
    from bns_gcn_b200 import fused, ops
    seen = []
    plain = ops.cvt_rows_fp8

    def spy(src, out=None):
        seen.append(src.shape[0])
        return plain(src, out)
    monkeypatch.setattr(ops, "cvt_rows_fp8", spy)
    case = _case("sage", _setup(monkeypatch, "sampled50", True))
    g = case.g
    h_u, _ = _inputs(case, 256, 256, seed=5)
    halo = ops.cvt_rows_bf16(h_u[case.n_in:].contiguous())
    rs32 = g.recip(case.in_norm)
    ah = fused._aggregate(g, h_u[:case.n_in], rs32, None, 'fp8', halo)
    assert seen == [case.n_in]
    hq = torch.cat([_q(h_u[:case.n_in]), halo.double()])
    v, u = case.v, case.u
    val = R.aggregate(hq, v, u, case.n_in) * rs32.double().unsqueeze(1)
    bnd = R.aggregate(hq.abs(), v, u, case.n_in) * rs32.double().unsqueeze(1)
    R.assert_close("fp8 + comm bf16 forward", ah, val, bnd, tol=TOL)


def test_fp8_resumes_bit_for_bit(built, tmp_path, monkeypatch):
    from tests.test_resume_gpu import _args, _check_resume
    _check_resume(_args(4, backend="p2p", agg_dtype="fp8"), tmp_path, monkeypatch, fused=True)
    (tmp_path / "gcn").mkdir()
    _check_resume(_args(1, backend="nccl", model="gcn", agg_dtype="fp8"), tmp_path / "gcn", monkeypatch, fused=True)
