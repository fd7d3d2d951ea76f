"""``--model transformer`` end to end: the exchange is unscaled, ``--cuda-graph`` replays bit-identical to eager epochs,
``--resume`` bit for bit, the partition-parallel evaluation (transductive and inductive) against the whole-graph
``Evaluator``, and a short ``main.py`` run.  Training against the CPU oracle is in test_transformer_parity_gpu."""
import argparse
import re

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / b.norm().clamp(min=1e-30)).item()


def test_the_exchange_is_unscaled(built):
    """``setup`` hands the feature buffer a ratio of 1.0 for every peer at sampling rate 0.3, where ``get_send_size``
    gives the sampled shares."""
    from bns_gcn_b200 import train
    from bns_gcn_b200.data import make_graph, partition_graph
    from bns_gcn_b200.helper.comm import run_threads
    from tests.harness import make_args
    parts = partition_graph(make_graph("tiny", seed=0), 3, "random", seed=0)

    def fn(comm, r):
        p = parts[r]
        a = make_args(model="transformer", n_partitions=3, sampling_rate=0.3, n_layers=2, heads=2)
        a.n_feat, a.n_class, a.n_train = p.meta["n_feat"], p.meta["n_class"], p.meta["n_train"]
        st = train.setup(p.graph, p.node_dict, p.gpb, a, DEV)
        return list(st.ratio), train.get_send_size(st.boundary, 0.3)[1]
    for r, (ratio, shares) in enumerate(run_threads(3, fn, device=DEV)):
        assert ratio == [0 if i == r else 1.0 for i in range(3)]
        assert all(0 < x < 1 for i, x in enumerate(shares) if i != r)


@pytest.mark.parametrize("kw", [dict(heads=1, n_layers=2), dict(heads=2, n_layers=2),
                                dict(heads=2, n_layers=3, n_linear=1)], ids=["1head", "2heads", "2heads-n-linear1"])
def test_transformer_replayed_run_equals_the_eager_run(built, tmp_path, monkeypatch, capsys, kw):
    from tests.test_cuda_graph_cli_gpu import _args, _check_same, _train
    kw = dict(model="transformer", **kw)
    eager = _train(_args(**kw), monkeypatch, capsys, tmp_path / "eager")
    graphed = _train(_args(cuda_graph=True, **kw), monkeypatch, capsys, tmp_path / "graph")
    _check_same(eager, graphed)
    assert eager["fused"] is False and graphed["fused"] is False
    keys = set(eager["model"])
    for i in range(kw["n_layers"] - kw.get("n_linear", 0)):
        assert {f"layers.{i}.{lin}.{p}" for lin in ("lin_key", "lin_query", "lin_value", "lin_skip")
                for p in ("weight", "bias")} <= keys


def test_transformer_resumes_bit_for_bit(built, tmp_path, monkeypatch):
    from tests.test_resume_gpu import _args, _check_resume
    _check_resume(_args(1, model="transformer", heads=2), tmp_path, monkeypatch, fused=False)


@pytest.mark.parametrize("n_parts", [1, 2, 3])
@pytest.mark.parametrize("heads,n_linear", [(1, 0), (2, 0), (2, 1)])
def test_transformer_partition_logits_equal_the_whole_graph_evaluation(built, heads, n_linear, n_parts):
    """Each rank's logits after one training epoch == the whole-graph evaluation's rows of its nodes, within the bar
    the GAT cases of test_parallel_eval_gpu use."""
    from bns_gcn_b200 import train
    from bns_gcn_b200.data import make_graph, partition_graph
    from bns_gcn_b200.helper.utils import get_layer_size
    from tests.harness import make_args
    from tests.test_parallel_eval_gpu import TOL, _full_handle, _parallel, _whole_graph
    fg = make_graph("tiny", seed=5)
    parts = partition_graph(fg, n_parts, "random", seed=0)
    args = make_args(n_partitions=n_parts, sampling_rate=0.5, dropout=0.3, eval=True, model="transformer",
                     heads=heads, n_linear=n_linear)
    res = _parallel(parts, args, DEV)
    sd = res[0][4]
    g, _ = _whole_graph(fg, n_parts, "random", DEV)
    a = argparse.Namespace(**vars(args))
    a.n_feat, a.n_class, a.n_train = fg.n_feat, fg.n_class, int(fg.train_mask.sum())
    net = train.create_model(get_layer_size(fg.n_feat, a.n_hidden, fg.n_class, a.n_layers), a)
    net.load_state_dict(sd, strict=True)
    net.to(DEV).eval()
    with torch.no_grad():
        full = net(_full_handle(g, DEV), g.feat.to(DEV)).cpu()
    assert torch.isfinite(full).all()
    for gid, logits, _, _, _ in res:
        assert _rel(logits, full[gid]) <= TOL, (heads, n_linear, n_parts)


@pytest.mark.parametrize("n_parts", [1, 2, 3])
@pytest.mark.parametrize("kw", [dict(heads=1), dict(heads=2), dict(heads=2, n_linear=1)],
                         ids=["1head", "2heads", "2heads-n-linear1"])
def test_transformer_inductive_eval_parts_equal_the_whole_graph_evaluator(built, kw, n_parts):
    """``--parallel-eval --inductive``: after one training epoch, each rank's logits on its part of the val graph and
    of the test graph == the whole-graph ``Evaluator``'s rows of the same nodes, within the bar and with the checks
    test_parallel_eval_inductive_gpu applies to GAT."""
    from bns_gcn_b200.data import make_graph
    from tests.harness import make_args
    from tests.test_parallel_eval_inductive_gpu import _check, _parallel
    fg = make_graph("tiny", seed=5)
    args = make_args(n_partitions=n_parts, sampling_rate=0.5, dropout=0.3, eval=True, parallel_eval=True,
                     inductive=True, model="transformer", **kw)
    _check(fg, args, _parallel(fg, args))


def test_main_trains_and_evaluates_a_transformer(built, tmp_path):
    """``python -m bns_gcn_b200.main --model transformer`` with heads, --cuda-graph and --parallel-eval prints its
    epoch lines and the test result."""
    from tests.test_cuda_graph_cli_gpu import _main
    out = _main(tmp_path, ["--dataset", "small", "--model", "transformer", "--heads", "2", "--n-hidden", "64",
                           "--n-layers", "3", "--n-partitions", "1", "--n-epochs", "4", "--log-every", "2",
                           "--cuda-graph", "--parallel-eval", "--fix-seed"])
    epochs = {int(e) for e in re.findall(r"Process 000 \| Epoch (\d+) \|", out)}
    assert 3 in epochs and epochs <= {0, 1, 2, 3}, out[-3000:]
    assert len(re.findall(r"Epoch 0000[13] \| (?:Validation )?Accuracy \d+\.\d\d%", out)) == 2, out[-3000:]
    assert len(re.findall(r"Test Result \| Accuracy \d+\.\d\d%", out)) == 1, out[-3000:]
