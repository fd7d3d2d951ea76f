"""``--model graphsage-pool`` end to end: one training epoch against the CPU oracle (``tests/sage_pool_oracle.py``:
``SAGEPoolConvRef`` on the oracle's explicit edge lists, run by its ``OracleRank`` with the exchange unscaled),
``--cuda-graph`` replays bit-identical to eager epochs, ``--resume`` bit for bit, the exchange's ratio, and the
partition-parallel evaluation (transductive and inductive) against the whole-graph ``Evaluator``."""
import argparse

import pytest
import torch

from tests.sage_pool_oracle import oracle_kind
from tests.test_parity_gpu import TOL

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
AMPLIFIED = 1e-4        # |g| / max |g| below which Adam's step is decided by rounding noise


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / b.norm().clamp(min=1e-30)).item()


@pytest.mark.parametrize("kw", [
    dict(n_parts=1, sampling_rate=1.0),
    dict(n_parts=2, sampling_rate=1.0),
    dict(n_parts=3, sampling_rate=0.5),
    dict(n_parts=3, sampling_rate=0.3, backend="p2p", n_layers=3),
    dict(n_parts=2, sampling_rate=0.5, shape="tiny"),
    dict(n_parts=2, sampling_rate=0.5, n_layers=3, n_linear=1),
    dict(n_parts=2, sampling_rate=0.7, n_layers=3, norm="batch"),
    dict(n_parts=3, sampling_rate=0.4, backend="p2p", shape="tiny", norm="batch", n_linear=1, n_layers=3),
], ids=["p1", "p2", "p3", "p3-p2p", "tiny-ce", "p2-n-linear1", "p2-batch", "p3-p2p-ce-batch-n-linear1"])
def test_sage_pool_training_parity(built, monkeypatch, kw):
    from bns_gcn_b200.data import make_graph, partition_graph
    from tests import harness
    kw = dict(kw)
    shape = kw.pop("shape", "tiny-ml")
    P = kw.pop("n_parts")
    bn = kw.get("norm") == "batch"
    # --norm batch divides its column sums by the number of train nodes (test_parity_gpu's sync-bn case): every node
    # trains.  Then the batch norm's mean subtraction makes sum_v d rst_v = 0 per column, and gradients built from that
    # sum cancel: the bias of a graph layer in front of the norm (exactly 0), and an fc_pool column whose every row has a
    # winner with z > 0 (sum over the winners of d m = W_neigh^T sum_v d rst_v = 0).  Such a gradient is rounding noise
    # of either implementation, and Adam's first step turns it into anything in [-lr, lr]: those weights are held to
    # the bound of the step, 2 lr (the pre-norm biases' gradients are not compared; see test_gatv2_parity_gpu).
    fg = make_graph(shape, seed=0, **({"train": 1.0} if bn else {}))
    parts = partition_graph(fg, P, "random", seed=0)
    args = harness.make_args(dataset=shape, model="graphsage-pool", n_partitions=P, multilabel=(shape == "tiny-ml"),
                             **{"n_layers": 2, **kw})
    noise = {5 * i for i in range(args.n_layers - 1)} if bn else set()     # layers.i.bias: parameter 5 i
    prod = harness.run_product(parts, args, "cuda:0", 1)
    selected = [[prod[r]["selected"][0] for r in range(P)]]
    with oracle_kind(monkeypatch):
        orc = harness.run_oracle(parts, args, 1, selected if P > 1 else None)
    for r in range(P):
        for k in list(prod[r]["layers"]) + ["logits", "feat0"]:
            a = prod[r]["layers"][k] if k.startswith("layer") else prod[r][k]
            b = orc[r]["layers"][k] if k.startswith("layer") else orc[r][k]
            assert _rel(a, b) < TOL, (r, k, _rel(a, b))
        assert abs(prod[r]["loss"][0] - orc[r]["loss"][0]) <= 1e-4 * abs(orc[r]["loss"][0]), r
        for i, (a, b) in enumerate(zip(prod[r]["grads"], orc[r]["grads"])):
            assert i in noise or _rel(a, b) < TOL, (r, "grad", i, _rel(a, b))
        for i, (a, b, g) in enumerate(zip(prod[r]["params"], orc[r]["params"], orc[r]["grads"])):
            diff = (a - b).abs()
            noisy = (g.abs() < AMPLIFIED * g.abs().max()) | (i in noise) if bn else torch.zeros_like(diff, dtype=bool)
            assert diff[~noisy].norm() < TOL * b.norm(), (r, "param", i, (diff[~noisy].norm() / b.norm()).item())
            assert torch.all(diff[noisy] <= 2 * args.lr * (1 + 1e-5)), (r, "param", i)
        for j in range(P):
            if j != r:
                assert torch.equal(prod[j]["one_hops"][0][r], prod[r]["selected"][0][j])


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
        a = make_args(model="graphsage-pool", n_partitions=3, sampling_rate=0.3, n_layers=2)
        a.n_feat, a.n_class, a.n_train = p.meta["n_feat"], p.meta["n_class"], p.meta["n_train"]
        st = train.setup(p.graph, p.node_dict, p.gpb, a, DEV)
        return list(st.ratio), train.get_send_size(st.boundary, 0.3)[1]
    for r, (ratio, shares) in enumerate(run_threads(3, fn, device=DEV)):
        assert ratio == [0 if i == r else 1.0 for i in range(3)]
        assert all(0 < x < 1 for i, x in enumerate(shares) if i != r)


@pytest.mark.parametrize("kw", [dict(n_layers=2), dict(n_layers=3, n_linear=1)], ids=["2layers", "n-linear1"])
def test_sage_pool_replayed_run_equals_the_eager_run(built, tmp_path, monkeypatch, capsys, kw):
    from tests.test_cuda_graph_cli_gpu import _args, _check_same, _train
    kw = dict(model="graphsage-pool", **kw)
    eager = _train(_args(**kw), monkeypatch, capsys, tmp_path / "eager")
    graphed = _train(_args(cuda_graph=True, **kw), monkeypatch, capsys, tmp_path / "graph")
    _check_same(eager, graphed)
    assert eager["fused"] is False and graphed["fused"] is False


def test_sage_pool_resumes_bit_for_bit(built, tmp_path, monkeypatch):
    from tests.test_resume_gpu import _args, _check_resume
    _check_resume(_args(1, model="graphsage-pool"), tmp_path, monkeypatch, fused=False)


@pytest.mark.parametrize("n_parts", [1, 2, 3])
@pytest.mark.parametrize("n_linear", [0, 1])
def test_sage_pool_partition_logits_equal_the_whole_graph_evaluation(built, n_linear, n_parts):
    """Each rank's logits after one training epoch == the whole-graph evaluation's rows of its nodes, within 1e-5."""
    from bns_gcn_b200 import train
    from bns_gcn_b200.data import make_graph, partition_graph
    from bns_gcn_b200.helper.utils import get_layer_size
    from tests.harness import make_args
    from tests.test_parallel_eval_gpu import _full_handle, _parallel, _whole_graph
    fg = make_graph("tiny", seed=5)
    parts = partition_graph(fg, n_parts, "random", seed=0)
    args = make_args(n_partitions=n_parts, sampling_rate=0.5, dropout=0.3, eval=True, model="graphsage-pool",
                     n_linear=n_linear)
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
        assert _rel(logits, full[gid]) <= 1e-5, (n_linear, n_parts)


@pytest.mark.parametrize("n_parts", [1, 2, 3])
def test_sage_pool_inductive_eval_parts_equal_the_whole_graph_evaluator(built, monkeypatch, n_parts):
    """``--parallel-eval --inductive``: after one training epoch, each rank's logits on its part of the val graph and
    of the test graph == the whole-graph ``Evaluator``'s rows of the same nodes within 1e-5, with the other checks
    test_parallel_eval_inductive_gpu applies to GAT."""
    from bns_gcn_b200.data import make_graph
    from tests import test_parallel_eval_inductive_gpu as ind
    from tests.harness import make_args
    from tests.test_parallel_eval_inductive_gpu import _check, _parallel
    monkeypatch.setattr(ind, "TOL", 1e-5)
    fg = make_graph("tiny", seed=5)
    args = make_args(n_partitions=n_parts, sampling_rate=0.5, dropout=0.3, eval=True, parallel_eval=True,
                     inductive=True, model="graphsage-pool")
    _check(fg, args, _parallel(fg, args))
