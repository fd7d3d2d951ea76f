"""Partition-parallel evaluation of inductive runs (``--eval --parallel-eval --inductive``): each rank's logits on its
part of the val graph (the train | val subgraph) and of the test graph (the full graph) against the whole-graph
``Evaluator``'s, the summed counts, ``train.run``'s driver with ``eval_parts`` against the rank-0 ``Evaluator`` run,
and a resume."""
import argparse
import os
import re

import pytest
import torch

pytestmark = pytest.mark.gpu

TOL = 1e-4
DEV = torch.device("cuda:0")


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / b.norm().clamp(min=1e-30)).item()


def _eval_parts(fg, args):
    from bns_gcn_b200.data import eval_partitions
    return {w: eval_partitions(fg, w, args) for w in ("val", "test")}


def _parallel(fg, args, train_epochs=1):
    """Every rank: setup on its inductive training part, ``train_epochs`` epochs, then the inductive
    ``ParallelEvaluator`` on its evaluation parts.  Returns per rank {which: (global ids in that graph's partition
    numbering, logits, counts)} and the state dict.  Training needs ``--use-pp`` (the feature buffer refuses a run
    without it, as the reference's does), so a model without it is evaluated at its seeded initial weights."""
    import copy
    from bns_gcn_b200 import train
    from bns_gcn_b200.data import partition_graph
    from bns_gcn_b200.evaluate import ParallelEvaluator, acc_counts
    from bns_gcn_b200.helper.comm import run_threads
    from bns_gcn_b200.helper.utils import get_layer_size
    P = args.n_partitions
    parts = partition_graph(fg, P, args.partition_method, seed=0, inductive=True)
    ev_parts = _eval_parts(fg, args)
    initial = None
    if not args.use_pp:
        a = argparse.Namespace(**vars(args))
        a.n_feat, a.n_class, a.n_train = fg.n_feat, fg.n_class, int(fg.train_mask.sum())
        torch.manual_seed(a.seed)
        initial = train.create_model(get_layer_size(fg.n_feat, a.n_hidden, fg.n_class, a.n_layers), a)

    def fn(comm, r):
        p = parts[r]
        a = argparse.Namespace(**vars(args))
        a.n_feat, a.n_class, a.n_train = p.meta["n_feat"], p.meta["n_class"], p.meta["n_train"]
        if initial is None:
            st = train.setup(p.graph, p.node_dict, p.gpb, a, DEV)
            for e in range(train_epochs):
                train.train_epoch(st, e)
            model = st.model
        else:
            model = copy.deepcopy(initial).to(DEV)
        mine = {w: (q[r].graph, q[r].node_dict, q[r].gpb) for w, q in ev_parts.items()}
        ev = ParallelEvaluator.inductive_from_parts(a, mine, DEV, comm)
        out = {}
        for w in ("val", "test"):
            if w == "test":
                ev.use_test_graph()
            logits = ev.logits(model)
            mask = ev.val_mask if w == "val" else ev.test_mask
            c = acc_counts(logits[mask], ev.labels[mask])
            comm.all_reduce_sum(c)
            gid = ev_parts[w][r].node_dict["_ID"][:ev_parts[w][r].graph.n_in]
            out[w] = (gid.cpu(), logits.cpu(), c.cpu())
        sd = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
        return out, sd
    return run_threads(P, fn, device=str(DEV))


def _whole(fg, args, sd):
    """The whole-graph ``Evaluator``'s logits on ``val_g`` / ``test_g``, each with the map from the evaluation
    partition's node ids to that graph's."""
    from bns_gcn_b200 import train
    from bns_gcn_b200.data.partition import assign_parts
    from bns_gcn_b200.data.store import eval_graph_of
    from bns_gcn_b200.evaluate import eval_graphs
    from bns_gcn_b200.helper.utils import get_layer_size
    a = argparse.Namespace(**vars(args))
    a.n_feat, a.n_class, a.n_train = fg.n_feat, fg.n_class, int(fg.train_mask.sum())
    net = train.create_model(get_layer_size(fg.n_feat, a.n_hidden, fg.n_class, a.n_layers), a)
    net.load_state_dict(sd, strict=True)
    net.to(DEV).eval()
    val_g, test_g = eval_graphs(fg, True, DEV)
    out = {}
    for w, g in (("val", val_g), ("test", test_g)):
        with torch.no_grad():
            logits = net(g.handle, g.ndata["feat"]).cpu()
        part = assign_parts(eval_graph_of(fg, w), args.n_partitions, args.partition_method, 0, "vol", None)
        out[w] = (logits, torch.argsort(part, stable=True), g.ndata["label"].cpu(), g.ndata[w + "_mask"].cpu())
    return out


def _close_calls(full, labels, mask, tol):
    """Masked nodes (multi-label: entries) whose whole-graph decision lies within ``tol`` of flipping."""
    f = full[mask]
    if labels.dim() > 1:
        return int((f.abs() <= tol * full.abs().max()).sum())
    top2 = f.topk(2, dim=1).values
    return int(((top2[:, 0] - top2[:, 1]) <= tol * full.abs().max()).sum())


def _check(fg, args, res):
    from bns_gcn_b200.evaluate import acc_counts
    sd = res[0][1]
    for r in range(1, len(res)):
        assert all(torch.equal(sd[k], res[r][1][k]) for k in sd)          # the weights are replicated
    whole = _whole(fg, args, sd)
    for w in ("val", "test"):
        full, orig, labels, mask = whole[w]
        assert torch.isfinite(full).all() and mask.any()
        seen = torch.zeros(full.shape[0], dtype=torch.bool)
        for out, _ in res:
            gid, logits, counts = out[w]
            ids = orig[gid]
            seen[ids] = True
            assert logits.shape == (gid.numel(), fg.n_class)
            assert _rel(logits, full[ids]) <= TOL, (w, _rel(logits, full[ids]))
        assert seen.all()                                                  # every node of that graph is some rank's
        want = acc_counts(full[mask], labels[mask])
        got = res[0][0][w][2]
        assert all(torch.equal(o[w][2], got) for o, _ in res)             # every rank holds the same sums
        if not torch.equal(got, want):
            # only a decision within the tolerance of flipping may differ
            assert (got - want).abs().max() <= _close_calls(full, labels, mask, TOL), (w, got, want)
            assert _close_calls(full, labels, mask, TOL) > 0, (w, got, want)


MODELS = {
    "graphsage": dict(model="graphsage"),
    "graphsage-no-pp": dict(model="graphsage", use_pp=False),
    "graphsage-batchnorm": dict(model="graphsage", norm="batch"),
    "graphsage-linear": dict(model="graphsage", n_linear=1),
    "gcn": dict(model="gcn"),
    "gcn-no-pp": dict(model="gcn", use_pp=False),
    "gcn-batchnorm": dict(model="gcn", norm="batch"),
    "graphsage-multilabel": dict(model="graphsage", shape="tiny-ml", multilabel=True),
    "gat-1head": dict(model="gat", heads=1),
    "gat-2heads": dict(model="gat", heads=2),
}


@pytest.mark.parametrize("n_parts", [1, 2, 3])
@pytest.mark.parametrize("case", sorted(MODELS))
def test_eval_part_logits_equal_the_whole_graph_evaluator(built, case, n_parts):
    """After one training epoch on ``tiny`` (without ``--use-pp``: the initial weights), each rank's logits on its part
    of the val graph and of the test graph == the whole-graph ``Evaluator``'s rows of the same nodes (1e-4); the summed
    counts == the whole graph's."""
    from bns_gcn_b200.data import make_graph
    from tests.harness import make_args
    kw = dict(MODELS[case])
    fg = make_graph(kw.pop("shape", "tiny"), seed=5)
    args = make_args(n_partitions=n_parts, sampling_rate=0.5, dropout=0.3, eval=True, parallel_eval=True,
                     inductive=True, **kw)
    _check(fg, args, _parallel(fg, args))


def test_metis_eval_parts_equal_the_whole_graph_evaluator(built):
    from bns_gcn_b200.data import make_graph
    from tests.harness import make_args
    fg = make_graph("small", seed=0)
    args = make_args(dataset="small", n_partitions=3, partition_method="metis", sampling_rate=0.5, n_hidden=32,
                     eval=True, parallel_eval=True, inductive=True)
    _check(fg, args, _parallel(fg, args))


# ---- the driver -----------------------------------------------------------------------------------------------------

def _driver(tmp_path, monkeypatch, parallel, n_parts=2, **kw):
    """``train.run`` at ``n_parts`` in-process ranks, inductive, in ``tmp_path``: with ``--parallel-eval`` and
    ``eval_parts`` (the whole graph's builders raise), or the rank-0 ``Evaluator`` on the given full graph."""
    from bns_gcn_b200 import train
    from bns_gcn_b200.data import make_graph, partition_graph
    from bns_gcn_b200.helper.comm import run_threads
    from tests.harness import make_args
    fg = make_graph("tiny", seed=0)
    parts = partition_graph(fg, n_parts, "random", seed=0, inductive=True)
    args = make_args(**dict(dict(dataset="tiny", model="graphsage", sampling_rate=0.5, dropout=0.3,
                                 n_partitions=n_parts, n_epochs=6, log_every=2, eval=True, parallel_eval=parallel,
                                 inductive=True, graph_name=f"tiny-{n_parts}-random-vol-induc"), **kw))
    m = parts[0].meta
    args.n_feat, args.n_class, args.n_train = m["n_feat"], m["n_class"], m["n_train"]
    ev_parts = _eval_parts(fg, args) if parallel else None
    os.makedirs(tmp_path, exist_ok=True)
    monkeypatch.chdir(tmp_path)
    if parallel:
        def no_whole_graph(*a, **k):
            raise AssertionError("the whole graph must not be built under --parallel-eval")
        for name in ("bns_gcn_b200.data.make_graph", "bns_gcn_b200.data.load_graph",
                     "bns_gcn_b200.data.files.load_graph", "bns_gcn_b200.data.store.load_graph"):
            monkeypatch.setattr(name, no_whole_graph)

    def fn(comm, r):
        a = argparse.Namespace(**vars(args))
        p = parts[r]
        a.n_feat, a.n_class, a.n_train = p.meta["n_feat"], p.meta["n_class"], p.meta["n_train"]
        if parallel:
            mine = {w: (q[r].graph, q[r].node_dict, q[r].gpb) for w, q in ev_parts.items()}
            train.run(p.graph, p.node_dict, p.gpb, a, DEV, eval_parts=mine)
        else:
            train.run(p.graph, p.node_dict, p.gpb, a, DEV, full_graph=fg)
    try:
        run_threads(n_parts, fn, device=str(DEV))
    finally:
        monkeypatch.undo()
    return args


def test_run_with_eval_parts_matches_the_rank0_evaluator(built, tmp_path, monkeypatch, capsys):
    """The same ``Epoch ... | Accuracy`` lines (printed and in the result file), ``Max Validation Accuracy`` and
    ``Test Result`` line, and the same checkpoints as the whole-graph run; each line printed once (by rank 0)."""
    from bns_gcn_b200.evaluate import checkpoint_path, result_file_name
    outs, files = {}, {}
    for name, parallel in (("whole", False), ("parallel", True)):
        capsys.readouterr()
        args = _driver(tmp_path / name, monkeypatch, parallel)
        outs[name] = capsys.readouterr().out
        d = tmp_path / name
        with open(d / result_file_name(args)) as f:
            files[name] = f.read().splitlines()
        files[name + "_ckpt"] = {e: torch.load(d / checkpoint_path(args, e)) for e in (1, 3, 5)}
        files[name + "_final"] = torch.load(d / checkpoint_path(args))
    assert len(files["whole"]) == 3 and all(re.fullmatch(r"Epoch \d{5} \| Accuracy \d+\.\d\d%", ln)
                                            for ln in files["whole"]), files["whole"]
    assert files["parallel"] == files["whole"]
    for pat in (r"Epoch \d{5} \| Accuracy .*", r"Max Validation Accuracy .*", r"Test Result \| Accuracy .*"):
        assert re.findall(pat, outs["parallel"]) == re.findall(pat, outs["whole"]), pat
    assert outs["parallel"].count("Test Result | Accuracy") == 1 and outs["parallel"].count("model saved") == 1
    for key in ("_ckpt", "_final"):
        w, p = files["whole" + key], files["parallel" + key]
        for sd_w, sd_p in ([(w[e], p[e]) for e in w] if key == "_ckpt" else [(w, p)]):
            assert list(sd_w) == list(sd_p) and all(torch.equal(sd_w[k], sd_p[k]) for k in sd_w)


def test_resume_with_parallel_eval_inductive_restores_the_best_model(built, tmp_path, monkeypatch, capsys):
    """6 epochs saving every 2, against 2 epochs and a ``--resume`` to 6: the result lines, ``Max Validation
    Accuracy``, the test line, the final checkpoint and the saved ``best_acc`` / ``best_model`` are identical."""
    from bns_gcn_b200 import state
    from bns_gcn_b200.evaluate import checkpoint_path, result_file_name
    outs, files = {}, {}
    for name, runs in (("whole", [dict(n_epochs=6)]), ("split", [dict(n_epochs=2), dict(n_epochs=6, resume=True)])):
        capsys.readouterr()
        for kw in runs:
            args = _driver(tmp_path / name, monkeypatch, True, save_state_every=2, seed=5, **kw)
        outs[name] = capsys.readouterr().out
        monkeypatch.chdir(tmp_path / name)
        with open(result_file_name(args)) as f:
            files[name] = f.read().splitlines()
        files[name + "_final"] = torch.load(checkpoint_path(args))
        files[name + "_state"] = state.load(args, 0)
        monkeypatch.undo()
    assert "resumes after 2 epochs" in outs["split"]
    assert len(files["whole"]) == 3 and files["split"] == files["whole"]
    for pat in (r"Max Validation Accuracy .*", r"Test Result \| Accuracy .*"):
        assert re.findall(pat, outs["split"])[-1] == re.findall(pat, outs["whole"])[-1]
    w, s = files["whole_final"], files["split_final"]
    assert all(torch.equal(w[k], s[k]) for k in w)
    ws, ss = files["whole_state"], files["split_state"]
    assert ws["best_acc"] == ss["best_acc"] and ws["best_acc"] > 0
    assert all(torch.equal(ws["best_model"][k], ss["best_model"][k]) for k in ws["best_model"])


# ---- the bench shape ------------------------------------------------------------------------------------------------

def test_reddit_shape_inductive_eval_parts_equal_the_whole_graph(built):
    """The Reddit shape at 4 in-process ranks, inductive: 3-layer GraphSAGE, hidden 256, --use-pp, after one training
    epoch at sampling rate 0.1 -- each rank's val and test logits within 1e-4 of the whole-graph evaluation."""
    free, _ = torch.cuda.mem_get_info(0)
    if free / 2 ** 30 < 40:
        pytest.skip("needs ~40 GB of free device memory (full-size graph + 4 in-process ranks)")
    from bns_gcn_b200.data import make_graph
    from tests.harness import make_args
    fg = make_graph("reddit", seed=0)
    args = make_args(dataset="reddit", model="graphsage", n_layers=3, n_hidden=256, sampling_rate=0.1, dropout=0.5,
                     n_partitions=4, eval=True, parallel_eval=True, inductive=True, backend="p2p")
    res = _parallel(fg, args)
    sd = res[0][1]
    whole = _whole(fg, args, sd)
    for w in ("val", "test"):
        full, orig = whole[w][0], whole[w][1]
        for out, _ in res:
            gid, logits, _ = out[w]
            assert _rel(logits, full[orig[gid]]) <= TOL, w
