"""``--save-state-every`` / ``--resume``: a run stopped after k epochs, torn down (new ``TrainState``, exchange buffers
and reducer, as a new process has) and resumed for k more epochs computes what the uninterrupted 2k-epoch run
computes, bit for bit: every per-epoch loss, every entry of the model's ``state_dict``, both Adam moments and the step
(``torch.equal``).

The fused step draws every random number from Philox keyed by the epoch, so this holds at any rank count; the op-by-op
path's ``nn.Dropout`` draws from torch's CUDA generator, which the state restores per rank, so those cases run one
rank."""
import argparse
import functools
import os
import re

import pytest
import torch

from tests.harness import make_args

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


@functools.lru_cache(maxsize=None)
def _parts(n: int, all_train: bool = False):
    """``all_train``: every node a training node (SyncBatchNorm divides its column sums over all inner nodes by the
    number of training nodes, as the reference does: a train fraction below 1 can make the variance negative)."""
    from bns_gcn_b200.data import make_graph, partition_graph
    return partition_graph(make_graph("small", seed=0, **({"train": 1.0} if all_train else {})), n, "random", seed=0)


def _args(n_parts, **kw):
    kw = {"dataset": "small", "n_hidden": 64, "dropout": 0.5, "sampling_rate": 0.3, "n_partitions": n_parts,
          "graph_name": f"small-{n_parts}-random-vol-trans", **kw}
    return make_args(**kw)


def _snapshot(st):
    from bns_gcn_b200.state import _cpu
    return {"model": _cpu(st.model.state_dict()), "optimizer": _cpu(st.optimizer.state_dict())}


def _equal(a, b, where=""):
    """Bitwise equality of two nested dicts / lists of tensors and plain values."""
    if isinstance(a, torch.Tensor):
        assert isinstance(b, torch.Tensor) and a.dtype == b.dtype and torch.equal(a, b), where
    elif isinstance(a, dict):
        assert set(a) == set(b), (where, sorted(a), sorted(b))
        for k in a:
            _equal(a[k], b[k], f"{where}/{k}")
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), where
        for i, (x, y) in enumerate(zip(a, b)):
            _equal(x, y, f"{where}[{i}]")
    else:
        assert a == b, (where, a, b)


def _phase(args, k: int, phase: str, graph_warmup: int = 0, all_train: bool = False):
    """``phase``: "whole" trains 2k epochs, "first" k epochs and saves, "second" resumes and trains k more.
    ``graph_warmup`` > 0: after the eager epochs (the first phase's, or a resumed run's), a ``train.GraphedEpoch`` with
    that many warm-up epochs runs the rest as replays.  Returns per rank ``{"loss": {epoch: loss}, "replayed": [epochs],
    "fused": bool, "model": ..., "optimizer": ...}``."""
    from bns_gcn_b200 import state, train
    from bns_gcn_b200.helper.comm import run_threads
    parts = _parts(args.n_partitions, all_train)

    def body(r):
        p = parts[r]
        a = argparse.Namespace(**vars(args))
        a.n_feat, a.n_class, a.n_train = p.meta["n_feat"], p.meta["n_class"], p.meta["n_train"]
        saved = state.load(a, r) if phase == "second" else None
        st = train.setup(p.graph, p.node_dict, p.gpb, a, DEV)
        start = state.restore(st, saved) if saved is not None else 0
        stop = start + (2 * k if phase == "whole" else k)
        losses, replayed = {}, []
        if graph_warmup and phase != "first":
            ge = train.GraphedEpoch(st, warmup=graph_warmup)
            e0 = start + graph_warmup
            for e in range(e0, stop):
                losses[e] = ge().detach().clone()
                replayed.append(e)
        else:
            for e in range(start, stop):
                losses[e] = train.train_epoch(st, e).detach().clone()
        torch.cuda.synchronize()
        assert int(st.epoch_dev.item()) == stop
        if phase == "first":
            state.save(st, stop)
        return dict(_snapshot(st), loss={e: v.cpu() for e, v in losses.items()}, replayed=replayed,
                    fused=st.arena is not None)

    def fn(comm, r):
        if args.n_partitions > 1:
            return body(r)
        # one rank runs on the calling thread: give it what run_threads gives several (own stream, autograd inline)
        dev = torch.device(DEV)
        prev, prev_stream = torch.autograd.is_multithreading_enabled(), torch.cuda.current_stream(dev)
        torch.autograd.set_multithreading_enabled(False)
        torch.cuda.set_stream(torch.cuda.Stream(dev))
        try:
            return body(r)
        finally:
            torch.cuda.synchronize(dev)
            torch.cuda.set_stream(prev_stream)
            torch.autograd.set_multithreading_enabled(prev)
    return run_threads(args.n_partitions, fn, device=DEV)


def _check_resume(args, tmp_path, monkeypatch, fused: bool, k: int = 3, all_train: bool = False):
    monkeypatch.chdir(tmp_path)
    whole = _phase(args, k, "whole", all_train=all_train)
    first = _phase(args, k, "first", all_train=all_train)
    second = _phase(args, k, "second", all_train=all_train)
    for r in range(args.n_partitions):
        assert whole[r]["fused"] is fused and second[r]["fused"] is fused
        for e in range(2 * k):
            got = (first if e < k else second)[r]["loss"][e]
            assert torch.isfinite(got), (r, e, got)
            assert torch.equal(got, whole[r]["loss"][e]), (r, e, got, whole[r]["loss"][e])
        _equal(second[r]["model"], whole[r]["model"], f"rank {r} model")
        _equal(second[r]["optimizer"], whole[r]["optimizer"], f"rank {r} optimizer")
    # the resumed epochs are not a replay of the first ones
    assert not torch.equal(whole[0]["loss"][k], whole[0]["loss"][0])
    return whole, second


@pytest.mark.parametrize("model", ["graphsage", "gcn"])
@pytest.mark.parametrize("n_parts,backend", [(1, "nccl"), (4, "p2p"), (4, "nccl")], ids=["p1", "p4-p2p", "p4-nccl"])
def test_fused_step_resumes_bit_for_bit(built, tmp_path, monkeypatch, model, n_parts, backend):
    whole, _ = _check_resume(_args(n_parts, model=model, backend=backend), tmp_path, monkeypatch, fused=True)
    step = whole[0]["optimizer"]["step"]
    assert step.dtype == torch.int64 and int(step) == 6


def test_fused_step_with_every_bf16_mode_resumes_bit_for_bit(built, tmp_path, monkeypatch):
    args = _args(4, backend="p2p", agg_dtype="bf16", comm_dtype="bf16", dense_dtype="bf16")
    _check_resume(args, tmp_path, monkeypatch, fused=True)


@pytest.mark.parametrize("kw", [dict(model="gat", heads=2, n_layers=2), dict(norm="batch"), dict(n_linear=1)],
                         ids=["gat-heads2", "batch-norm", "n-linear"])
def test_op_by_op_path_resumes_bit_for_bit(built, tmp_path, monkeypatch, kw):
    """One rank: GAT (its feature dropout's fallback is ``nn.Dropout``), ``--norm batch`` (SyncBatchNorm's running
    statistics are buffers of the state dict) and ``--n-linear 1`` at dropout 0.5 (its ``nn.Dropout`` draws from the
    CUDA generator the state restores)."""
    whole, second = _check_resume(_args(1, **kw), tmp_path, monkeypatch, fused=False,
                                  all_train=kw.get("norm") == "batch")
    if kw.get("norm") == "batch":
        assert any(k.endswith("running_mean") for k in second[0]["model"])


def test_op_by_op_resume_needs_the_cuda_generator(built, tmp_path, monkeypatch):
    """The control of the ``--n-linear`` case: without the generator's state the resumed masks differ."""
    import bns_gcn_b200.state as state_mod
    args = _args(1, n_linear=1)
    monkeypatch.chdir(tmp_path)
    whole = _phase(args, 3, "whole")
    _phase(args, 3, "first")
    monkeypatch.setattr(state_mod.torch.cuda, "set_rng_state", lambda *a, **kw: None)
    second = _phase(args, 3, "second")
    assert not torch.equal(second[0]["loss"][3], whole[0]["loss"][3])


def test_graphed_epoch_after_resume(built, tmp_path, monkeypatch):
    """``train.GraphedEpoch`` built on a resumed run (its warm-up and capture read ``epoch_dev`` and ``step_dev``; the
    flag sequence numbers start over in the new buffers): its replays equal the uninterrupted run's replays at the same
    epoch indices."""
    monkeypatch.chdir(tmp_path)
    args, k = _args(1), 4
    whole = _phase(args, k, "whole", graph_warmup=2)             # epochs 0, 1 eager, 2..7 replayed
    _phase(args, k, "first")                                     # epochs 0..3 eager, saved
    second = _phase(args, k, "second", graph_warmup=2)           # epochs 4, 5 eager, 6, 7 replayed
    assert whole[0]["replayed"] == list(range(2, 2 * k)) and second[0]["replayed"] == [6, 7]
    for e in (6, 7):
        assert torch.equal(second[0]["loss"][e], whole[0]["loss"][e]), e
    _equal(second[0]["model"], whole[0]["model"], "model")
    _equal(second[0]["optimizer"], whole[0]["optimizer"], "optimizer")


# ---- train.run end to end ---------------------------------------------------------------------------------------

def _run(args, fg):
    from bns_gcn_b200 import train
    from bns_gcn_b200.helper.comm import run_threads
    parts = _parts(args.n_partitions)

    def fn(comm, r):
        a = argparse.Namespace(**vars(args))
        p = parts[r]
        a.n_feat, a.n_class, a.n_train = p.meta["n_feat"], p.meta["n_class"], p.meta["n_train"]
        st, _ = train.run(p.graph, p.node_dict, p.gpb, a, DEV, full_graph=fg)
        return st.args.seed
    return run_threads(args.n_partitions, fn, device=DEV)


def _losses(out: str):
    """``{(process, epoch): loss text}`` of the run's log lines."""
    return {(int(m[0]), int(m[1])): m[2] for m in
            re.findall(r"Process (\d+) \| Epoch (\d+) \|.*\| Loss (\S+)", out)}


@pytest.mark.parametrize("parallel", [False, True], ids=["eval", "parallel-eval"])
def test_run_resumes_with_evaluation(built, tmp_path, monkeypatch, capsys, parallel):
    """``train.run`` at 2 in-process ranks, ``--eval`` (rank 0 evaluates the full graph) or ``--parallel-eval``:
    8 epochs saving every 4, against 4 epochs and a ``--resume`` to 8.  The result lines, the log's losses of epochs
    4-7, "Max Validation Accuracy", the test line and the final checkpoint are identical; the periodic checkpoints stay
    plain state dicts."""
    from bns_gcn_b200 import state, train
    from bns_gcn_b200.data import make_graph
    from bns_gcn_b200.evaluate import checkpoint_path, load_checkpoint, result_file_name
    from bns_gcn_b200.helper.utils import get_layer_size
    fg = None if parallel else make_graph("small", seed=0)
    base = _args(2, backend="p2p", eval=True, parallel_eval=parallel, log_every=2, save_state_every=4, seed=5)
    meta = _parts(2)[0].meta
    base.n_feat, base.n_class, base.n_train = meta["n_feat"], meta["n_class"], meta["n_train"]
    outs, files = {}, {}
    for name, runs in (("whole", [dict(n_epochs=8)]), ("split", [dict(n_epochs=4), dict(n_epochs=8, resume=True)])):
        d = tmp_path / name
        d.mkdir()
        monkeypatch.chdir(d)
        capsys.readouterr()
        for kw in runs:
            seeds = _run(argparse.Namespace(**dict(vars(base), **kw)), fg)
            assert seeds == [5, 5]
        outs[name] = capsys.readouterr().out
        with open(result_file_name(base)) as f:
            files[name] = f.read().splitlines()
        files[name + "_final"] = torch.load(checkpoint_path(base))
        files[name + "_state"] = state.load(base, 0)
    assert "resumes after 4 epochs" in outs["split"]
    assert len(files["whole"]) == 4 and files["split"] == files["whole"]
    lw, ls = _losses(outs["whole"]), _losses(outs["split"])
    for key in [(r, e) for r in range(2) for e in (5, 7)]:
        assert ls[key] == lw[key], key
    for pat in (r"Max Validation Accuracy .*", r"Test Result \| Accuracy .*"):
        assert re.findall(pat, outs["split"])[-1] == re.findall(pat, outs["whole"])[-1]
    _equal(files["split_final"], files["whole_final"], "final checkpoint")
    for key in ("model", "optimizer", "best_model", "best_acc", "epochs", "seed"):
        _equal(files["split_state"][key], files["whole_state"][key], key)
    # the reference-format checkpoints keep their format
    monkeypatch.chdir(tmp_path / "split")
    net = train.create_model(get_layer_size(base.n_feat, base.n_hidden, base.n_class, base.n_layers), base)
    for e in (1, 3, 5, 7):
        assert os.path.exists(checkpoint_path(base, e))
        load_checkpoint(net, checkpoint_path(base, e))
        sd = torch.load(checkpoint_path(base, e))
        assert list(sd) == [k for k, _ in net.named_parameters()]
