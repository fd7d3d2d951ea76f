"""``--cuda-graph`` on the GPU: ``train.run`` with the flag trains what the same run without it trains, bit for bit --
every printed loss, the final weights, Adam's moments and step, the evaluation lines, the saved state -- and a run
resumed across the two modes ends where the uninterrupted run ends.  The stamp kernel behind the graph mode's
``Comm(s)`` / ``Reduce(s)`` agrees with CUDA events.  The command line runs end to end, on one GPU and (skipped on a
box with fewer GPUs) under torchrun at world 2 and 4."""
import argparse
import functools
import math
import os
import re
import subprocess
import sys

import pytest
import torch

from tests.harness import make_args

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_EPOCHS = 8


@functools.lru_cache(maxsize=None)
def _graph(all_train: bool = False, inductive: bool = False):
    from bns_gcn_b200.data import make_graph, partition_graph
    fg = make_graph("small", seed=0, **({"train": 1.0} if all_train else {}))
    return fg, partition_graph(fg, 1, "random", seed=0, inductive=inductive)


def _args(**kw):
    kw = {"dataset": "small", "n_hidden": 64, "dropout": 0.5, "sampling_rate": 0.3, "n_epochs": N_EPOCHS,
          "log_every": 1, "seed": 3, **kw}
    kw.setdefault("graph_name", f"small-1-random-vol-{'induc' if kw.get('inductive') else 'trans'}")
    return make_args(**kw)


def _losses(out: str):
    return {int(m[0]): m[1] for m in re.findall(r"Process 000 \| Epoch (\d+) \|.*\| Loss (\S+)", out)}


def _cpu(sd):
    from bns_gcn_b200.state import _cpu
    return _cpu(sd)


def _equal(a, b, where=""):
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


def _steps(opt):
    """Adam's step counter(s): the fused step's device counter, or torch Adam's per-parameter steps."""
    if hasattr(opt, "step_dev"):
        return {int(opt.step_dev.item())}
    return {int(s["step"].item()) for s in opt.state.values()}


def _train(args, monkeypatch, capsys, cwd, fg=None, all_train=False):
    """One rank of ``train.run`` in ``cwd``; returns its stdout, the final state and the number of replays."""
    from bns_gcn_b200 import train
    from bns_gcn_b200.data import eval_partitions
    from bns_gcn_b200.helper.comm import run_threads
    graph, parts = _graph(all_train, args.inductive)
    p = parts[0]
    replays = []

    class Counting(train.GraphedEpoch):
        def __call__(self):
            replays.append(1)
            return super().__call__()
    monkeypatch.setattr(train, "GraphedEpoch", Counting)
    eval_parts = None
    if args.eval and getattr(args, "parallel_eval", False) and args.inductive:
        eval_parts = {w: eval_partitions(graph, w, args) for w in ("val", "test")}

    def fn(comm, r):
        a = argparse.Namespace(**vars(args))
        a.n_feat, a.n_class, a.n_train = p.meta["n_feat"], p.meta["n_class"], p.meta["n_train"]
        mine = None if eval_parts is None else {w: (q[0].graph, q[0].node_dict, q[0].gpb) for w, q in eval_parts.items()}
        st, res = train.run(p.graph, p.node_dict, p.gpb, a, DEV, full_graph=fg, eval_parts=mine)
        return {"model": _cpu(st.model.state_dict()), "optimizer": _cpu(st.optimizer.state_dict()),
                "epochs": int(st.epoch_dev.item()), "steps": _steps(st.optimizer), "loss": res["loss"],
                "fused": st.arena is not None}
    os.makedirs(cwd, exist_ok=True)
    monkeypatch.chdir(cwd)
    capsys.readouterr()
    try:
        out = run_threads(1, fn)[0]
    finally:
        monkeypatch.undo()
    out["stdout"] = capsys.readouterr().out
    out["replays"] = len(replays)
    return out


def _check_same(eager, graphed, n_epochs=N_EPOCHS, start=0):
    le, lg = _losses(eager["stdout"]), _losses(graphed["stdout"])
    assert sorted(le) == list(range(start, n_epochs)) and lg == le, (le, lg)
    assert eager["loss"] == graphed["loss"] and math.isfinite(graphed["loss"])
    _equal(graphed["model"], eager["model"], "model")
    _equal(graphed["optimizer"], eager["optimizer"], "optimizer")
    assert graphed["epochs"] == eager["epochs"] == n_epochs
    assert graphed["steps"] == eager["steps"] == {n_epochs}
    assert eager["replays"] == 0 and graphed["replays"] == n_epochs - start - min(3, n_epochs - start)


@pytest.mark.parametrize("kw", [
    dict(model="graphsage", n_layers=3),
    dict(model="graphsage", n_layers=4),
    dict(model="gcn", n_layers=3),
    dict(model="graphsage", n_layers=3, agg_dtype="fp8", dense_dtype="bf16"),
    dict(model="gat", heads=2, n_layers=2),
    dict(model="graphsage", n_layers=3, n_linear=1),
    dict(model="graphsage", n_layers=3, norm="batch"),
], ids=["sage3", "sage4", "gcn", "sage-fp8-bf16", "gat-heads2", "n-linear1", "batch-norm"])
def test_replayed_run_equals_the_eager_run(built, tmp_path, monkeypatch, capsys, kw):
    all_train = kw.get("norm") == "batch"
    eager = _train(_args(**kw), monkeypatch, capsys, tmp_path / "eager", all_train=all_train)
    graphed = _train(_args(cuda_graph=True, **kw), monkeypatch, capsys, tmp_path / "graph", all_train=all_train)
    _check_same(eager, graphed)
    assert eager["fused"] is graphed["fused"] is (kw.get("model") != "gat" and "n_linear" not in kw
                                                  and "norm" not in kw)
    # Time(s) of the timed epochs (5 .. 7); one rank exchanges and all-reduces nothing
    for line in re.findall(r"Epoch 0000[5-7] \|.*", graphed["stdout"]):
        t, c, r = (float(x) for x in re.search(r"Time\(s\) (\S+) \| Comm\(s\) (\S+) \| Reduce\(s\) (\S+)", line).groups())
        assert t > 0 and c == 0.0 and r == 0.0, line


@pytest.mark.parametrize("parallel", [False, True], ids=["whole-graph", "parallel-inductive"])
def test_evaluation_between_replays(built, tmp_path, monkeypatch, capsys, parallel):
    """``--eval`` on the whole graph (transductive), and ``--eval --parallel-eval --inductive``: every accuracy line,
    the best model and the test line equal the eager run's."""
    kw = dict(eval=True, log_every=2)
    if parallel:
        kw.update(parallel_eval=True, inductive=True)
    fg = None if parallel else _graph()[0]
    eager = _train(_args(**kw), monkeypatch, capsys, tmp_path / "eager", fg=fg)
    graphed = _train(_args(cuda_graph=True, **kw), monkeypatch, capsys, tmp_path / "graph", fg=fg)
    assert graphed["replays"] == N_EPOCHS - 3
    _equal(graphed["model"], eager["model"], "model")
    pats = [r"Epoch \d{5} \| (?:Validation )?Accuracy .*", r"Max Validation Accuracy .*", r"Test Result \| Accuracy .*"]
    for pat in pats:
        got, want = re.findall(pat, graphed["stdout"]), re.findall(pat, eager["stdout"])
        assert got == want and want, (pat, got, want)
    assert len(re.findall(pats[0], eager["stdout"])) == N_EPOCHS // 2


def _state_files(cwd, args):
    from bns_gcn_b200 import state
    d = state._current(os.path.join(str(cwd), state.state_dir(args)))
    return {n: open(os.path.join(d, n), "rb").read() for n in ("shared.pt", "rank0.pt")}


@pytest.mark.parametrize("kw", [dict(), dict(n_linear=1)], ids=["fused", "op-by-op"])
def test_state_and_resume_across_modes(built, tmp_path, monkeypatch, capsys, kw):
    """The state saved after 8 epochs under ``--cuda-graph`` is byte-equal to the eager run's.  Eager 4 epochs resumed
    to 8 with ``--cuda-graph``, and ``--cuda-graph`` 4 epochs (3 eager, 1 replay) resumed eagerly to 8, end with the
    uninterrupted run's weights, Adam state and counters."""
    save = dict(save_state_every=4, **kw)
    whole = _train(_args(**save), monkeypatch, capsys, tmp_path / "whole")
    whole_g = _train(_args(cuda_graph=True, **save), monkeypatch, capsys, tmp_path / "whole_g")
    _check_same(whole, whole_g)
    a = _args(**save)
    assert _state_files(tmp_path / "whole_g", a) == _state_files(tmp_path / "whole", a)
    for first, second in ((False, True), (True, False)):
        d = tmp_path / f"split_{int(first)}{int(second)}"
        one = _train(_args(n_epochs=4, cuda_graph=first, **save), monkeypatch, capsys, d)
        assert one["replays"] == (1 if first else 0) and one["epochs"] == 4
        two = _train(_args(resume=True, cuda_graph=second, **save), monkeypatch, capsys, d)
        assert "resumes after 4 epochs" in two["stdout"]
        assert two["replays"] == (1 if second else 0)          # epochs 4, 5, 6 eager, 7 replayed
        _equal(two["model"], whole["model"], "model")
        _equal(two["optimizer"], whole["optimizer"], "optimizer")
        assert two["epochs"] == N_EPOCHS and two["steps"] == {N_EPOCHS}
        lw, l1, l2 = _losses(whole["stdout"]), _losses(one["stdout"]), _losses(two["stdout"])
        assert {**l1, **l2} == lw


# ---- the stamps -----------------------------------------------------------------------------------------------------

def test_stamps_time_a_known_kernel_like_events(built):
    """Two stamps captured around ``torch.cuda._sleep`` give, per replay, the interval CUDA events give around the same
    kernel launched eagerly: medians of 5 alternating measurements within 10 % + 20 us (the kernel spins for a fixed
    number of cycles, so clock changes between the two launches move both sides)."""
    from bns_gcn_b200 import ops
    dev = torch.device(DEV)
    s = torch.cuda.Stream(dev)
    cycles = 20_000_000
    with torch.cuda.stream(s):
        slots = torch.zeros(2, dtype=torch.int64, device=dev)
        torch.cuda._sleep(cycles)
        ops.stamp_globaltimer(slots[0:1])
        torch.cuda.synchronize(dev)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            ops.stamp_globaltimer(slots[0:1])
            torch.cuda._sleep(cycles)
            ops.stamp_globaltimer(slots[1:2])
        ev_ms, st_ms = [], []
        for _ in range(5):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(s)
            torch.cuda._sleep(cycles)
            e1.record(s)
            torch.cuda.synchronize(dev)
            ev_ms.append(e0.elapsed_time(e1))
            slots.fill_(-1)
            g.replay()
            torch.cuda.synchronize(dev)
            v = slots.cpu()
            assert v[1] > v[0] > 0, v
            st_ms.append(int(v[1] - v[0]) * 1e-6)
    ev, st = sorted(ev_ms)[2], sorted(st_ms)[2]
    print(f"[stamps] sleep {cycles} cycles: events {ev:.4f} ms, stamps {st:.4f} ms")
    assert abs(st - ev) <= 0.1 * ev + 0.02, (ev_ms, st_ms)


def test_stamps_are_monotone_within_a_replay(built):
    """A captured chain of stamps on two streams (the second forked from the first and joined back, as the comm and
    reducer streams are): every stamp is at least the one before it in stream order, across three replays, and each
    replay's stamps are later than the previous replay's."""
    from bns_gcn_b200 import ops
    dev = torch.device(DEV)
    main, side = torch.cuda.Stream(dev), torch.cuda.Stream(dev)
    n = 8
    with torch.cuda.stream(main):
        slots = torch.zeros(3 * n, dtype=torch.int64, device=dev)
        ops.stamp_globaltimer(slots[0:1])
        torch.cuda.synchronize(dev)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=main):
            for i in range(n):
                ops.stamp_globaltimer(slots[i:i + 1])
                torch.cuda._sleep(20_000 * (i % 3))
            side.wait_stream(main)
            for i in range(n, 2 * n):
                ops.stamp_globaltimer(slots[i:i + 1], side)
                with torch.cuda.stream(side):
                    torch.cuda._sleep(10_000)
            main.wait_stream(side)
            for i in range(2 * n, 3 * n):
                ops.stamp_globaltimer(slots[i:i + 1])
        last = 0
        for _ in range(3):
            g.replay()
            torch.cuda.synchronize(dev)
            v = slots.cpu().tolist()
            assert all(b >= a for a, b in zip(v, v[1:])), v
            assert v[0] > last and v[-1] > v[0], (last, v)
            last = v[-1]
        d = sorted({b - a for a, b in zip(v, v[1:]) if b > a})
        print(f"[stamps] smallest nonzero step between consecutive stamps: {d[0] if d else None} ns")


def test_timed_capture_on_one_rank_has_no_interval(built):
    """One rank exchanges nothing and all-reduces nothing: a timed capture opens no interval and reads 0.0, 0.0, as
    the eager timers give; ``timed=False`` captures no stamp buffer at all."""
    from bns_gcn_b200 import train
    from bns_gcn_b200.helper import context as ctx
    from bns_gcn_b200.helper.comm import SoloComm
    fg, parts = _graph()
    p = parts[0]
    dev = torch.device(DEV)
    ctx.set_comm(SoloComm())
    prev = torch.autograd.is_multithreading_enabled()
    torch.autograd.set_multithreading_enabled(False)
    try:
        with torch.cuda.stream(torch.cuda.Stream(dev)):
            for timed in (False, True):
                ctx.reset()
                ctx.set_comm(SoloComm())
                a = _args()
                a.n_feat, a.n_class, a.n_train = p.meta["n_feat"], p.meta["n_class"], p.meta["n_train"]
                st = train.setup(p.graph, p.node_dict, p.gpb, a, dev)
                ge = train.GraphedEpoch(st, warmup=1, timed=timed)
                ge()
                torch.cuda.synchronize(dev)
                if timed:
                    assert ge.stamps.names == {} and ge.interval_seconds() == (0.0, 0.0)
                else:
                    assert ge.stamps is None
                assert ctx.buffer.stamps is None and ctx.reducer.stamps is None
    finally:
        torch.autograd.set_multithreading_enabled(prev)
        ctx.reset()


# ---- the command line -----------------------------------------------------------------------------------------------

def _main(cwd, argv, world=1, port=29810, timeout=1500):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    env.pop("CUDA_VISIBLE_DEVICES", None)
    if world == 1:
        cmd = [sys.executable, "-m", "bns_gcn_b200.main"]
    else:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
               "--master-addr", "127.0.0.1", "--master-port", str(port), "-m", "bns_gcn_b200.main"]
    os.makedirs(cwd, exist_ok=True)
    p = subprocess.run(cmd + argv, cwd=str(cwd), env=env, capture_output=True, text=True, timeout=timeout)
    assert p.returncode == 0, (p.stdout[-4000:], p.stderr[-4000:])
    return p.stdout


def _timings(out):
    return {(int(m[0]), int(m[1])): (float(m[2]), float(m[3]), float(m[4])) for m in
            re.findall(r"Process (\d+) \| Epoch (\d+) \| Time\(s\) (\S+) \| Comm\(s\) (\S+) \| Reduce\(s\) (\S+)", out)}


@pytest.mark.timeout(1800)
def test_cli_reddit_inductive_parallel_eval(built, tmp_path):
    """The Reddit shape from the command line, one partition, inductive, partition-parallel evaluation, 12 epochs
    logged every 4: three ``Epoch`` lines, of which the ones after the 5 untimed epochs carry finite ``Comm(s)`` /
    ``Reduce(s)`` (epoch 3 prints nan, as an eager run does), their accuracy lines and ``Test Result``."""
    out = _main(tmp_path, ["--dataset", "reddit", "--n-partitions", "1", "--use-pp", "--n-layers", "4", "--n-hidden",
                           "256", "--inductive", "--eval", "--parallel-eval", "--cuda-graph", "--n-epochs", "12",
                           "--log-every", "4", "--fix-seed"])
    t = _timings(out)
    assert sorted(t) == [(0, 3), (0, 7), (0, 11)], out[-3000:]
    for e in (7, 11):
        assert all(math.isfinite(x) for x in t[(0, e)]) and t[(0, e)][0] > 0, t
    assert len(re.findall(r"Epoch 000(?:03|07|11) \| Accuracy \d+\.\d\d%", out)) == 3, out[-3000:]
    assert len(re.findall(r"Test Result \| Accuracy \d+\.\d\d%", out)) == 1, out[-3000:]


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("world,backend", [(2, "p2p"), (4, "p2p"), (2, "nccl")], ids=["w2-p2p", "w4-p2p", "w2-nccl"])
def test_torchrun_replays_equal_eager(built, tmp_path, world, backend):
    """One process per GPU: ``--cuda-graph`` against the eager run of the same command -- every rank's printed losses,
    and the saved final weights and Adam state, bit for bit; ``Comm(s)`` of the timed epochs finite and positive."""
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs, this box has {torch.cuda.device_count()}")
    argv = ["--dataset", "small", "--n-partitions", str(world), "--backend", backend, "--use-pp", "--n-layers", "3",
            "--n-hidden", "64", "--sampling-rate", "0.3", "--dropout", "0.5", "--fix-seed", "--seed", "7", "--no-eval",
            "--n-epochs", str(N_EPOCHS), "--log-every", "1", "--save-state-every", str(N_EPOCHS)]
    port = 29820 + 10 * world + (5 if backend == "nccl" else 0)
    eager = _main(tmp_path / "eager", argv, world, port)
    graphed = _main(tmp_path / "graph", argv + ["--cuda-graph"], world, port + 1)
    pat = r"Process (\d+) \| Epoch (\d+) \|.*\| Loss (\S+)"
    le, lg = sorted(re.findall(pat, eager)), sorted(re.findall(pat, graphed))
    assert len(le) == world * N_EPOCHS and lg == le
    from bns_gcn_b200 import state
    name = f"small-{world}-metis-vol-trans"
    a = argparse.Namespace(graph_name=name)
    for d in ("eager", "graph"):
        assert state._current(os.path.join(str(tmp_path / d), state.state_dir(a))) is not None
    se = torch.load(os.path.join(state._current(os.path.join(str(tmp_path / "eager"), state.state_dir(a))), "shared.pt"))
    sg = torch.load(os.path.join(state._current(os.path.join(str(tmp_path / "graph"), state.state_dir(a))), "shared.pt"))
    _equal(sg["model"], se["model"], "model")
    _equal(sg["optimizer"], se["optimizer"], "optimizer")
    t = _timings(graphed)
    for r in range(world):
        for e in range(5, N_EPOCHS):
            time_s, comm_s, reduce_s = t[(r, e)]
            assert math.isfinite(comm_s) and comm_s > 0 and math.isfinite(reduce_s), (r, e, t[(r, e)])
