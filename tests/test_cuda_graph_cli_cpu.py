"""``--cuda-graph`` without a GPU: the flag, the refusals ``train.run`` raises before any setup work, the resume
fingerprint, and the log line's ``Comm(s)`` / ``Reduce(s)`` computed from a stamp buffer (a host-side fake of the
device buffer a timed replay writes)."""
import argparse
import re

import pytest

from tests.harness import make_args


def test_flag_parses_in_both_spellings_and_defaults_off(built):
    from bns_gcn_b200.helper.parser import create_parser
    assert create_parser([]).cuda_graph is False
    assert create_parser(["--cuda-graph"]).cuda_graph is True
    assert create_parser(["--cuda_graph"]).cuda_graph is True


def _refusal(n_ranks, **kw):
    """What ``train.run`` raises on every in-process rank; ``None`` arguments: setup would fail on them at once."""
    from bns_gcn_b200 import train
    from bns_gcn_b200.helper.comm import run_threads
    args = make_args(cuda_graph=True, n_partitions=n_ranks, **kw)

    def fn(comm, r):
        with pytest.raises(ValueError) as e:
            train.run(None, None, None, argparse.Namespace(**vars(args)), "cuda:0")
        return str(e.value)
    return run_threads(n_ranks, fn)


def test_in_process_ranks_and_staged_nccl_are_refused_together(built, tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)                  # --resume finds no state here: the refusal must come first
    for msg in _refusal(4, backend="nccl", resume=True):
        assert msg.startswith("--cuda-graph: "), msg
        assert "threads of one process" in msg and "staged --backend nccl at 4 partitions" in msg, msg


def test_in_process_ranks_are_refused_on_p2p(built):
    for msg in _refusal(2, backend="p2p"):
        assert "threads of one process" in msg and "staged" not in msg, msg


class _Comm:
    def __init__(self, kind, size):
        self.kind, self.size, self.rank = kind, size, 0


@pytest.mark.parametrize("kind,size,backend,want", [
    ("solo", 1, "nccl", []),
    ("dist", 2, "nccl", []),
    ("dist", 2, "p2p", []),
    ("dist", 8, "p2p", []),
    ("dist", 3, "nccl", ["staged"]),
    ("dist", 4, "staged", ["staged"]),
    ("thread", 2, "p2p", ["threads"]),
    ("thread", 4, "nccl", ["threads", "staged"]),
])
def test_refusal_rules(built, kind, size, backend, want):
    from bns_gcn_b200 import train
    why = train.cuda_graph_refusals(make_args(backend=backend, n_partitions=size), _Comm(kind, size))
    assert len(why) == len(want), why
    for w, text in zip(want, why):
        assert w in text, (w, text)


def test_resume_fingerprint_ignores_the_flag(built):
    from bns_gcn_b200 import state
    eager, graphed = vars(make_args()), vars(make_args(cuda_graph=True))
    assert "cuda_graph" not in dict(state.FINGERPRINT)
    assert state.fingerprint(eager) == state.fingerprint(graphed)
    assert state.fingerprint_mismatches(eager, graphed) == [] and state.fingerprint_mismatches(graphed, eager) == []


def _fake_stamps(names, values):
    import torch
    from bns_gcn_b200.helper.timer.replay_stamps import ReplayStamps
    s = ReplayStamps(len(values) // 2, "cpu")
    s.names = dict(names)
    s.slots.copy_(torch.tensor(values, dtype=torch.int64))
    return s


def test_log_line_from_a_stamp_buffer(built):
    from bns_gcn_b200 import train
    t0 = 1_760_000_000_000_000_000                   # nanoseconds of a %globaltimer reading
    names = {"forward_1": ("comm", 0), "forward_2": ("comm", 1), "backward_2": ("comm", 2), "backward_1": ("comm", 3),
             "reduce": ("reduce", 4)}
    values = [t0, t0 + 1_250_000,                   # forward_1: 1.25 ms
              t0 + 3_000_000, t0 + 3_500_000,       # forward_2: 0.5 ms
              t0 + 6_000_000, t0 + 8_000_000,       # backward_2: 2 ms
              t0 + 9_000_000, t0 + 9_250_000,       # backward_1: 0.25 ms
              t0 + 10_000_000, t0 + 10_700_000]     # reduce: 0.7 ms
    s = _fake_stamps(names, values)
    sec = s.seconds(s.read())
    assert sec["comm"] == pytest.approx(4.0e-3, abs=1e-12) and sec["reduce"] == pytest.approx(0.7e-3, abs=1e-12)
    line = train.log_line(3, 11, [0.05, 0.07], [sec["comm"], 0.006], [sec["reduce"], 0.0013], 1.234567)
    assert line == "Process 003 | Epoch 00011 | Time(s) 0.0600 | Comm(s) 0.0050 | Reduce(s) 0.0010 | Loss 1.2346"


def test_one_rank_has_no_intervals(built):
    """One rank exchanges and all-reduces nothing: zero, as the eager epoch's timers give."""
    from bns_gcn_b200 import train
    s = _fake_stamps({}, [0] * 6)
    sec = s.seconds(s.read())
    assert sec == {"comm": 0.0, "reduce": 0.0}
    line = train.log_line(0, 9, [0.02], [sec["comm"]], [sec["reduce"]], 0.5)
    assert re.search(r"Comm\(s\) 0\.0000 \| Reduce\(s\) 0\.0000", line), line
    assert "nan" in train.log_line(0, 4, [], [], [], 0.5)          # no timed epoch yet, as before


def test_stamp_slots_are_bounded(built):
    from bns_gcn_b200.helper.timer.replay_stamps import ReplayStamps
    s = ReplayStamps(1, "cpu")
    s.names["reduce"] = ("reduce", 0)
    with pytest.raises(RuntimeError, match="holds 1"):
        with s.interval("forward_1", None):
            pass
    with pytest.raises(Exception, match="already exists"):
        with s.interval("reduce", None):
            pass
