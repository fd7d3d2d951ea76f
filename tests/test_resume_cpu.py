"""``--save-state-every`` / ``--resume`` on the host: the flags, the fingerprint check, the refusals, and the save
protocol (a save that fails part way never replaces the complete state before it)."""
import os
import types

import pytest
import torch

from tests.harness import make_args


def _args(**kw):
    kw = {"dataset": "small", "graph_name": "small-2-random-vol-trans", "n_partitions": 2, "n_hidden": 64,
          "dropout": 0.5, **kw}
    a = make_args(**kw)
    a.n_feat, a.n_class, a.n_train = 32, 7, 3600
    return a


def test_parser_flags(built):
    from bns_gcn_b200.helper.parser import create_parser
    a = create_parser([])
    assert a.save_state_every == 0 and a.resume is False
    for spelling in ("--save-state-every", "--save_state_every"):
        assert create_parser([spelling, "5"]).save_state_every == 5
    assert create_parser(["--resume"]).resume is True
    with pytest.raises(SystemExit):
        create_parser(["--save-state-every", "x"])


def test_fingerprint_names_every_difference(built):
    from bns_gcn_b200.state import FINGERPRINT, fingerprint, fingerprint_mismatches
    saved = vars(_args())
    old = fingerprint(saved)
    assert fingerprint_mismatches(saved, dict(saved)) == []
    changed = dict(model="gcn", n_layers=4, n_hidden=128, n_feat=16, n_class=9, heads=2, norm="batch", n_linear=1,
                   use_pp=False, dropout=0.1, lr=0.5, weight_decay=1e-4, sampling_rate=0.3, sampler_seed=7,
                   n_partitions=4, graph_name="other", backend="p2p", agg_dtype="bf16", comm_dtype="bf16",
                   dense_dtype="bf16")
    assert set(changed) == {k for k, _ in FINGERPRINT}
    why = fingerprint_mismatches(saved, dict(saved, **changed))
    assert len(why) == len(changed), why
    for k, v in changed.items():
        assert f"{k} is {v!r}, the state's {old[k]!r}" in why, (k, why)
    for k, v in changed.items():                          # one at a time: exactly that field
        assert fingerprint_mismatches(saved, dict(saved, **{k: v})) == [f"{k} is {v!r}, the state's {old[k]!r}"]


def test_fingerprint_accepts_run_length_logging_eval_and_seed(built):
    from bns_gcn_b200.state import fingerprint_mismatches
    saved = vars(_args())
    other = dict(saved, n_epochs=3000, log_every=1, eval=True, parallel_eval=True, inductive=False, seed=12345,
                 save_state_every=7, resume=True)
    assert fingerprint_mismatches(saved, other) == []
    # a dict without the newer flags stands for their defaults
    old = {k: v for k, v in saved.items() if k not in ("agg_dtype", "comm_dtype", "dense_dtype", "sampler_seed")}
    assert fingerprint_mismatches(old, saved) == []


def test_resume_without_state_names_the_path(built, tmp_path, monkeypatch):
    from bns_gcn_b200 import state
    monkeypatch.chdir(tmp_path)
    a = _args(resume=True)
    with pytest.raises(ValueError, match="no complete training state") as e:
        state.load(a, 0)
    assert os.path.join("checkpoint", "small-2-random-vol-trans_state") in str(e.value)
    # a save that never finished: its directory is not a state
    tmp = os.path.join("checkpoint", "small-2-random-vol-trans_state", "incomplete")
    os.makedirs(tmp)
    torch.save({"epochs": 4}, os.path.join(tmp, "shared.pt"))
    with pytest.raises(ValueError, match="no complete training state") as e:
        state.load(a, 0)
    assert tmp in str(e.value) and "incomplete" in str(e.value)


def test_resume_without_state_refuses_in_run(built, tmp_path, monkeypatch):
    """``train.run`` refuses before any setup work (the graph argument is never touched)."""
    from bns_gcn_b200 import train
    from bns_gcn_b200.helper import context as ctx
    monkeypatch.chdir(tmp_path)
    try:
        with pytest.raises(ValueError, match="no complete training state"):
            train.run(None, None, None, _args(resume=True, n_partitions=1))
    finally:
        ctx.reset()


def _fake_state(args, w):
    """What ``state.save`` reads of a ``TrainState``, on the host: the op-by-op path with a plain Adam."""
    model = torch.nn.Linear(4, 3)
    with torch.no_grad():
        model.weight.fill_(w)
    opt = torch.optim.Adam(model.parameters(), lr=args.lr)
    model(torch.ones(2, 4)).sum().backward()
    opt.step()
    return types.SimpleNamespace(args=args, feat=torch.zeros(1), arena=None, model=model, optimizer=opt)


def test_save_protocol_keeps_the_complete_state(built, tmp_path, monkeypatch):
    from bns_gcn_b200 import state
    from bns_gcn_b200.helper import context as ctx
    from bns_gcn_b200.helper.comm import SoloComm
    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(torch.cuda, "get_rng_state", lambda device=None: torch.get_rng_state())
    ctx.set_comm(SoloComm())
    try:
        a = _args(seed=99)
        st1 = _fake_state(a, 1.0)
        d1 = state.save(st1, 4)
        s = state.load(a, 0)
        assert s["dir"] == d1 and s["epochs"] == 4 and s["seed"] == 99 and s["path"] == "op-by-op"
        assert torch.equal(s["model"]["weight"], st1.model.weight.detach())
        assert torch.equal(s["optimizer"]["state"][0]["exp_avg"], st1.optimizer.state[st1.model.weight]["exp_avg"])
        # a second save that fails before CURRENT moves: the first state is still the current one, complete
        real = os.replace

        def crash(src, dst):
            raise OSError("simulated crash")
        monkeypatch.setattr(os, "replace", crash)
        with pytest.raises(OSError, match="simulated crash"):
            state.save(_fake_state(a, 2.0), 8)
        monkeypatch.setattr(os, "replace", real)
        s = state.load(a, 0)
        assert s["dir"] == d1 and s["epochs"] == 4 and torch.equal(s["model"]["weight"], st1.model.weight.detach())
        # the next save completes, supersedes and removes the old one (and the leftover of the failed one)
        st3 = _fake_state(a, 3.0)
        d3 = state.save(st3, 12)
        s = state.load(a, 0)
        assert s["dir"] == d3 and s["epochs"] == 12 and torch.equal(s["model"]["weight"], st3.model.weight.detach())
        root = state.state_dir(a)
        assert sorted(os.listdir(root)) == sorted(["CURRENT", os.path.basename(d3)])
        # another run's settings are refused, naming the state's directory and every difference
        with pytest.raises(ValueError, match="saved by a different run") as e:
            state.load(_args(seed=99, lr=0.5, n_hidden=32), 0)
        assert d3 in str(e.value) and "lr is 0.5" in str(e.value) and "n_hidden is 32" in str(e.value)
    finally:
        ctx.reset()
