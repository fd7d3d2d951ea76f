"""``--agg-dtype``: the flag parses, defaults to f32, and ``train.check_agg_dtype`` (what ``train.setup`` calls) refuses
bf16 with a message naming every reason whenever the fused training step would not run."""
import pytest
import torch

from tests.harness import make_args


def _check(monkeypatch, **kw):
    from bns_gcn_b200 import train
    from bns_gcn_b200.module import dense
    from bns_gcn_b200.train import get_layer_size
    monkeypatch.setattr(dense, "MODE", "tc")
    dev = kw.pop("_dev", torch.device("cuda", 0))
    kw = {"model": "graphsage", "n_hidden": 256, **kw}
    a = make_args(**kw)
    # GCN's fused layer 0 takes the precomputed features as they are: their width must be a multiple of 4
    a.n_feat, a.n_class = (604 if a.model == "gcn" else 602), 41
    return train.check_agg_dtype(a, get_layer_size(a.n_feat, a.n_hidden, a.n_class, a.n_layers), dev)


def test_parser_flag(built):
    from bns_gcn_b200.helper.parser import create_parser
    assert create_parser([]).agg_dtype == "f32"
    assert create_parser(["--agg-dtype", "bf16"]).agg_dtype == "bf16"
    assert create_parser(["--agg_dtype", "bf16"]).agg_dtype == "bf16"
    with pytest.raises(SystemExit):
        create_parser(["--agg-dtype", "fp16"])


def test_default_and_eligible(built, monkeypatch):
    monkeypatch.delenv("BNS_FUSED", raising=False)
    assert _check(monkeypatch) is False
    assert _check(monkeypatch, agg_dtype="f32", model="gat") is False        # f32 never refuses anything
    assert _check(monkeypatch, agg_dtype="bf16") is True
    assert _check(monkeypatch, agg_dtype="bf16", model="gcn") is True


@pytest.mark.parametrize("kw,reason", [
    (dict(model="gat"), "--model gat"),
    (dict(norm="batch"), "--norm batch"),
    (dict(n_linear=1), "--n-linear 1"),
    (dict(use_pp=False), "no --use-pp"),
    (dict(n_hidden=260), "not a multiple of 8"),
], ids=["gat", "batch-norm", "n-linear", "no-use-pp", "hidden-260"])
def test_refused_configurations(built, monkeypatch, kw, reason):
    monkeypatch.delenv("BNS_FUSED", raising=False)
    with pytest.raises(ValueError, match="--agg-dtype bf16 needs the fused training step") as e:
        _check(monkeypatch, agg_dtype="bf16", **kw)
    assert reason in str(e.value)


def test_refused_without_fused_step(built, monkeypatch):
    monkeypatch.setenv("BNS_FUSED", "0")
    with pytest.raises(ValueError, match="BNS_FUSED=0"):
        _check(monkeypatch, agg_dtype="bf16")


def test_refused_on_cpu(built, monkeypatch):
    monkeypatch.delenv("BNS_FUSED", raising=False)
    with pytest.raises(ValueError, match="no CUDA device"):
        _check(monkeypatch, agg_dtype="bf16", _dev=torch.device("cpu"))
