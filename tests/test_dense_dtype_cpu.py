"""``--dense-dtype``: the flag parses, defaults to f32, and ``train.check_dense_dtype`` (what ``train.setup`` calls) refuses
bf16 with a message naming every reason whenever the fused training step would not run; f32 never refuses anything."""
import pytest
import torch

from tests.harness import make_args


def _check(monkeypatch, **kw):
    from bns_gcn_b200 import train
    from bns_gcn_b200.module import dense
    from bns_gcn_b200.train import get_layer_size
    monkeypatch.setattr(dense, "MODE", "tc")
    dev = kw.pop("_dev", torch.device("cuda", 0))
    drop = kw.pop("_drop_attr", False)
    n_feat = kw.pop("_n_feat", None)
    kw = {"model": "graphsage", "n_hidden": 256, **kw}
    a = make_args(**kw)
    if drop:
        assert not hasattr(a, "dense_dtype")
    a.n_feat, a.n_class = n_feat or (604 if a.model == "gcn" else 602), 41
    return train.check_dense_dtype(a, get_layer_size(a.n_feat, a.n_hidden, a.n_class, a.n_layers), dev)


def test_parser_flag(built):
    from bns_gcn_b200.helper.parser import create_parser
    assert create_parser([]).dense_dtype == "f32"
    assert create_parser(["--dense-dtype", "bf16"]).dense_dtype == "bf16"
    assert create_parser(["--dense_dtype", "bf16"]).dense_dtype == "bf16"
    assert create_parser(["--dense-dtype", "f32"]).dense_dtype == "f32"
    for bad in ("fp16", "tf32", "bf16x3"):
        with pytest.raises(SystemExit):
            create_parser(["--dense-dtype", bad])


def test_default_and_eligible(built, monkeypatch):
    monkeypatch.delenv("BNS_FUSED", raising=False)
    assert _check(monkeypatch, _drop_attr=True) is False                    # args without the attribute: f32
    assert _check(monkeypatch, dense_dtype="bf16") is True
    assert _check(monkeypatch, dense_dtype="bf16", model="gcn") is True
    # the three flags compose
    assert _check(monkeypatch, dense_dtype="bf16", agg_dtype="bf16", comm_dtype="bf16") is True


def test_f32_never_refuses(built, monkeypatch):
    monkeypatch.setenv("BNS_FUSED", "0")
    assert _check(monkeypatch, dense_dtype="f32", model="gat", norm="batch", n_linear=1, use_pp=False, n_hidden=6,
                  _dev=torch.device("cpu")) is False


@pytest.mark.parametrize("kw,reason", [
    (dict(model="gat"), "--model gat"),
    (dict(norm="batch"), "--norm batch"),
    (dict(n_linear=1), "--n-linear 1"),
    (dict(use_pp=False), "no --use-pp"),
    (dict(n_hidden=258), "layer widths 258 do not fit the fused step"),
    (dict(n_hidden=2048), "layer widths 2048 do not fit the fused step"),
    (dict(_n_feat=601), "layer widths 1202 do not fit the fused step"),
], ids=["gat", "batch-norm", "n-linear", "no-use-pp", "hidden-258", "hidden-2048", "input-width"])
def test_refused_configurations(built, monkeypatch, kw, reason):
    monkeypatch.delenv("BNS_FUSED", raising=False)
    with pytest.raises(ValueError, match="--dense-dtype bf16 needs the fused training step") as e:
        _check(monkeypatch, dense_dtype="bf16", **kw)
    assert reason in str(e.value)


def test_refused_without_fused_step(built, monkeypatch):
    monkeypatch.setenv("BNS_FUSED", "0")
    with pytest.raises(ValueError, match="BNS_FUSED=0"):
        _check(monkeypatch, dense_dtype="bf16")


def test_refused_on_cpu(built, monkeypatch):
    monkeypatch.delenv("BNS_FUSED", raising=False)
    with pytest.raises(ValueError, match="no CUDA device"):
        _check(monkeypatch, dense_dtype="bf16", _dev=torch.device("cpu"))


def test_refusal_names_every_reason(built, monkeypatch):
    monkeypatch.setenv("BNS_FUSED", "0")
    with pytest.raises(ValueError) as e:
        _check(monkeypatch, dense_dtype="bf16", model="gat", norm="batch", n_linear=1, use_pp=False, n_hidden=18,
               _dev=torch.device("cpu"))
    for reason in ("BNS_FUSED=0", "--model gat", "--norm batch", "--n-linear 1", "no --use-pp", "no CUDA device",
                   "layer widths 18"):
        assert reason in str(e.value), reason
