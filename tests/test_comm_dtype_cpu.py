"""``--comm-dtype``: the flag parses, defaults to f32, ``train.check_comm_dtype`` (what ``train.setup`` calls) refuses bf16
with a message naming every reason whenever the fused training step would not run, and the byte counts of the exchange
(``feature_buffer.slab_layout`` / ``wire_bytes``) match hand-computed values."""
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
    kw = {"model": "graphsage", "n_hidden": 256, **kw}
    a = make_args(**kw)
    if drop:
        assert not hasattr(a, "comm_dtype")
    a.n_feat, a.n_class = (604 if a.model == "gcn" else 602), 41
    return train.check_comm_dtype(a, get_layer_size(a.n_feat, a.n_hidden, a.n_class, a.n_layers), dev)


def test_parser_flag(built):
    from bns_gcn_b200.helper.parser import create_parser
    assert create_parser([]).comm_dtype == "f32"
    assert create_parser(["--comm-dtype", "bf16"]).comm_dtype == "bf16"
    assert create_parser(["--comm_dtype", "bf16"]).comm_dtype == "bf16"
    assert create_parser(["--comm-dtype", "f32"]).comm_dtype == "f32"
    with pytest.raises(SystemExit):
        create_parser(["--comm-dtype", "fp16"])


def test_default_and_eligible(built, monkeypatch):
    monkeypatch.delenv("BNS_FUSED", raising=False)
    assert _check(monkeypatch, _drop_attr=True) == "f32"                    # args without the attribute: f32
    assert _check(monkeypatch, comm_dtype="f32", model="gat", norm="batch") == "f32"     # f32 never refuses anything
    assert _check(monkeypatch, comm_dtype="bf16") == "bf16"
    assert _check(monkeypatch, comm_dtype="bf16", model="gcn") == "bf16"
    assert _check(monkeypatch, comm_dtype="bf16", agg_dtype="bf16") == "bf16"


@pytest.mark.parametrize("kw,reason", [
    (dict(model="gat"), "--model gat"),
    (dict(norm="batch"), "--norm batch"),
    (dict(n_linear=1), "--n-linear 1"),
    (dict(use_pp=False), "no --use-pp"),
    (dict(n_hidden=260), "exchanged width 260 is not a multiple of 8"),
], ids=["gat", "batch-norm", "n-linear", "no-use-pp", "hidden-260"])
def test_refused_configurations(built, monkeypatch, kw, reason):
    monkeypatch.delenv("BNS_FUSED", raising=False)
    with pytest.raises(ValueError, match="--comm-dtype bf16 needs the fused training step") as e:
        _check(monkeypatch, comm_dtype="bf16", **kw)
    assert reason in str(e.value)


def test_refusal_names_every_reason(built, monkeypatch):
    monkeypatch.setenv("BNS_FUSED", "0")
    with pytest.raises(ValueError) as e:
        _check(monkeypatch, comm_dtype="bf16", model="gat", norm="batch", n_linear=1, use_pp=False, n_hidden=20,
               _dev=torch.device("cpu"))
    for reason in ("BNS_FUSED=0", "--model gat", "--norm batch", "--n-linear 1", "no --use-pp", "no CUDA device",
                   "exchanged width 20"):
        assert reason in str(e.value), reason


def test_refused_without_fused_step(built, monkeypatch):
    monkeypatch.setenv("BNS_FUSED", "0")
    with pytest.raises(ValueError, match="BNS_FUSED=0"):
        _check(monkeypatch, comm_dtype="bf16")


def test_refused_on_cpu(built, monkeypatch):
    monkeypatch.delenv("BNS_FUSED", raising=False)
    with pytest.raises(ValueError, match="no CUDA device"):
        _check(monkeypatch, comm_dtype="bf16", _dev=torch.device("cpu"))


def test_slab_and_wire_bytes(built):
    """n_in = 100 inner rows, 37 halo rows received, 29 rows sent, width 64, two communicating layers."""
    from bns_gcn_b200.helper.feature_buffer import slab_layout, wire_bytes
    f = slab_layout(100, 37, 29, 64, 2, "f32")
    row = 64 * 4
    assert (f["inner_bytes"], f["halo_bytes"], f["bwd_bytes"]) == (100 * row, 37 * row, 29 * row)
    layer = (100 + 37 + 29) * row                                   # 42,496 bytes, no padding between regions
    assert f["fwd_off"] == [0, layer] and f["halo_off"] == [100 * row, layer + 100 * row]
    assert f["bwd_off"] == [137 * row, layer + 137 * row]
    assert f["ids_off"] == 84992 and f["slab_bytes"] == 84992 + 37 * 8        # 2 * 42,496 is already 256-aligned
    b = slab_layout(100, 37, 29, 64, 2, "bf16")
    # inner 25,600 (f32, aligned); halo 37 * 128 = 4,736 -> 4,864; backward 29 * 128 = 3,712 -> 3,840
    assert (b["inner_bytes"], b["halo_bytes"], b["bwd_bytes"]) == (25600, 4864, 3840)
    assert b["fwd_off"] == [0, 34304] and b["halo_off"] == [25600, 59904] and b["bwd_off"] == [30464, 64768]
    assert b["ids_off"] == 68608 and b["slab_bytes"] == 68608 + 296
    assert all(o % 256 == 0 for k in ("fwd_off", "halo_off", "bwd_off") for o in b[k])
    # empty segments still get one row, as the f32 layout does
    e = slab_layout(8, 0, 0, 8, 1, "bf16")
    assert (e["inner_bytes"], e["halo_bytes"], e["bwd_bytes"], e["slab_bytes"]) == (256, 256, 256, 776)
    assert wire_bytes(29, 37, 64, "f32") == {"fwd_send": 29 * 256, "fwd_recv": 37 * 256, "bwd_send": 37 * 256,
                                             "bwd_recv": 29 * 256}
    assert wire_bytes(29, 37, 64, "bf16") == {"fwd_send": 29 * 128, "fwd_recv": 37 * 128, "bwd_send": 37 * 128,
                                              "bwd_recv": 29 * 128}
