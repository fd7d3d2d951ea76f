"""``--comm-dtype fp8``: the flag parses, ``train.check_comm_dtype`` returns ``'fp8'`` alone and beside the other
narrow modes, refuses it with every reason where the fused training step would not run (an exchanged width that is not
a multiple of 16 among them), the byte counts of the exchange (``feature_buffer.slab_layout`` / ``wire_bytes``) match
hand-computed values, and a state saved under bf16 does not resume under fp8."""
import pytest
import torch

from tests.harness import make_args
from tests.test_comm_dtype_cpu import _check


def test_parser_accepts_fp8(built):
    from bns_gcn_b200.helper.parser import create_parser
    assert create_parser(["--comm-dtype", "fp8"]).comm_dtype == "fp8"
    assert create_parser(["--comm_dtype", "fp8"]).comm_dtype == "fp8"
    with pytest.raises(SystemExit):
        create_parser(["--comm-dtype", "e4m3"])


def test_check_returns_fp8(built, monkeypatch):
    monkeypatch.delenv("BNS_FUSED", raising=False)
    assert _check(monkeypatch, comm_dtype="fp8") == "fp8"
    assert _check(monkeypatch, comm_dtype="fp8", model="gcn") == "fp8"
    assert _check(monkeypatch, comm_dtype="fp8", agg_dtype="fp8") == "fp8"
    assert _check(monkeypatch, comm_dtype="fp8", dense_dtype="bf16") == "fp8"
    assert _check(monkeypatch, comm_dtype="fp8", agg_dtype="fp8", dense_dtype="bf16") == "fp8"


def test_hidden_264_bf16_yes_fp8_no(built, monkeypatch):
    monkeypatch.delenv("BNS_FUSED", raising=False)
    assert _check(monkeypatch, comm_dtype="bf16", n_hidden=264) == "bf16"
    with pytest.raises(ValueError, match="--comm-dtype fp8 needs the fused training step") as e:
        _check(monkeypatch, comm_dtype="fp8", n_hidden=264)
    assert "exchanged width 264 is not a multiple of 16" in str(e.value)


@pytest.mark.parametrize("kw,reason", [
    (dict(model="gat"), "--model gat"),
    (dict(norm="batch"), "--norm batch"),
    (dict(n_linear=1), "--n-linear 1"),
    (dict(use_pp=False), "no --use-pp"),
], ids=["gat", "batch-norm", "n-linear", "no-use-pp"])
def test_refused_configurations(built, monkeypatch, kw, reason):
    monkeypatch.delenv("BNS_FUSED", raising=False)
    with pytest.raises(ValueError, match="--comm-dtype fp8 needs the fused training step") as e:
        _check(monkeypatch, comm_dtype="fp8", **kw)
    assert reason in str(e.value)


def test_refusal_names_every_reason(built, monkeypatch):
    monkeypatch.setenv("BNS_FUSED", "0")
    with pytest.raises(ValueError) as e:
        _check(monkeypatch, comm_dtype="fp8", model="gat", norm="batch", n_linear=1, use_pp=False, n_hidden=264,
               _dev=torch.device("cpu"))
    for reason in ("BNS_FUSED=0", "--model gat", "--norm batch", "--n-linear 1", "no --use-pp", "no CUDA device",
                   "exchanged width 264 is not a multiple of 16"):
        assert reason in str(e.value), reason


def test_slab_and_wire_bytes(built):
    """n_in = 100 inner rows, 37 halo rows received, 29 rows sent, width 64, two communicating layers: inner f32 rows |
    halo codes | halo scales | backward codes | backward scales, each on 256 bytes."""
    from bns_gcn_b200.helper.feature_buffer import slab_layout, wire_bytes
    f = slab_layout(100, 37, 29, 64, 2, "fp8")
    # inner 25,600; halo codes 37 * 64 = 2,368 -> 2,560; scales 148 -> 256; backward 29 * 64 = 1,856 -> 2,048; 116 -> 256
    assert (f["inner_bytes"], f["halo_bytes"], f["halo_scale_bytes"], f["bwd_bytes"], f["bwd_scale_bytes"]) == \
        (25600, 2560, 256, 2048, 256)
    layer = 25600 + 2560 + 256 + 2048 + 256                            # 30,720
    assert f["fwd_off"] == [0, layer]
    assert f["halo_off"] == [25600, layer + 25600]
    assert f["halo_scale_off"] == [28160, layer + 28160]
    assert f["bwd_off"] == [28416, layer + 28416]
    assert f["bwd_scale_off"] == [30464, layer + 30464]
    assert f["ids_off"] == 2 * layer and f["slab_bytes"] == 2 * layer + 37 * 8
    assert all(o % 256 == 0 for k in ("fwd_off", "halo_off", "halo_scale_off", "bwd_off", "bwd_scale_off") for o in f[k])
    # empty segments still get one row, as the other layouts do; a 1-row scale region is one 256-byte block
    e = slab_layout(8, 0, 0, 16, 1, "fp8")
    assert (e["inner_bytes"], e["halo_bytes"], e["halo_scale_bytes"], e["bwd_bytes"], e["bwd_scale_bytes"]) == \
        (512, 256, 256, 256, 256)
    assert e["slab_bytes"] == 1536 + 8
    # a scale region that ends exactly on 256 bytes gets no padding
    assert slab_layout(8, 64, 64, 16, 1, "fp8")["halo_scale_bytes"] == 256
    assert slab_layout(8, 65, 64, 16, 1, "fp8")["halo_scale_bytes"] == 512
    assert wire_bytes(29, 37, 64, "fp8") == {"fwd_send": 29 * 68, "fwd_recv": 37 * 68, "bwd_send": 37 * 68,
                                             "bwd_recv": 29 * 68}
    assert wire_bytes(0, 0, 64, "fp8") == {"fwd_send": 0, "fwd_recv": 0, "bwd_send": 0, "bwd_recv": 0}


def test_benchmark_shape_byte_counts(built):
    """The per-rank feature bytes of one epoch (two communicating layers, forward and backward) at the benchmark's
    hidden 256 and sampling rate 0.1, as ``tools/bench_comm_dtype.py`` counts them: bf16 -> fp8 roughly halves."""
    from tools.bench_comm_dtype import byte_counts
    b = byte_counts()
    mb = {k: (round(r["bf16"]["per_epoch_sent"] / 1e6, 1), round(r["fp8"]["per_epoch_sent"] / 1e6, 1))
          for k, r in b.items() if k.startswith("reddit")}
    assert mb == {"reddit_P2": (23.9, 12.1), "reddit_P4": (35.8, 18.2), "reddit_P8": (41.7, 21.2)}
    p = b["papers100m_per_rank_P8"]
    assert (round(p["bf16"]["per_epoch_sent"] / 1e9, 1), round(p["fp8"]["per_epoch_sent"] / 1e9, 1)) == (19.9, 10.1)
    assert round(b["reddit_P4"]["fp8"]["slab_bytes"] / 1e6, 1) == 137.6
    assert round(b["reddit_P8"]["fp8"]["slab_bytes"] / 1e6, 1) == 81.0
    for r in b.values():                        # F + 4 bytes against 2F: (256 + 4) / 512
        assert r["fp8"]["per_epoch_sent"] * 512 == r["bf16"]["per_epoch_sent"] * 260


def test_resume_across_comm_dtype_refused(built):
    from bns_gcn_b200.state import fingerprint_mismatches
    saved = vars(make_args(comm_dtype="bf16"))
    why = fingerprint_mismatches(saved, dict(saved, comm_dtype="fp8"))
    assert why == ["comm_dtype is 'fp8', the state's 'bf16'"]
    assert fingerprint_mismatches(dict(saved, comm_dtype="fp8"), dict(saved, comm_dtype="fp8")) == []
