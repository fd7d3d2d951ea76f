"""``--dense-dtype fp8``: the flag parses under both spellings, ``train.check_dense_dtype`` returns ``'fp8'`` where the
fused training step runs (composing with the other two fp8 flags) and refuses it, naming every reason, where it does
not; and the host restatement of the fp8 GEMM (``tests/dense_fp8_reference.py``: codes times scales in float64) agrees
with ``tests/fp8_reference.py``'s dequantized rows."""
import pytest
import torch

from tests import dense_fp8_reference as D
from tests import fp8_reference as Q
from tests.test_dense_dtype_cpu import _check


def test_parser_flag(built):
    from bns_gcn_b200.helper.parser import create_parser
    assert create_parser(["--dense-dtype", "fp8"]).dense_dtype == "fp8"
    assert create_parser(["--dense_dtype", "fp8"]).dense_dtype == "fp8"
    for bad in ("e4m3", "fp8e5m2", "int8"):
        with pytest.raises(SystemExit):
            create_parser(["--dense-dtype", bad])


def test_returns_fp8_where_eligible(built, monkeypatch):
    monkeypatch.delenv("BNS_FUSED", raising=False)
    assert _check(monkeypatch, dense_dtype="fp8") == "fp8"
    assert _check(monkeypatch, dense_dtype="fp8", model="gcn") == "fp8"
    assert _check(monkeypatch, dense_dtype="fp8", agg_dtype="fp8", comm_dtype="fp8") == "fp8"
    assert _check(monkeypatch, dense_dtype="bf16") is True                  # bf16 unchanged
    assert _check(monkeypatch, dense_dtype="f32") is False


@pytest.mark.parametrize("kw,reason", [
    (dict(model="gat"), "--model gat"),
    (dict(norm="batch"), "--norm batch"),
    (dict(n_linear=1), "--n-linear 1"),
    (dict(use_pp=False), "no --use-pp"),
    (dict(n_hidden=258), "layer widths 258 do not fit the fused step"),
    (dict(_n_feat=601), "layer widths 1202 do not fit the fused step"),
], ids=["gat", "batch-norm", "n-linear", "no-use-pp", "hidden-258", "input-width"])
def test_refused_configurations(built, monkeypatch, kw, reason):
    monkeypatch.delenv("BNS_FUSED", raising=False)
    with pytest.raises(ValueError) as e:
        _check(monkeypatch, dense_dtype="fp8", **kw)
    assert str(e.value).startswith("--dense-dtype fp8 needs the fused training step")
    assert reason in str(e.value)


def test_refusal_names_every_reason(built, monkeypatch):
    monkeypatch.setenv("BNS_FUSED", "0")
    with pytest.raises(ValueError) as e:
        _check(monkeypatch, dense_dtype="fp8", model="gat", norm="batch", n_linear=1, use_pp=False, n_hidden=18,
               _dev=torch.device("cpu"))
    msg = str(e.value)
    assert msg.startswith("--dense-dtype fp8 needs the fused training step")
    for reason in ("BNS_FUSED=0", "--model gat", "--norm batch", "--n-linear 1", "no --use-pp", "no CUDA device",
                   "layer widths 18"):
        assert reason in msg, reason


def test_no_width_rule_of_its_own(built, monkeypatch):
    """Hidden 40 is not a multiple of 16 (``--agg-dtype fp8`` refuses it) but the dense operands are padded."""
    monkeypatch.delenv("BNS_FUSED", raising=False)
    assert _check(monkeypatch, dense_dtype="fp8", n_hidden=40) == "fp8"


def _rows(n, k, g):
    x = torch.randn(n, k, generator=g, dtype=torch.float64).float()
    x *= torch.exp2(torch.randint(-30, 30, (n, 1), generator=g).float())
    return x


def test_host_restatement_matches_dequantized_rows():
    """``(sum qa qb) sa sb`` equals ``deq(A) deq(B)^T`` (every code times a power of two is exact in float64), and the
    bound is the magnitude sum of the dequantized rows; the epilogue terms in order."""
    g = torch.Generator().manual_seed(5)
    for M, N, K in ((7, 5, 4), (33, 44, 1204), (3, 256, 44)):
        a, b = _rows(M, K, g), _rows(N, K, g)
        (qa, sa), (qb, sb) = Q.quantize_rows(a), Q.quantize_rows(b)
        da, db = Q.dequantize(qa, sa), Q.dequantize(qb, sb)
        bias, add, rs = torch.randn(N, generator=g), torch.randn(M, N, generator=g), torch.randn(M, generator=g)
        ref, bnd = D.tn(qa, sa, qb, sb, bias, add, rs)
        want = (da @ db.t() + bias.double() + add.double()) * rs.double()[:, None]
        wbnd = (da.abs() @ db.abs().t() + bias.double().abs() + add.double().abs()) * rs.double().abs()[:, None]
        assert torch.allclose(ref, want, rtol=1e-12, atol=0) and torch.allclose(bnd, wbnd, rtol=1e-12, atol=0)
        assert (bnd >= ref.abs() * (1 - 1e-12)).all()


def test_host_restatement_nan_rows_and_columns():
    """A row that held NaN or +-Inf has scale NaN and zero codes: only its own output row (A) or column (B) is NaN."""
    a = torch.randn(4, 8)
    b = torch.randn(3, 8)
    a[1, 2] = float("inf")
    b[2, 5] = float("nan")
    (qa, sa), (qb, sb) = Q.quantize_rows(a), Q.quantize_rows(b)
    ref, _ = D.tn(qa, sa, qb, sb)
    nan = torch.isnan(ref)
    assert nan[1].all() and nan[:, 2].all()
    assert nan.sum() == 3 + 4 - 1
