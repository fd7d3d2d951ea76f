"""``--agg-dtype fp8`` on the host: the flag, its refusals, the quantization rule of tests/fp8_reference.py stated on
crafted rows, and the resume fingerprint."""
import pytest
import torch

from tests import fp8_reference as Q
from tests.harness import make_args
from tests.test_agg_dtype_cpu import _check


def _u8(codes):
    return codes.view(torch.uint8).tolist()


def test_parser_accepts_fp8(built):
    from bns_gcn_b200.helper.parser import create_parser
    assert create_parser(["--agg-dtype", "fp8"]).agg_dtype == "fp8"
    assert create_parser(["--agg_dtype", "fp8"]).agg_dtype == "fp8"
    with pytest.raises(SystemExit):
        create_parser(["--agg-dtype", "e4m3"])


def test_check_returns(built, monkeypatch):
    monkeypatch.delenv("BNS_FUSED", raising=False)
    assert _check(monkeypatch) is False
    assert _check(monkeypatch, agg_dtype="bf16") is True
    assert _check(monkeypatch, agg_dtype="fp8") == "fp8"
    assert _check(monkeypatch, agg_dtype="fp8", model="gcn") == "fp8"


@pytest.mark.parametrize("kw,reason", [
    (dict(model="gat"), "--model gat"),
    (dict(norm="batch"), "--norm batch"),
    (dict(n_linear=1), "--n-linear 1"),
    (dict(use_pp=False), "no --use-pp"),
    (dict(n_hidden=264), "not a multiple of 16"),
], ids=["gat", "batch-norm", "n-linear", "no-use-pp", "hidden-264"])
def test_refused_configurations(built, monkeypatch, kw, reason):
    monkeypatch.delenv("BNS_FUSED", raising=False)
    with pytest.raises(ValueError, match="--agg-dtype fp8 needs the fused training step") as e:
        _check(monkeypatch, agg_dtype="fp8", **kw)
    assert reason in str(e.value)


def test_refusal_names_every_reason(built, monkeypatch):
    monkeypatch.setenv("BNS_FUSED", "0")
    with pytest.raises(ValueError) as e:
        _check(monkeypatch, agg_dtype="fp8", model="gat", norm="batch", n_hidden=264, _dev=torch.device("cpu"))
    for reason in ("BNS_FUSED=0", "--model gat", "--norm batch", "no CUDA device", "not a multiple of 16"):
        assert reason in str(e.value), reason


def test_hidden_264_is_fine_for_bf16(built, monkeypatch):
    monkeypatch.delenv("BNS_FUSED", raising=False)
    assert _check(monkeypatch, agg_dtype="bf16", n_hidden=264) is True


def test_scale_rule_edges():
    x = torch.tensor([[448.0, 1.0], [448.00003, 0.0], [449.0, 0.0], [224.0, 0.0], [224.00002, 0.0], [1.0, 0.0],
                      [0.0, 0.0], [-0.0, 0.0], [2.0 ** -126, 0.0], [1e-40, -1e-45], [3.0e38, 0.0]])
    e, bad = Q.scale_exponents(x)
    assert e.tolist() == [0, 1, 1, -1, 0, -8, 0, 0, -126, -126, 120]
    assert not bad.any()
    codes, scale = Q.quantize_rows(x)
    assert scale.tolist()[:6] == [1.0, 2.0, 2.0, 0.5, 1.0, 2.0 ** -8]
    assert _u8(codes[0]) == [0x7e, 0x38]                  # 448 is the largest code; 1.0 = 0x38
    assert codes.float().abs().max() <= 448.0             # never saturates


def test_ties_round_to_even_and_subnormal_codes():
    # scale 1 (max 448): 400 lies halfway between 384 (0x7c, even) and 416 (0x7d); 432 between 416 and 448 (0x7e, even)
    x = torch.tensor([[448.0, 400.0, 432.0, -400.0, 2.0 ** -9, 3 * 2.0 ** -10, 2.0 ** -10, 2.0 ** -11, -2.0 ** -9]])
    codes, scale = Q.quantize_rows(x)
    assert scale.item() == 1.0
    assert _u8(codes[0]) == [0x7e, 0x7c, 0x7e, 0xfc, 0x01, 0x02, 0x00, 0x00, 0x81]
    # 3 * 2^-10 is halfway between codes 1 and 2 (even: 2); 2^-10 halfway between 0 and 1 (even: 0)


def test_zero_and_tiny_rows():
    codes, scale = Q.quantize_rows(torch.tensor([[0.0, 0.0], [-0.0, 0.0], [1e-39, -1e-39], [1e-45, 0.0]]))
    assert scale.tolist() == [1.0, 1.0, 2.0 ** -126, 2.0 ** -126]
    assert _u8(codes[0]) == [0, 0] and _u8(codes[1]) == [0x80, 0]
    assert (Q.dequantize(codes, scale)[2] == torch.tensor([1e-39, -1e-39]).double()).tolist() == [False, False]
    assert Q.dequantize(codes, scale)[2, 0] > 0 and Q.dequantize(codes, scale)[2, 1] < 0


@pytest.mark.parametrize("v", [float("nan"), float("inf"), -float("inf")])
def test_nonfinite_rows(v):
    x = torch.tensor([[1.0, v, 3.0], [1.0, 2.0, 3.0]])
    codes, scale = Q.quantize_rows(x)
    assert torch.isnan(scale[0]) and _u8(codes[0]) == [0, 0, 0]
    assert scale[1].item() == 2.0 ** -7
    d = Q.dequantize(codes, scale)
    assert torch.isnan(d[0]).all() and torch.isfinite(d[1]).all()


def test_dequantized_within_half_a_code():
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(200, 64, generator=gen) * torch.exp2(torch.randint(-30, 30, (200, 1), generator=gen).float())
    codes, scale = Q.quantize_rows(x)
    d = Q.dequantize(codes, scale)
    # 3 mantissa bits: a relative error of at most 2^-4 for normal codes; below the smallest normal, half a subnormal step
    err = (d - x.double()).abs()
    lim = torch.maximum(x.double().abs() * 2.0 ** -4, scale.double().unsqueeze(1) * 2.0 ** -10)
    assert bool((err <= lim).all())


def test_fingerprint_refuses_bf16_to_fp8(built):
    from bns_gcn_b200.state import fingerprint_mismatches
    saved = vars(make_args(agg_dtype="bf16"))
    why = fingerprint_mismatches(saved, dict(saved, agg_dtype="fp8"))
    assert why == ["agg_dtype is 'fp8', the state's 'bf16'"]
    assert fingerprint_mismatches(saved, dict(saved)) == []
