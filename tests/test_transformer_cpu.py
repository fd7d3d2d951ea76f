"""``--model transformer`` on the host: the parser, the model's construction (GAT's stack with ``TransformerConv``
layers), checkpoint keys, initialisation order and padding, the head and width limits and the refused constructor
arguments, the dtype flags' refusal, the exchange ratio, and the oracle's ``transformer`` kind against the layer's
float64 restatement."""
import math

import pytest
import torch
from torch import nn

from tests.harness import make_args


def _model(**kw):
    from bns_gcn_b200 import train
    args = make_args(model="transformer", n_train=50, **kw)
    return train.create_model([10, args.n_hidden, args.n_hidden, 3][:args.n_layers + 1], args)


def test_parser_takes_transformer():
    from bns_gcn_b200.helper.parser import build_parser, create_parser
    assert create_parser(["--model", "transformer", "--heads", "4"]).model == "transformer"
    assert "transformer" in build_parser().format_help()


def test_model_is_gat_stack_with_transformer_layers():
    from bns_gcn_b200.module.model import GAT
    from bns_gcn_b200.module.sync_bn import SyncBatchNorm
    from bns_gcn_b200.module.transformer import TransformerConv
    torch.manual_seed(0)
    m = _model(heads=2, n_layers=3, n_hidden=8, dropout=0.3)
    assert type(m) is GAT and m.use_pp
    assert all(isinstance(layer, TransformerConv) for layer in m.layers)
    assert [layer._layer_index for layer in m.layers] == [0, 1, 2]
    assert all(layer.feat_drop.p == 0.3 and layer.attn_drop.p == 0.3 for layer in m.layers)
    assert all(layer._num_heads == 2 for layer in m.layers)
    assert all(isinstance(n, nn.LayerNorm) for n in m.norm)
    m = _model(heads=1, n_layers=3, n_hidden=8, n_linear=1, norm="batch")
    assert isinstance(m.layers[2], nn.Linear)
    assert all(isinstance(n, SyncBatchNorm) and n.whole_size == 50 for n in m.norm)


def test_checkpoint_keys_and_init_order():
    """Keys ``lin_key``, ``lin_query``, ``lin_value`` (``[H * C, in]``) and ``lin_skip`` (``[C, in]``), each with a
    bias, created in that order with ``nn.Linear``'s own initialisation."""
    from bns_gcn_b200.module.transformer import TransformerConv
    torch.manual_seed(5)
    layer = TransformerConv(12, 6, 3, 0.5, 0.5)
    names = [f"{lin}.{p}" for lin in ("lin_key", "lin_query", "lin_value", "lin_skip") for p in ("weight", "bias")]
    assert list(layer.state_dict()) == names
    assert [n for n, _ in layer.named_parameters()] == names
    assert layer.lin_key.weight.shape == (18, 12) and layer.lin_skip.weight.shape == (6, 12)
    torch.manual_seed(5)
    want = [nn.Linear(12, 18), nn.Linear(12, 18), nn.Linear(12, 18), nn.Linear(12, 6)]
    for lin, w in zip((layer.lin_key, layer.lin_query, layer.lin_value, layer.lin_skip), want):
        assert torch.equal(lin.weight, w.weight) and torch.equal(lin.bias, w.bias)
    m = _model(heads=2, n_layers=2, n_hidden=8)
    assert {k for k in m.state_dict() if k.startswith("layers.1.")} == {f"layers.1.{n}" for n in names}
    no_root = TransformerConv(12, 6, 1, root_weight=False, bias=False)
    assert list(no_root.state_dict()) == ["lin_key.weight", "lin_query.weight", "lin_value.weight"]


def test_padding_is_zero_rows_of_q_k_v_and_keeps_the_unpadded_scale():
    """C = 5 pads every head to 8: zero rows of the query, key and value weights and biases; k and v are stacked."""
    from bns_gcn_b200.module.transformer import TransformerConv
    layer = TransformerConv(12, 5, 3)
    H, C, Cp, wq, bq, wkv, bkv = layer._padded_params()
    assert (H, C, Cp) == (3, 5, 8)
    assert wq.shape == (24, 12) and bq.shape == (24,) and wkv.shape == (48, 12) and bkv.shape == (48,)
    for w, b, lin in ((wq, bq, layer.lin_query), (wkv[:24], bkv[:24], layer.lin_key),
                      (wkv[24:], bkv[24:], layer.lin_value)):
        w3, b2 = w.view(3, 8, 12), b.view(3, 8)
        assert torch.equal(w3[:, :5], lin.weight.view(3, 5, 12)) and torch.all(w3[:, 5:] == 0)
        assert torch.equal(b2[:, :5], lin.bias.view(3, 5)) and torch.all(b2[:, 5:] == 0)
    unpadded = TransformerConv(12, 8, 2)
    _, _, Cp, wq8, _, wkv8, _ = unpadded._padded_params()
    assert Cp == 8 and wq8 is unpadded.lin_query.weight
    assert torch.equal(wkv8, torch.cat([unpadded.lin_key.weight, unpadded.lin_value.weight]))
    # the pad columns add 0 to every dot product: the padded scores equal the unpadded ones
    x = torch.randn(7, 12)
    with torch.no_grad():
        q = (x @ wq.t() + bq).view(7, 3, 8)
        k = (x @ wkv[:24].t() + bkv[:24]).view(7, 3, 8)
        q0, k0 = layer.lin_query(x).view(7, 3, 5), layer.lin_key(x).view(7, 3, 5)
    assert torch.allclose((q * k).sum(-1) / math.sqrt(5), (q0 * k0).sum(-1) / math.sqrt(5), rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("heads,hidden,what", [(9, 8, "heads = 9"), (0, 8, "heads = 0"),
                                                (8, 129, "8 \\* 132 exceeds 1024"), (1, 1025, "1 \\* 1028")])
def test_limits_are_refused_when_the_model_is_built(heads, hidden, what):
    with pytest.raises(NotImplementedError, match=what):
        _model(heads=heads, n_layers=2, n_hidden=hidden)
    _model(heads=4, n_layers=2, n_hidden=256)                 # 4 * 256 = 1024 is taken


def test_unsupported_constructor_arguments_are_refused():
    from bns_gcn_b200.module.transformer import TransformerConv
    for kw in (dict(beta=True), dict(edge_dim=4), dict(concat=True)):
        with pytest.raises(NotImplementedError, match="TransformerConv"):
            TransformerConv(8, 4, 1, **kw)


@pytest.mark.parametrize("flag", ["agg", "comm", "dense"])
def test_dtype_flags_refuse_transformer(flag):
    from bns_gcn_b200 import train
    args = make_args(model="transformer", n_hidden=64, **{f"{flag}_dtype": "bf16"})
    with pytest.raises(ValueError, match="--model transformer \\(only graphsage and gcn have the fused step\\)"):
        getattr(train, f"check_{flag}_dtype")(args, [16, 64, 64, 4], torch.device("cpu"))


@pytest.mark.parametrize("rank", [0, 1, 2])
def test_exchange_ratio_is_one_for_transformer(monkeypatch, rank):
    from bns_gcn_b200 import train
    monkeypatch.setattr(train, "_rank_size", lambda: (rank, 3))
    boundary = [torch.arange(n) for n in (10, 7, 4)]
    _, ratio = train.get_send_size(boundary, 0.3)
    assert train.exchange_ratio("transformer", ratio) == [0 if i == rank else 1.0 for i in range(3)]
    for model in ("graphsage", "gcn", "gat", "gatv2"):
        assert train.exchange_ratio(model, ratio) is ratio
    assert [r for i, r in enumerate(ratio) if i != rank] != [1.0, 1.0]


def test_attention_stack_names_every_model_on_gat_stack():
    from bns_gcn_b200 import train
    assert train.ATTENTION_STACK == ('gat', 'gatv2', 'graphsage-pool', 'transformer')


def test_reference_gradients_match_central_differences():
    """The float64 restatement's autograd gradients of ``<rst, d>`` against central differences, every 7th element
    of q, k and v."""
    from tests.transformer_reference import tconv_attention_reference
    gen = torch.Generator().manual_seed(1)
    H, Fp, n_u, n_v, nnz = 2, 4, 9, 6, 25
    src, dst = torch.randint(0, n_u, (nnz,), generator=gen), torch.randint(0, n_v, (nnz,), generator=gen)
    q, k, val = (torch.randn(n, H * Fp, generator=gen, dtype=torch.float64) for n in (n_v, n_u, n_u))
    d = torch.randn(n_v, H * Fp, generator=gen, dtype=torch.float64)
    _, dq, dk, dv, _ = tconv_attention_reference(q, k, val, src, dst, n_v, H, Fp, d, 0.5)
    eps = 1e-6
    for t, g in ((q, dq), (k, dk), (val, dv)):
        for i in range(0, t.numel(), 7):
            tp, tm = t.clone(), t.clone()
            tp.view(-1)[i] += eps
            tm.view(-1)[i] -= eps
            args_p = [tp if x is t else x for x in (q, k, val)]
            args_m = [tm if x is t else x for x in (q, k, val)]
            fp = (tconv_attention_reference(*args_p, src, dst, n_v, H, Fp, d, 0.5)[0] * d).sum()
            fm = (tconv_attention_reference(*args_m, src, dst, n_v, H, Fp, d, 0.5)[0] * d).sum()
            assert abs((fp - fm).item() / (2 * eps) - g.view(-1)[i].item()) < 1e-6


def test_oracle_kind_initialises_and_computes_like_the_layer():
    """The oracle's ``TransformerConvRef`` draws the same initial parameters as ``TransformerConv`` under one seed, and
    its forward and gradients equal the float64 restatement of tests/transformer_reference.py on a random edge list."""
    from bns_gcn_b200.module.transformer import TransformerConv
    from oracle.bns_oracle import EdgeList
    from tests.transformer_oracle import TransformerConvRef
    from tests.transformer_reference import transformer_layer_reference
    torch.manual_seed(3)
    layer = TransformerConv(12, 6, 2, 0.0, 0.0)
    torch.manual_seed(3)
    ref = TransformerConvRef(12, 6, 2, 0.0, 0.0)
    assert list(layer.state_dict()) == list(ref.state_dict())
    assert all(torch.equal(a, b) for a, b in zip(layer.state_dict().values(), ref.state_dict().values()))
    gen = torch.Generator().manual_seed(4)
    n_u, n_v, nnz = 30, 20, 120
    u, v = torch.randint(0, n_u, (nnz,), generator=gen), torch.randint(0, n_v, (nnz,), generator=gen)
    g = EdgeList(u, v, n_u, n_v)
    hs = torch.randn(n_u, 12, generator=gen).requires_grad_(True)
    got = ref(g, (hs, hs[:n_v]))
    assert got.shape == (n_v, 2, 6)
    d = torch.randn(n_v, 2, 6, generator=gen)
    got.backward(d)
    lins = (ref.lin_query, ref.lin_key, ref.lin_value, ref.lin_skip)
    params = [t.detach().double().requires_grad_(True) for lin in lins for t in (lin.weight, lin.bias)]
    x = hs.detach().double().requires_grad_(True)
    want = transformer_layer_reference(x, u, v, n_v, *params, 2, 6)
    (want * d.double()).sum().backward()
    assert torch.allclose(got.double(), want, rtol=1e-5, atol=1e-6)
    assert torch.allclose(hs.grad.double(), x.grad, rtol=1e-5, atol=1e-6)
    for p, w in zip([t for lin in lins for t in (lin.weight, lin.bias)], params):
        assert torch.allclose(p.grad.double(), w.grad, rtol=1e-5, atol=1e-5)


def test_oracle_kind_runs_a_transformer_configuration(monkeypatch):
    """``oracle_kind`` runs ``--model transformer`` through the oracle's rank with ``TransformerRef`` and a ratio of
    1.0; its loss falls."""
    from bns_gcn_b200.data import make_graph, partition_graph
    from oracle import bns_oracle as O
    from tests import harness
    from tests.transformer_oracle import TransformerRef, oracle_kind
    fg = make_graph("tiny", seed=0)
    parts = partition_graph(fg, 2, "random", seed=0)
    args = make_args(model="transformer", n_layers=2, heads=2, n_partitions=2, sampling_rate=0.5)
    built, ratios = [], []
    real = O.OracleRank.__init__

    def spy(self, *a, **kw):
        real(self, *a, **kw)
        built.append(type(self.net))
        ratios.append(list(self.ratio))
    monkeypatch.setattr(O.OracleRank, "__init__", spy)
    with oracle_kind(monkeypatch):
        out = harness.run_oracle(parts, args, 3, None)
    assert built == [TransformerRef, TransformerRef]
    assert sorted(ratios) == [[0, 1.0], [1.0, 0]]
    loss = [sum(o["loss"][e] for o in out) for e in range(3)]
    assert loss[2] < loss[0]
