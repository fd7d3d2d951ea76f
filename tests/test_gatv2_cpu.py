"""``--model gatv2`` on the host: the parser, the model's construction (GAT's stack with ``GATv2Conv`` layers), the
head and width limits, the dtype flags' refusal, and the parameter names and initialisation order."""
import pytest
import torch
from torch import nn

from tests.harness import make_args


def _model(**kw):
    from bns_gcn_b200 import train
    args = make_args(model="gatv2", n_train=50, **kw)
    return train.create_model([10, args.n_hidden, args.n_hidden, 3][:args.n_layers + 1], args)


def test_parser_takes_gatv2():
    from bns_gcn_b200.helper.parser import build_parser, create_parser
    assert create_parser(["--model", "gatv2", "--heads", "4"]).model == "gatv2"
    assert "gatv2" in build_parser().format_help()


def test_model_is_gat_with_gatv2_layers():
    from bns_gcn_b200.module.gatv2 import GATv2Conv
    from bns_gcn_b200.module.model import GAT
    torch.manual_seed(0)
    m = _model(heads=2, n_layers=3, n_hidden=8)
    assert type(m) is GAT and m.use_pp
    assert all(isinstance(layer, GATv2Conv) for layer in m.layers)
    assert [layer._layer_index for layer in m.layers] == [0, 1, 2]
    assert all(isinstance(n, nn.LayerNorm) for n in m.norm)
    m = _model(heads=1, n_layers=3, n_hidden=8, n_linear=1)
    assert isinstance(m.layers[2], nn.Linear)


def test_checkpoint_keys_and_init_order():
    """Keys ``layers.i.fc_src.weight`` / ``.bias``, ``fc_dst.*`` and ``attn``; no separate bias; initialisation draws
    fc_src.weight, fc_dst.weight, then attn (xavier-normal, ReLU gain) after the two Linear constructors, biases 0."""
    from bns_gcn_b200.module.gatv2 import GATv2Conv
    torch.manual_seed(5)
    layer = GATv2Conv(12, 6, 3, 0.5, 0.5)
    assert list(layer.state_dict()) == ["attn", "fc_src.weight", "fc_src.bias", "fc_dst.weight", "fc_dst.bias"]
    assert layer.attn.shape == (1, 3, 6) and layer.fc_src.weight.shape == (18, 12)
    torch.manual_seed(5)
    fs, fd = nn.Linear(12, 18), nn.Linear(12, 18)
    attn = torch.empty(1, 3, 6)
    gain = nn.init.calculate_gain("relu")
    nn.init.xavier_normal_(fs.weight, gain=gain)
    nn.init.xavier_normal_(fd.weight, gain=gain)
    nn.init.xavier_normal_(attn, gain=gain)
    assert torch.equal(layer.fc_src.weight, fs.weight) and torch.equal(layer.fc_dst.weight, fd.weight)
    assert torch.equal(layer.attn, attn)
    assert torch.all(layer.fc_src.bias == 0) and torch.all(layer.fc_dst.bias == 0)
    m = _model(heads=2, n_layers=2, n_hidden=8)
    assert {k for k in m.state_dict() if k.startswith("layers.1.")} == {
        "layers.1.attn", "layers.1.fc_src.weight", "layers.1.fc_src.bias", "layers.1.fc_dst.weight",
        "layers.1.fc_dst.bias"}


@pytest.mark.parametrize("heads,hidden,what", [(9, 8, "heads = 9"), (0, 8, "heads = 0"),
                                                (8, 129, "8 \\* 132 exceeds 1024"), (1, 1025, "1 \\* 1028")])
def test_limits_are_refused_when_the_model_is_built(heads, hidden, what):
    with pytest.raises(NotImplementedError, match=what):
        _model(heads=heads, n_layers=2, n_hidden=hidden)


def test_unsupported_constructor_arguments_are_refused():
    from bns_gcn_b200.module.gatv2 import GATv2Conv
    for kw in (dict(residual=True), dict(activation=torch.relu), dict(share_weights=True)):
        with pytest.raises(NotImplementedError, match="GATv2Conv"):
            GATv2Conv(8, 4, 1, **kw)


@pytest.mark.parametrize("flag", ["agg", "comm", "dense"])
def test_dtype_flags_refuse_gatv2(flag):
    from bns_gcn_b200 import train
    args = make_args(model="gatv2", n_hidden=64, **{f"{flag}_dtype": "bf16"})
    with pytest.raises(ValueError, match="--model gatv2 \\(only graphsage and gcn have the fused step\\)"):
        getattr(train, f"check_{flag}_dtype")(args, [16, 64, 64, 4], torch.device("cpu"))


def test_oracle_kind_initialises_and_computes_like_the_layer():
    """The oracle's ``GATv2ConvRef`` draws the same initial parameters as ``GATv2Conv`` under one seed, and its
    forward equals the float64 restatement of tests/gatv2_reference.py on a random edge list."""
    from bns_gcn_b200.module.gatv2 import GATv2Conv
    from oracle.bns_oracle import EdgeList
    from tests.gatv2_oracle import GATv2ConvRef
    from tests.gatv2_reference import gatv2_attention_reference
    torch.manual_seed(3)
    layer = GATv2Conv(12, 6, 2, 0.0, 0.0)
    torch.manual_seed(3)
    ref = GATv2ConvRef(12, 6, 2, 0.0, 0.0)
    assert list(layer.state_dict()) == list(ref.state_dict())
    assert all(torch.equal(a, b) for a, b in zip(layer.state_dict().values(), ref.state_dict().values()))
    gen = torch.Generator().manual_seed(4)
    n_u, n_v, nnz = 30, 20, 120
    u, v = torch.randint(0, n_u, (nnz,), generator=gen), torch.randint(0, n_v, (nnz,), generator=gen)
    g = EdgeList(u, v, n_u, n_v)
    hs, hd = torch.randn(n_u, 12, generator=gen), torch.randn(n_v, 12, generator=gen)
    with torch.no_grad():
        got = ref(g, (hs, hd))
        zs, zd = ref.fc_src(hs), ref.fc_dst(hd)
    want = gatv2_attention_reference(zs, zd, ref.attn.detach(), u, v, n_v, 2, 6, torch.zeros(n_v, 12))[0]
    assert torch.allclose(got.double().reshape(n_v, 12), want, rtol=1e-5, atol=1e-6)


def test_oracle_kind_runs_a_gatv2_configuration(monkeypatch):
    """``oracle_kind`` runs ``--model gatv2`` through the oracle's rank with ``GATv2Ref``; its loss falls."""
    from bns_gcn_b200.data import make_graph, partition_graph
    from tests import harness
    from tests.gatv2_oracle import GATv2Ref, oracle_kind
    fg = make_graph("tiny", seed=0)
    parts = partition_graph(fg, 2, "random", seed=0)
    args = make_args(model="gatv2", n_layers=2, heads=2, n_partitions=2, sampling_rate=1.0)
    from oracle import bns_oracle as O
    built = []
    real = O.OracleRank.__init__

    def spy(self, *a, **kw):
        real(self, *a, **kw)
        built.append(type(self.net))
    monkeypatch.setattr(O.OracleRank, "__init__", spy)
    with oracle_kind(monkeypatch):
        out = harness.run_oracle(parts, args, 3, None)
    assert built == [GATv2Ref, GATv2Ref]
    loss = [sum(o["loss"][e] for o in out) for e in range(3)]
    assert loss[2] < loss[0]
