"""``--model graphsage-pool`` on the host: the parser, the model's construction (GAT's stack with one-head
``SAGEPoolConv`` layers), the width limit, the dtype flags' refusal, the parameter names and initialisation order, the
exchange ratio, and the oracle's ``graphsage-pool`` kind against the layer's restatement."""
import pytest
import torch
from torch import nn

from tests.harness import make_args


def _model(**kw):
    from bns_gcn_b200 import train
    args = make_args(model="graphsage-pool", n_train=50, **kw)
    return train.create_model([kw.pop("n_feat", 10), args.n_hidden, args.n_hidden, 3][:args.n_layers + 1], args)


def test_parser_takes_graphsage_pool():
    from bns_gcn_b200.helper.parser import build_parser, create_parser
    assert create_parser(["--model", "graphsage-pool"]).model == "graphsage-pool"
    assert "graphsage-pool" in build_parser().format_help()


def test_model_is_gat_stack_with_sage_pool_layers():
    from bns_gcn_b200.module.model import GAT
    from bns_gcn_b200.module.sage_pool import SAGEPoolConv
    from bns_gcn_b200.module.sync_bn import SyncBatchNorm
    torch.manual_seed(0)
    m = _model(heads=4, n_layers=3, n_hidden=8, dropout=0.3)
    assert type(m) is GAT and m.use_pp
    assert all(isinstance(layer, SAGEPoolConv) for layer in m.layers)
    assert all(layer.feat_drop.p == 0.3 for layer in m.layers)
    assert all(isinstance(n, nn.LayerNorm) for n in m.norm)
    m = _model(n_layers=3, n_hidden=8, n_linear=1, norm="batch")
    assert isinstance(m.layers[2], nn.Linear)
    assert all(isinstance(n, SyncBatchNorm) and n.whole_size == 50 for n in m.norm)


def test_checkpoint_keys_and_init_order():
    """Keys ``bias``, ``fc_pool.weight`` / ``.bias``, ``fc_self.weight``, ``fc_neigh.weight``; the constructors draw in
    the order fc_pool, fc_self, fc_neigh, then the three weights are redrawn xavier-uniform (ReLU gain) in that order;
    fc_pool.bias keeps nn.Linear's draw and bias is 0."""
    from bns_gcn_b200.module.sage_pool import SAGEPoolConv
    torch.manual_seed(5)
    layer = SAGEPoolConv(12, 6, 0.5)
    assert list(layer.state_dict()) == ["bias", "fc_pool.weight", "fc_pool.bias", "fc_self.weight", "fc_neigh.weight"]
    assert [n for n, _ in layer.named_parameters()] == list(layer.state_dict())
    assert layer.fc_pool.weight.shape == (12, 12) and layer.fc_self.weight.shape == (6, 12)
    torch.manual_seed(5)
    fp, fs, fn = nn.Linear(12, 12), nn.Linear(12, 6, bias=False), nn.Linear(12, 6, bias=False)
    gain = nn.init.calculate_gain("relu")
    for lin in (fp, fs, fn):
        nn.init.xavier_uniform_(lin.weight, gain=gain)
    assert torch.equal(layer.fc_pool.weight, fp.weight) and torch.equal(layer.fc_pool.bias, fp.bias)
    assert torch.equal(layer.fc_self.weight, fs.weight) and torch.equal(layer.fc_neigh.weight, fn.weight)
    assert torch.all(layer.bias == 0)
    m = _model(n_layers=2, n_hidden=8)
    assert {k for k in m.state_dict() if k.startswith("layers.1.")} == {
        "layers.1.bias", "layers.1.fc_pool.weight", "layers.1.fc_pool.bias", "layers.1.fc_self.weight",
        "layers.1.fc_neigh.weight"}


def test_padding_is_zero_rows_of_fc_pool_and_zero_columns_of_fc_neigh():
    from bns_gcn_b200.module.sage_pool import SAGEPoolConv
    layer = SAGEPoolConv(602, 16)
    wp, bp, wn = layer._padded_params()
    assert wp.shape == (604, 602) and bp.shape == (604,) and wn.shape == (16, 604)
    assert torch.equal(wp[:602], layer.fc_pool.weight) and torch.all(wp[602:] == 0) and torch.all(bp[602:] == 0)
    assert torch.equal(wn[:, :602], layer.fc_neigh.weight) and torch.all(wn[:, 602:] == 0)
    wp, bp, wn = SAGEPoolConv(256, 16)._padded_params()
    assert wp.shape == (256, 256) and wn.shape == (16, 256)


@pytest.mark.parametrize("n_feat", [1025, 1027, 2000])
def test_padded_width_above_1024_is_refused_when_the_model_is_built(n_feat):
    with pytest.raises(NotImplementedError, match=f"padded input width {(n_feat + 3) // 4 * 4} exceeds 1024"):
        _model(n_feat=n_feat, n_layers=2, n_hidden=8)
    with pytest.raises(NotImplementedError, match="exceeds 1024"):
        _model(n_layers=2, n_hidden=1100)
    _model(n_feat=1021, n_layers=2, n_hidden=8)           # pads to 1024


@pytest.mark.parametrize("flag", ["agg", "comm", "dense"])
def test_dtype_flags_refuse_graphsage_pool(flag):
    from bns_gcn_b200 import train
    args = make_args(model="graphsage-pool", n_hidden=64, **{f"{flag}_dtype": "bf16"})
    with pytest.raises(ValueError, match="--model graphsage-pool \\(only graphsage and gcn have the fused step\\)"):
        getattr(train, f"check_{flag}_dtype")(args, [16, 64, 64, 4], torch.device("cpu"))


@pytest.mark.parametrize("rank", [0, 1, 2])
def test_exchange_ratio_is_one_for_graphsage_pool_only(monkeypatch, rank):
    from bns_gcn_b200 import train
    monkeypatch.setattr(train, "_rank_size", lambda: (rank, 3))
    boundary = [torch.arange(n) for n in (10, 7, 4)]
    _, ratio = train.get_send_size(boundary, 0.3)
    assert train.exchange_ratio("graphsage-pool", ratio) == [0 if i == rank else 1.0 for i in range(3)]
    for model in ("graphsage", "gcn", "gat", "gatv2"):
        assert train.exchange_ratio(model, ratio) is ratio
    assert [r for i, r in enumerate(ratio) if i != rank] != [1.0, 1.0]


def test_max_reference_takes_the_first_winner_and_credits_it_once():
    from tests.sage_pool_reference import MaxByWinner, max_first
    z = torch.tensor([[1., 0.], [2., 0.], [2., 0.], [0., 3.]], dtype=torch.float64)
    # row 0: entries from sources 1, 2, 1 (source 1 twice; all three tie in both columns); row 1: none; row 2: source 3
    u, v = torch.tensor([1, 2, 1, 3]), torch.tensor([0, 0, 0, 2])
    m, first = max_first(z, u, v, 3)
    assert m.tolist() == [[2., 0.], [0., 0.], [0., 3.]]
    assert first.tolist() == [[0, 0], [-1, -1], [3, 3]]
    zr = z.clone().requires_grad_(True)
    MaxByWinner.apply(zr, u, v, 3).backward(torch.ones(3, 2, dtype=torch.float64))
    assert zr.grad.tolist() == [[0., 0.], [1., 1.], [0., 0.], [1., 1.]]        # source 1 credited once


def test_oracle_kind_initialises_and_computes_like_the_layer():
    """The oracle's ``SAGEPoolConvRef`` draws the same initial parameters as ``SAGEPoolConv`` under one seed, and its
    forward and gradients equal the float64 restatement of tests/sage_pool_reference.py on a random edge list with
    multi-edges."""
    from bns_gcn_b200.module.sage_pool import SAGEPoolConv
    from oracle.bns_oracle import EdgeList
    from tests.sage_pool_oracle import SAGEPoolConvRef
    from tests.sage_pool_reference import sage_pool_layer_reference
    torch.manual_seed(3)
    layer = SAGEPoolConv(12, 6, 0.0)
    torch.manual_seed(3)
    ref = SAGEPoolConvRef(12, 6, 0.0)
    assert list(layer.state_dict()) == list(ref.state_dict())
    assert all(torch.equal(a, b) for a, b in zip(layer.state_dict().values(), ref.state_dict().values()))
    gen = torch.Generator().manual_seed(4)
    n_u, n_v, nnz = 30, 20, 120
    u, v = torch.randint(0, n_u, (nnz,), generator=gen), torch.randint(0, n_v, (nnz,), generator=gen)
    g = EdgeList(u, v, n_u, n_v)
    with torch.no_grad():
        ref.bias.copy_(torch.randn(6, generator=gen))
    hs = torch.randn(n_u, 12, generator=gen).requires_grad_(True)
    got = ref(g, (hs, hs[:n_v]))
    assert got.shape == (n_v, 1, 6)
    d = torch.randn(n_v, 6, generator=gen)
    got.squeeze(1).backward(d)
    params = [p.detach().double().requires_grad_(True) for p in (ref.fc_pool.weight, ref.fc_pool.bias,
                                                                 ref.fc_self.weight, ref.fc_neigh.weight, ref.bias)]
    x = hs.detach().double().requires_grad_(True)
    want = sage_pool_layer_reference(x, u, v, n_v, *params)
    (want * d.double()).sum().backward()
    assert torch.allclose(got.squeeze(1).double(), want, rtol=1e-5, atol=1e-6)
    assert torch.allclose(hs.grad.double(), x.grad, rtol=1e-5, atol=1e-6)
    for p, w in zip((ref.fc_pool.weight, ref.fc_pool.bias, ref.fc_self.weight, ref.fc_neigh.weight, ref.bias), params):
        assert torch.allclose(p.grad.double(), w.grad, rtol=1e-5, atol=1e-5)


def test_oracle_kind_runs_a_graphsage_pool_configuration(monkeypatch):
    """``oracle_kind`` runs ``--model graphsage-pool`` through the oracle's rank with ``SAGEPoolRef`` and a ratio of
    1.0; its loss falls."""
    from bns_gcn_b200.data import make_graph, partition_graph
    from oracle import bns_oracle as O
    from tests import harness
    from tests.sage_pool_oracle import SAGEPoolRef, oracle_kind
    fg = make_graph("tiny", seed=0)
    parts = partition_graph(fg, 2, "random", seed=0)
    args = make_args(model="graphsage-pool", n_layers=2, n_partitions=2, sampling_rate=0.5)
    built, ratios = [], []
    real = O.OracleRank.__init__

    def spy(self, *a, **kw):
        real(self, *a, **kw)
        built.append(type(self.net))
        ratios.append(list(self.ratio))
    monkeypatch.setattr(O.OracleRank, "__init__", spy)
    with oracle_kind(monkeypatch):
        out = harness.run_oracle(parts, args, 3, None)
    assert built == [SAGEPoolRef, SAGEPoolRef]
    assert sorted(ratios) == [[0, 1.0], [1.0, 0]]
    loss = [sum(o["loss"][e] for o in out) for e in range(3)]
    assert loss[2] < loss[0]
