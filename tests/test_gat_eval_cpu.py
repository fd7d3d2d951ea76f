"""CPU side of GAT's evaluation forward: the oracle reproduces the reference's GAT evaluation logits
(tests/golden/ref_gat_eval_p2.pt), and the limits of the one-pass attention kernel are named."""
import os

import torch

from tests.test_oracle_cpu import GOLD, _oracle_run, _rel


def test_oracle_gat_evaluation_forward_reproduces_the_reference():
    """make_golden_gat_eval.py trained the reference's GAT (2 heads, closing width 5) for two epochs and ran its evaluation
    forward (train.py:44-49: model.eval(); model(g, feat); GATConv's homogeneous call) on the whole graph.  The oracle,
    trained on the same index sets and evaluated the same way, gives the same logits, and holds the same weights."""
    import bns_gcn_b200  # noqa: F401
    from bns_gcn_b200.data import make_graph
    from oracle import bns_oracle as O
    gold = torch.load(os.path.join(GOLD, "ref_gat_eval_p2.pt"))
    cfg, ranks = gold["config"], gold["ranks"]
    assert cfg["model"] == "gat" and cfg["heads"] == 2
    sel = [[ranks[r]["selected"][e] for r in range(cfg["n_parts"])] for e in range(cfg["epochs"])]
    out = _oracle_run(cfg, sel)
    net = out[0].net
    for p, gp in zip(net.parameters(), ranks[0]["params"]):
        assert _rel(p.detach(), gp) < 1e-5
    fg = make_graph(cfg["shape"], seed=0, device=torch.device("cpu"))
    net.eval()
    out[0].trace = None
    with torch.no_grad():
        logits = net(O.EdgeList(fg.src, fg.dst(), fg.n_nodes, fg.n_nodes), fg.feat)
    want = ranks[0]["eval_logits"]
    assert logits.shape == want.shape == (fg.n_nodes, fg.n_class)
    assert _rel(logits, want) < 1e-5


def test_gat_unsupported_names_the_exceeded_limit():
    """Heads 1..8 and heads * (per-head width rounded up to 4) <= 1024, the limits of every GAT kernel; anything else is
    named, so GATConv can say which limit keeps it from being built."""
    from bns_gcn_b200.graph import gat_padded_width, gat_unsupported
    assert [gat_padded_width(f) for f in (1, 4, 5, 41, 256)] == [4, 4, 8, 44, 256]
    for H, Fo in ((1, 5), (2, 5), (4, 256), (8, 128), (1, 1024), (8, 125)):
        assert gat_unsupported(H, Fo) is None, (H, Fo)
    assert "heads" in gat_unsupported(9, 16)
    assert "1024" in gat_unsupported(8, 129)
    assert "1024" in gat_unsupported(1, 1025)
    assert gat_unsupported(2, 0) is not None


def test_gatconv_refuses_layers_beyond_the_kernel_limits():
    """A layer the attention kernels cannot run is refused when the model is built, naming the limit; a per-head width
    that is not a multiple of 4 builds (it runs padded)."""
    import pytest
    from bns_gcn_b200.module.gat import GATConv
    with pytest.raises(NotImplementedError, match="heads = 9 is outside 1..8"):
        GATConv(16, 16, 9)
    with pytest.raises(NotImplementedError, match="1028 exceeds 1024"):
        GATConv(16, 1025, 1)
    layer = GATConv(16, 41, 1)
    assert layer.fc.weight.shape == (41, 16) and layer.attn_l.shape == (1, 1, 41)


def test_gat_conv_full_graph_training_call_raises():
    """Training on the full graph is not a call the reference makes: GATConv refuses it before touching the graph."""
    import pytest
    from bns_gcn_b200.graph import FullGraphHandle
    from bns_gcn_b200.module.gat import GATConv
    layer = GATConv(8, 5, 2)
    g = FullGraphHandle(None, torch.ones(3), torch.ones(3))
    with pytest.raises(NotImplementedError):
        layer(g, torch.zeros(3, 8))
