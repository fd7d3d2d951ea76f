"""``--model gatv2`` end to end: ``GATv2Conv``'s training call against float64 (fc_src, fc_dst, the attention and every
gradient, padded per-head widths included), ``--cuda-graph`` replays bit-identical to eager epochs, ``--resume`` bit for
bit, the partition-parallel evaluation (transductive and inductive) against the whole-graph ``Evaluator``, and the
checkpoint keys.  Training against the CPU oracle is in test_gatv2_parity_gpu."""
import argparse

import pytest
import torch

from tests.gatv2_reference import gatv2_attention_reference
from tests.test_gat_train_attention_gpu import N_IN, SLOPE, _crafted

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / b.norm().clamp(min=1e-30)).item()


@pytest.mark.parametrize("H,Fo", [(3, 40), (1, 41), (2, 5)])
def test_gatv2conv_training_matches_float64(built, H, Fo):
    from bns_gcn_b200.module import dense
    from bns_gcn_b200.module.gatv2 import GATv2Conv
    F_in = 24
    case = _crafted(H, 91 + Fo)
    torch.manual_seed(Fo)
    layer = GATv2Conv(F_in, Fo, H, 0.0, 0.0).to(DEV).train()
    gen = torch.Generator().manual_seed(92)
    with torch.no_grad():                                  # (the biases are initialised to 0)
        layer.fc_src.bias.copy_(torch.randn(H * Fo, generator=gen))
        layer.fc_dst.bias.copy_(torch.randn(H * Fo, generator=gen))
    h_src = torch.randn(case.n_u, F_in, generator=gen)
    h_dst = torch.randn(N_IN, F_in, generator=gen)
    d = torch.randn(N_IN, H, Fo, generator=gen)
    hs, hd = h_src.to(DEV).requires_grad_(True), h_dst.to(DEV).requires_grad_(True)
    out = layer(case.g, (hs, hd))
    out.backward(d.to(DEV))
    got = [out, hs.grad, hd.grad, layer.fc_src.weight.grad, layer.fc_src.bias.grad, layer.fc_dst.weight.grad,
           layer.fc_dst.bias.grad, layer.attn.grad]
    ws, bs, wd, bd, at = (t.detach().double().cpu().requires_grad_(True) for t in
                          (layer.fc_src.weight, layer.fc_src.bias, layer.fc_dst.weight, layer.fc_dst.bias, layer.attn))
    xs, xd = h_src.double().requires_grad_(True), h_dst.double().requires_grad_(True)
    zs, zd = xs @ ws.t() + bs, xd @ wd.t() + bd
    # the attention of the float64 restatement runs on the layer's own z (its f32 GEMMs): an entry whose z_src + z_dst
    # lies within the GEMMs' rounding of 0 would otherwise take the other LeakyReLU branch in one of the two
    _, _, Fp, w_s, b_s, w_d, b_d, _ = layer._padded_params()
    with torch.no_grad():
        z32 = [dense.linear(x, w_, b_).view(-1, H, Fp)[..., :Fo].reshape(-1, H * Fo).double().cpu()
               for x, w_, b_ in ((hs, w_s, b_s), (hd, w_d, b_d))]
    rst, d_zs, d_zd, d_at, _ = gatv2_attention_reference(z32[0], z32[1], at.detach(), case.u, case.v, N_IN,
                                                         H, Fo, d.reshape(N_IN, H * Fo), SLOPE)
    ((zs * d_zs).sum() + (zd * d_zd).sum() + (at.reshape(-1) * d_at).sum()).backward()
    want = [rst.view(-1, H, Fo), xs.grad, xd.grad, ws.grad, bs.grad, wd.grad, bd.grad, at.grad]
    names = ["out", "d h_src", "d h_dst", "d fc_src.weight", "d fc_src.bias", "d fc_dst.weight", "d fc_dst.bias",
             "d attn"]
    for name, g_, w_ in zip(names, got, want):
        assert g_ is not None and g_.shape == w_.shape, (H, Fo, name)
        assert _rel(g_, w_) < (2e-5 if name == "out" else 5e-5), (H, Fo, name, _rel(g_, w_))


@pytest.mark.parametrize("kw", [dict(heads=1, n_layers=2), dict(heads=2, n_layers=2),
                                dict(heads=2, n_layers=3, n_linear=1)], ids=["1head", "2heads", "2heads-n-linear1"])
def test_gatv2_replayed_run_equals_the_eager_run(built, tmp_path, monkeypatch, capsys, kw):
    from tests.test_cuda_graph_cli_gpu import _args, _check_same, _train
    kw = dict(model="gatv2", **kw)
    eager = _train(_args(**kw), monkeypatch, capsys, tmp_path / "eager")
    graphed = _train(_args(cuda_graph=True, **kw), monkeypatch, capsys, tmp_path / "graph")
    _check_same(eager, graphed)
    assert eager["fused"] is False and graphed["fused"] is False
    keys = set(eager["model"])
    for i in range(kw["n_layers"] - kw.get("n_linear", 0)):
        assert {f"layers.{i}.{n}" for n in ("fc_src.weight", "fc_src.bias", "fc_dst.weight", "fc_dst.bias",
                                             "attn")} <= keys


def test_gatv2_resumes_bit_for_bit(built, tmp_path, monkeypatch):
    from tests.test_resume_gpu import _args, _check_resume
    _check_resume(_args(1, model="gatv2", heads=2), tmp_path, monkeypatch, fused=False)


@pytest.mark.parametrize("n_parts", [1, 2, 3])
@pytest.mark.parametrize("heads,n_linear", [(1, 0), (2, 0), (2, 1)])
def test_gatv2_partition_logits_equal_the_whole_graph_evaluation(built, heads, n_linear, n_parts):
    """Each rank's logits after one training epoch == the whole-graph evaluation's rows of its nodes, within the bar
    the GAT cases of test_parallel_eval_gpu use."""
    from bns_gcn_b200 import train
    from bns_gcn_b200.data import make_graph, partition_graph
    from bns_gcn_b200.helper.utils import get_layer_size
    from tests.harness import make_args
    from tests.test_parallel_eval_gpu import TOL, _full_handle, _parallel, _whole_graph
    fg = make_graph("tiny", seed=5)
    parts = partition_graph(fg, n_parts, "random", seed=0)
    args = make_args(n_partitions=n_parts, sampling_rate=0.5, dropout=0.3, eval=True, model="gatv2", heads=heads,
                     n_linear=n_linear)
    res = _parallel(parts, args, DEV)
    sd = res[0][4]
    g, _ = _whole_graph(fg, n_parts, "random", DEV)
    a = argparse.Namespace(**vars(args))
    a.n_feat, a.n_class, a.n_train = fg.n_feat, fg.n_class, int(fg.train_mask.sum())
    net = train.create_model(get_layer_size(fg.n_feat, a.n_hidden, fg.n_class, a.n_layers), a)
    net.load_state_dict(sd, strict=True)
    net.to(DEV).eval()
    with torch.no_grad():
        full = net(_full_handle(g, DEV), g.feat.to(DEV)).cpu()
    assert torch.isfinite(full).all()
    for gid, logits, _, _, _ in res:
        assert _rel(logits, full[gid]) <= TOL, (heads, n_linear, n_parts)


@pytest.mark.parametrize("n_parts", [1, 2, 3])
@pytest.mark.parametrize("kw", [dict(heads=1), dict(heads=2), dict(heads=2, n_linear=1)],
                         ids=["1head", "2heads", "2heads-n-linear1"])
def test_gatv2_inductive_eval_parts_equal_the_whole_graph_evaluator(built, kw, n_parts):
    """``--parallel-eval --inductive``: after one training epoch, each rank's logits on its part of the val graph and
    of the test graph == the whole-graph ``Evaluator``'s rows of the same nodes, within the bar and with the checks
    test_parallel_eval_inductive_gpu applies to GAT."""
    from bns_gcn_b200.data import make_graph
    from tests.harness import make_args
    from tests.test_parallel_eval_inductive_gpu import _check, _parallel
    fg = make_graph("tiny", seed=5)
    args = make_args(n_partitions=n_parts, sampling_rate=0.5, dropout=0.3, eval=True, parallel_eval=True,
                     inductive=True, model="gatv2", **kw)
    _check(fg, args, _parallel(fg, args))
