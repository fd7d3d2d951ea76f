"""GAT's evaluation forward on the full graph: the one-pass attention kernel (``bns_gat_infer_f32``), the homogeneous
call ``GATConv(g, h)`` and the model's evaluation branch against the oracle and the reference's own output, and
``train.run`` with ``--eval`` for ``--model gat``."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TOL = 1e-4


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / b.norm().clamp(min=1e-30)).item()


def _graph(n_src, degrees, gen, sorted_row=None, el=None):
    """CSR by destination: row r has ``degrees[r]`` sources drawn uniformly (repeats allowed); row ``sorted_row`` takes
    its sources in increasing order of ``el[:, 0]``, so its running maximum grows at every block of 32."""
    idx = []
    for r, d in enumerate(degrees):
        s = torch.randint(0, n_src, (d,), generator=gen)
        if r == sorted_row:
            s = s[torch.argsort(el[s, 0], stable=True)]
        idx.append(s)
    indptr = torch.zeros(len(degrees) + 1, dtype=torch.int64)
    indptr[1:] = torch.cumsum(torch.tensor(degrees, dtype=torch.int64), 0)
    return indptr, torch.cat(idx).to(torch.int32)


def _reference(indptr, indices, ft, el, er, bias, H, Fo, slope):
    """Float64 restatement over explicit entries: e = leaky_relu(el_u + er_v), softmax over each row, weighted sum."""
    n = indptr.numel() - 1
    v = torch.repeat_interleave(torch.arange(n), indptr[1:] - indptr[:-1])
    u = indices.long()
    e = torch.nn.functional.leaky_relu(el.double()[u] + er.double()[v], slope)                     # [nnz, H]
    m = torch.full((n, H), float("-inf"), dtype=torch.float64).scatter_reduce(0, v.unsqueeze(1).expand(-1, H), e, "amax")
    ex = torch.exp(e - m[v])
    den = torch.zeros(n, H, dtype=torch.float64).index_add(0, v, ex)
    a = ex / den[v]
    rst = torch.zeros(n, H, Fo, dtype=torch.float64).index_add(0, v, a.unsqueeze(-1) * ft.double()[u])
    return rst + bias.double().view(1, H, Fo), e


CASES = [(H, Fo) for H in (1, 2, 4, 8) for Fo in (5, 16, 41, 64, 128, 256) if H * ((Fo + 3) // 4 * 4) <= 1024]


@pytest.mark.parametrize("H,Fo", CASES)
def test_gat_infer_kernel_matches_the_float64_restatement(built, H, Fo):
    """graph.gat_infer == softmax-weighted sums in float64.  Rows of degree 1, 31, 32, 33, 64 and several thousand
    (one of them ordered so that the running maximum grows at every block), scores up to ~120 (exp without the max
    subtraction overflows in float32), both LeakyReLU branches, zero pad columns, a bias; a row without entries gets
    the bias alone; two launches are bit-identical."""
    from bns_gcn_b200 import ops
    from bns_gcn_b200.graph import gat_infer, gat_padded_width
    dev = torch.device("cuda:0")
    gen = torch.Generator().manual_seed(1000 * H + Fo)
    Fp = gat_padded_width(Fo)
    n_src = 5000
    # multiples of 1/64 below 64 in magnitude: el + er is exact in float32, so only the kernel's own rounding counts
    el = torch.round((torch.rand(n_src, H, generator=gen) * 120 - 60) * 64) / 64
    degrees = [1, 31, 32, 33, 64, 4000, 0, 2500, 1] + torch.randint(1, 80, (200,), generator=gen).tolist()
    indptr, indices = _graph(n_src, degrees, gen, sorted_row=5, el=el)
    n = len(degrees)
    er = torch.round((torch.rand(n, H, generator=gen) * 120 - 60) * 64) / 64
    ft = torch.randn(n_src, H, Fo, generator=gen)
    bias = torch.randn(H, Fo, generator=gen)
    want, e = _reference(indptr, indices, ft, el, er, bias, H, Fo, 0.2)
    assert e.max().item() > 89.0 and (e < 0).any() and (e > 0).any()      # exp(89) overflows float32; both branches
    ftp = torch.nn.functional.pad(ft, (0, Fp - Fo)).reshape(n_src, H * Fp)
    bp = torch.nn.functional.pad(bias, (0, Fp - Fo)).reshape(H * Fp)
    a = ops.DeviceGraph.from_csr(indptr.to(dev), indices.to(dev), n_src)
    args = (a, ftp.to(dev), el.to(dev), er.to(dev), H, Fp, 0.2, bp.to(dev))
    out = gat_infer(*args)
    torch.cuda.synchronize()
    got = out.cpu().view(n, H, Fp)
    deg = torch.tensor(degrees)
    has = deg > 0
    assert _rel(got[has][..., :Fo], want[has]) <= 1e-5
    for r in (0, 1, 2, 3, 4, 5, 7):                          # each special row on its own
        assert _rel(got[r, :, :Fo], want[r]) <= 1e-5, r
    assert torch.equal(got[~has][..., :Fo], bias.expand(int((~has).sum()), H, Fo))
    assert torch.all(got[..., Fo:] == 0)                     # pad columns: zero ft, zero bias
    assert torch.equal(gat_infer(*args), out)                # deterministic


def test_gat_infer_rejects_bad_arguments(built):
    """The C entry point answers BNS_E_INVALID with a message; the wrapper checks shapes before launching."""
    from bns_gcn_b200 import ops
    from bns_gcn_b200._lib import BnsError, lib
    from bns_gcn_b200.graph import gat_infer
    dev = torch.device("cuda:0")
    indptr = torch.tensor([0, 1, 2], dtype=torch.int64, device=dev)
    a = ops.DeviceGraph.from_csr(indptr, torch.tensor([1, 0], dtype=torch.int32, device=dev), 2)
    ft = torch.zeros(2, 16, device=dev)
    el = torch.zeros(2, 2, device=dev)
    out = torch.empty(2, 16, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    for H, Fp in ((9, 4), (2, 6), (2, 1024), (0, 8)):
        rc = lib.bns_gat_infer_f32(a._h, ft.data_ptr(), 16, H, Fp, el.data_ptr(), el.data_ptr(), 0.2, None,
                                   out.data_ptr(), 16, st)
        assert rc == -1 and b"bns_gat_infer_f32" in lib.bns_last_error()
    rc = lib.bns_gat_infer_f32(a._h, ft.data_ptr() + 4, 16, 2, 8, el.data_ptr(), el.data_ptr(), 0.2, None,
                               out.data_ptr(), 16, st)
    assert rc == -1 and b"aligned" in lib.bns_last_error()
    rc = lib.bns_gat_infer_f32(None, ft.data_ptr(), 16, 2, 8, el.data_ptr(), el.data_ptr(), 0.2, None, out.data_ptr(), 16, st)
    assert rc == -1
    with pytest.raises(BnsError):
        gat_infer(a, ft[:, :12], el, el, 2, 8, 0.2)            # ft narrower than heads * Fp
    with pytest.raises(BnsError):
        gat_infer(a, ft, el, el[:1], 2, 8, 0.2)                 # er rows != graph rows
    with pytest.raises(BnsError):
        gat_infer(a, ft.cpu(), el, el, 2, 8, 0.2)               # not on the device


def _full_handle(fg, dev):
    from bns_gcn_b200 import ops
    from bns_gcn_b200.graph import FullGraphHandle
    a = ops.DeviceGraph.from_csr(fg.indptr.to(dev), fg.src.int().to(dev), fg.n_nodes)
    return FullGraphHandle(a, fg.in_degrees().to(dev), fg.out_degrees().to(dev))


@pytest.mark.parametrize("n_linear", [0, 1])
@pytest.mark.parametrize("heads", [1, 2])
@pytest.mark.parametrize("shape", ["tiny", "tiny-ml"])
def test_gat_eval_branch_full_graph(built, shape, heads, n_linear):
    """module/model.py:96-132 in evaluation: GATConv's homogeneous call on the whole graph, heads averaged, against the
    oracle's GATRef with identical initial weights."""
    import torch.nn.functional as F
    from bns_gcn_b200.data import make_graph
    from bns_gcn_b200.module.model import GAT
    from oracle import bns_oracle as O
    dev = torch.device("cuda:0")
    fg = make_graph(shape, seed=3)
    layer_size = [fg.n_feat, 16, 16, fg.n_class]
    torch.manual_seed(0)
    net = GAT(layer_size, F.relu, use_pp=True, heads=heads, dropout=0.5, norm="layer", n_linear=n_linear)
    torch.manual_seed(0)
    ref = O.build_model("gat", layer_size, True, 0.5, "layer", None, n_linear, heads=heads)
    for a, b in zip(net.parameters(), ref.parameters()):
        assert torch.equal(a, b)                                   # same init order as the reference
    net.to(dev).eval()
    ref.eval()
    g = _full_handle(fg, dev)
    with torch.no_grad():
        out = net(g, fg.feat.to(dev)).cpu()
        want = ref(O.EdgeList(fg.src, fg.dst(), fg.n_nodes, fg.n_nodes), fg.feat)
        # one layer on its own, before the head mean: the [n, heads, out_feats] of dgl.nn.GATConv
        last = net.layers[net.n_conv - 1]
        h = torch.randn(fg.n_nodes, last.fc.in_features, generator=torch.Generator().manual_seed(1))
        lo = last(g, h.to(dev)).cpu()
        lo_ref = ref.layers[net.n_conv - 1](O.EdgeList(fg.src, fg.dst(), fg.n_nodes, fg.n_nodes), h)
    assert out.shape == want.shape == (fg.n_nodes, fg.n_class)
    assert _rel(out, want) < TOL
    assert lo.shape == lo_ref.shape and _rel(lo, lo_ref) < TOL


def test_gat_conv_full_graph_call_is_evaluation_only(built):
    """Training on the full graph keeps raising; a node without in-edges raises as dgl.nn.GATConv does."""
    from bns_gcn_b200 import ops
    from bns_gcn_b200.graph import FullGraphHandle
    from bns_gcn_b200.module.gat import GATConv
    dev = torch.device("cuda:0")
    layer = GATConv(8, 5, 2).to(dev)
    indptr = torch.tensor([0, 1, 1], dtype=torch.int64, device=dev)         # node 1 has no in-edge
    a = ops.DeviceGraph.from_csr(indptr, torch.tensor([0], dtype=torch.int32, device=dev), 2)
    g = FullGraphHandle(a, torch.tensor([1, 0], device=dev), torch.tensor([1, 0], device=dev))
    h = torch.randn(2, 8, device=dev)
    with pytest.raises(NotImplementedError):
        layer(g, h)
    layer.eval()
    with pytest.raises(RuntimeError, match="0-in-degree"):
        layer(g, h)


def test_cuda_gat_evaluation_reproduces_the_reference_golden(built):
    """tests/golden/ref_gat_eval_p2.pt: after two training epochs tests/golden/make_golden_gat_eval.py ran the reference's
    evaluation forward (train.py:44-49) of its GAT model, 2 heads, closing width 5, on the whole graph.  Its trained
    parameters, loaded by name into the CUDA GAT, give the same logits."""
    import torch.nn.functional as F
    from bns_gcn_b200.data import make_graph
    from bns_gcn_b200.module.model import GAT
    dev = torch.device("cuda:0")
    gold = torch.load(os.path.join(GOLD, "ref_gat_eval_p2.pt"))
    cfg, r0 = gold["config"], gold["ranks"][0]
    fg = make_graph(cfg["shape"], seed=0)
    params = dict(zip(r0["param_names"], r0["params"]))
    layer_size = [params["layers.0.fc.weight"].shape[1]] + [cfg["n_hidden"]] * (cfg["n_layers"] - 1) + [fg.n_class]
    net = GAT(layer_size, F.relu, use_pp=True, heads=cfg["heads"], dropout=0.0, norm="layer")
    assert [n for n, _ in net.named_parameters()] == r0["param_names"]
    net.load_state_dict(params, strict=True)
    net.to(dev).eval()
    with torch.no_grad():
        out = net(_full_handle(fg, dev), fg.feat.to(dev))
    want = r0["eval_logits"]
    assert out.shape == want.shape == (fg.n_nodes, fg.n_class)
    assert _rel(out, want) <= TOL


@pytest.mark.parametrize("inductive", [False, True], ids=["transductive", "inductive"])
def test_gat_run_with_eval_writes_checkpoints_and_results(built, tmp_path, monkeypatch, inductive):
    """train.run --model gat --eval (train.py:427-456): every log_every epochs rank 0 saves a checkpoint, evaluates
    on the full graph and appends the result line; at the end the best model is saved and tested.  No warning."""
    import argparse
    import warnings
    from tests.harness import make_args
    from bns_gcn_b200 import train
    from bns_gcn_b200.data import make_graph, partition_graph
    from bns_gcn_b200.evaluate import checkpoint_path, load_checkpoint, result_file_name
    from bns_gcn_b200.helper.comm import run_threads
    monkeypatch.chdir(tmp_path)
    fg = make_graph("tiny", seed=0)
    parts = partition_graph(fg, 2, "random", seed=0, inductive=inductive)
    args = make_args(dataset="tiny", model="gat", heads=2, sampling_rate=0.5, n_hidden=16, n_partitions=2, n_epochs=4,
                     log_every=2, eval=True, inductive=inductive,
                     graph_name="tiny-2-random-vol-" + ("induc" if inductive else "trans"))

    def fn(comm, r):
        a = argparse.Namespace(**vars(args))
        p = parts[r]
        a.n_feat, a.n_class, a.n_train = p.meta["n_feat"], p.meta["n_class"], p.meta["n_train"]
        st, stats = train.run(p.graph, p.node_dict, p.gpb, a, "cuda:0", full_graph=fg)
        return st.model if r == 0 else None

    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        model = run_threads(2, fn, device="cuda:0")[0]
    assert not [w for w in caught if "--eval" in str(w.message)], [str(w.message) for w in caught]
    with open(result_file_name(args)) as f:
        lines = f.read().strip().splitlines()
    key = "Accuracy" if inductive else "Validation Accuracy"
    assert len(lines) == 2 and all(ln.startswith("Epoch") and key in ln for ln in lines), lines
    if not inductive:
        assert all("Test Accuracy" in ln for ln in lines)
    for e in (1, 3):
        assert os.path.exists(checkpoint_path(args, e))
    assert os.path.exists(checkpoint_path(args))
    load_checkpoint(model, checkpoint_path(args, 3))
    sd = torch.load(checkpoint_path(args, 3))
    assert list(sd.keys()) == [k for k, _ in model.named_parameters()]
    assert all(k.startswith(("layers.", "norm.")) for k in sd)     # the reference's parameter names
