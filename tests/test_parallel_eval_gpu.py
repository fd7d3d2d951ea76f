"""Partition-parallel evaluation (``--parallel-eval``): the column-block attention kernel (``bns_gat_infer_block_f32``)
against the one-pass kernel and float64; each rank's logits on its partition, with the whole halo exchanged layer by
layer, against the whole-graph evaluation; the reference's own evaluation logits; and ``train.run``'s driver."""
import argparse
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TOL = 1e-4


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / b.norm().clamp(min=1e-30)).item()


# ---- the kernel ---------------------------------------------------------------------------------------------------

def _q(t):
    """Multiples of 1/64: el + er is exact in float32, so only the kernels' own rounding counts."""
    return torch.round(t * 64) / 64


def _block_case(H, Fp, n_blocks, gen):
    """Rows over 1 + n_blocks column blocks (block 0 = the inner matrix).  Returns per-block CSR / ft / el and er.
    Special rows: 0 all entries in block 0; 1 empty in block 0, entries later; 2 no entries anywhere; 3 entries in the
    last block only; 4 ~4,000 entries over every block; 5 scores ~1.5 in block 0 and ~120 in the last block (the
    maximum jumps by ~118: expf of minus that underflows to 0, below even the denormals); 6 one score of exactly 0; the rest random."""
    nb = 1 + n_blocks
    n_cols = [int(x) for x in torch.randint(200, 1200, (nb,), generator=gen)]
    n_rows = 160
    er = _q(torch.rand(n_rows, H, generator=gen) * 40 - 20)
    er[5] = 0.0
    el = [_q(torch.rand(c, H, generator=gen) * 40 - 20) for c in n_cols]
    el[0][:50] = _q(1.0 + torch.rand(50, H, generator=gen))             # row 5's block-0 sources
    el[-1][:50] = _q(119.0 + torch.rand(50, H, generator=gen))          # row 5's last-block sources
    rows = [[None] * n_rows for _ in range(nb)]
    for r in range(n_rows):
        for b in range(nb):
            if r in (0,):
                d = int(torch.randint(1, 70, (1,), generator=gen)) if b == 0 else 0
            elif r == 1:
                d = 0 if b == 0 else int(torch.randint(0, 40, (1,), generator=gen)) + (b == nb - 1)
            elif r == 2:
                d = 0
            elif r == 3:
                d = 37 if b == nb - 1 else 0
            elif r == 4:
                d = 4000 // nb
            elif r == 5:
                d = 33 if b in (0, nb - 1) else 0
            else:
                d = int(torch.randint(0, 50, (1,), generator=gen))
            if r == 5:
                s = torch.randint(0, 50, (d,), generator=gen)
            else:
                s = torch.randint(0, n_cols[b], (d,), generator=gen)
            rows[b][r] = s
    # row 6: one entry whose score is exactly 0 (el_u = -er_v) in block 0
    u0 = int(rows[0][6][0]) if rows[0][6].numel() else None
    if u0 is None:
        rows[0][6] = torch.tensor([7])
        u0 = 7
    el[0][u0] = -er[6]
    blocks = []
    for b in range(nb):
        degs = torch.tensor([t.numel() for t in rows[b]], dtype=torch.int64)
        indptr = torch.zeros(n_rows + 1, dtype=torch.int64)
        indptr[1:] = torch.cumsum(degs, 0)
        idx = torch.cat(rows[b]).to(torch.int32)
        ft = torch.randn(n_cols[b], H * Fp, generator=gen)
        blocks.append((indptr, idx, ft, el[b]))
    return blocks, er


def _concat(blocks, n_rows):
    """The same rows as ONE matrix over the concatenated columns, each row's entries in block order."""
    off, per_row = 0, [[] for _ in range(n_rows)]
    for indptr, idx, ft, el in blocks:
        for r in range(n_rows):
            per_row[r].append(idx[indptr[r]:indptr[r + 1]].long() + off)
        off += ft.shape[0]
    degs = torch.tensor([sum(t.numel() for t in pr) for pr in per_row], dtype=torch.int64)
    indptr = torch.zeros(n_rows + 1, dtype=torch.int64)
    indptr[1:] = torch.cumsum(degs, 0)
    idx = torch.cat([torch.cat(pr) for pr in per_row]).to(torch.int32)
    return indptr, idx, torch.cat([b[2] for b in blocks]), torch.cat([b[3] for b in blocks])


def _reference64(indptr, idx, ft, el, er, bias, H, Fp, slope):
    n = indptr.numel() - 1
    v = torch.repeat_interleave(torch.arange(n), indptr[1:] - indptr[:-1])
    u = idx.long()
    e = torch.nn.functional.leaky_relu(el.double()[u] + er.double()[v], slope)
    m = torch.full((n, H), float("-inf"), dtype=torch.float64).scatter_reduce(0, v.unsqueeze(1).expand(-1, H), e, "amax")
    ex = torch.exp(e - m[v])
    den = torch.zeros(n, H, dtype=torch.float64).index_add(0, v, ex)
    a = ex / den[v]
    rst = torch.zeros(n, H, Fp, dtype=torch.float64).index_add(0, v, a.unsqueeze(-1) * ft.double().view(-1, H, Fp)[u])
    return rst + bias.double().view(1, H, Fp)


def _run_blocks(gblocks, er, H, Fp, bias, dev):
    from bns_gcn_b200.graph import gat_infer_block
    n = er.shape[0]
    m = torch.empty(n, H, device=dev)
    l = torch.empty(n, H, device=dev)
    acc = torch.empty(n, H * Fp, device=dev)
    for k, (a, ft, el) in enumerate(gblocks):
        gat_infer_block(a, ft, el, er, H, Fp, 0.2, m, l, acc, k == 0, k == len(gblocks) - 1, bias, acc)
    return acc


# NV = ceil(heads * Fp / 128) = 1, 2, 4, 8 for each head count
KERNEL_CASES = [(H, Fp) for H, fps in ((1, (64, 256, 512, 1024)), (3, (40, 80, 160, 340)), (8, (16, 32, 64, 128)))
                for Fp in fps]


@pytest.mark.parametrize("n_blocks", [1, 2, 5])
@pytest.mark.parametrize("H,Fp", KERNEL_CASES)
def test_gat_infer_block_matches_one_pass_and_float64(built, H, Fp, n_blocks):
    """The inner block plus 1, 2 or 5 peer blocks, state carried between launches == bns_gat_infer_f32 on the
    concatenated matrix (1e-6) and the float64 restatement (1e-5), on the whole and on each special row; rows without
    entries get the bias alone; two runs are bit-identical."""
    from bns_gcn_b200 import ops
    from bns_gcn_b200.graph import gat_infer
    dev = torch.device("cuda:0")
    gen = torch.Generator().manual_seed(97 * H + Fp + 1000 * n_blocks)
    blocks, er = _block_case(H, Fp, n_blocks, gen)
    n = er.shape[0]
    bias = torch.randn(H * Fp, generator=gen)
    gblocks = [(ops.DeviceGraph.from_csr(ip.to(dev), ix.to(dev), ft.shape[0]), ft.to(dev), el.to(dev))
               for ip, ix, ft, el in blocks]
    got = _run_blocks(gblocks, er.to(dev), H, Fp, bias.to(dev), dev)
    ip, ix, ft, el = _concat(blocks, n)
    one = gat_infer(ops.DeviceGraph.from_csr(ip.to(dev), ix.to(dev), ft.shape[0]), ft.to(dev), el.to(dev), er.to(dev),
                    H, Fp, 0.2, bias.to(dev))
    want = _reference64(ip, ix, ft, el, er, bias, H, Fp, 0.2).view(n, H * Fp)
    torch.cuda.synchronize()
    got, one = got.cpu(), one.cpu()
    has = (ip[1:] - ip[:-1]) > 0
    assert _rel(got[has], one[has]) <= 1e-6 and _rel(got[has], want[has]) <= 1e-5
    for r in (0, 1, 3, 4, 5, 6):
        assert has[r] and _rel(got[r], one[r]) <= 1e-6 and _rel(got[r], want[r]) <= 1e-5, r
    assert torch.equal(got[~has], bias.expand(int((~has).sum()), -1)) and not has[2]
    again = _run_blocks(gblocks, er.to(dev), H, Fp, bias.to(dev), dev).cpu()
    assert torch.equal(again, got)


def test_gat_infer_block_rejects_bad_arguments(built):
    """NULL state, a misaligned accumulator and bns_gat_infer_f32's limits: BNS_E_INVALID naming the entry point."""
    from bns_gcn_b200 import ops
    from bns_gcn_b200._lib import BnsError, lib
    from bns_gcn_b200.graph import gat_infer_block
    dev = torch.device("cuda:0")
    a = ops.DeviceGraph.from_csr(torch.tensor([0, 1, 2], dtype=torch.int64, device=dev),
                                 torch.tensor([1, 0], dtype=torch.int32, device=dev), 2)
    ft = torch.zeros(2, 20, device=dev)
    el = torch.zeros(2, 2, device=dev)
    m, l, acc = torch.zeros(2, 2, device=dev), torch.zeros(2, 2, device=dev), torch.zeros(2, 20, device=dev)
    st = torch.cuda.current_stream().cuda_stream

    def call(H=2, Fp=8, mp=m.data_ptr(), lp=l.data_ptr(), ap=acc.data_ptr(), ldacc=16):
        return lib.bns_gat_infer_block_f32(a._h, ft.data_ptr(), 16, H, Fp, el.data_ptr(), el.data_ptr(), 0.2, mp, lp,
                                           ap, ldacc, 1, 1, None, acc.data_ptr(), 16, st)
    for kw in (dict(mp=None), dict(lp=None), dict(ap=None), dict(ap=acc.data_ptr() + 4), dict(ldacc=18),
               dict(ldacc=20),                                             # rst is acc, at another stride
               dict(H=9, Fp=4), dict(H=2, Fp=6), dict(H=2, Fp=1024), dict(H=0, Fp=8)):
        assert call(**kw) == -1, kw
        assert b"bns_gat_infer_block_f32" in lib.bns_last_error(), kw
    assert call() == 0
    with pytest.raises(BnsError):
        gat_infer_block(a, ft[:, :12], el, el, 2, 8, 0.2, m, l, acc[:, :16], True, True, None, acc[:, :16])
    with pytest.raises(BnsError):
        gat_infer_block(a, None, None, el, 2, 8, 0.2, m, l, acc[:, :16], True, True, None, acc[:, :16])
    with pytest.raises(BnsError):
        gat_infer_block(a, ft[:, :16], el, el, 2, 8, 0.2, m, l, acc[:, :16], True, True)     # last without rst


# ---- the model on partitions ----------------------------------------------------------------------------------------

def _whole_graph(fg, n_parts, method, dev):
    """The relabelled graph partition_graph cut (ids line up through node_dict['_ID']), and new id -> original id."""
    from bns_gcn_b200.data.partition import assign_parts, relabel
    part = assign_parts(fg, n_parts, method, 0, "vol", None)
    g, _ = relabel(fg, part, n_parts, dev)
    return g, torch.argsort(part, stable=True)


def _full_handle(fg, dev):
    from bns_gcn_b200 import ops
    from bns_gcn_b200.graph import FullGraphHandle
    a = ops.DeviceGraph.from_csr(fg.indptr.to(dev), fg.src.int().to(dev), fg.n_nodes)
    return FullGraphHandle(a, fg.in_degrees().to(dev), fg.out_degrees().to(dev))


def _parallel(parts, args, dev, train_epochs=1, params=None):
    """Every rank: setup, ``train_epochs`` training epochs (or the given parameters), then the partition-parallel
    evaluation.  Returns per rank (global ids of its inner nodes, logits, val acc, test acc, state dict)."""
    from bns_gcn_b200 import train
    from bns_gcn_b200.evaluate import ParallelEvaluator, build_partition_eval_graph
    from bns_gcn_b200.helper.comm import run_threads

    def fn(comm, r):
        p = parts[r]
        a = argparse.Namespace(**vars(args))
        a.n_feat, a.n_class, a.n_train = p.meta["n_feat"], p.meta["n_class"], p.meta["n_train"]
        st = train.setup(p.graph, p.node_dict, p.gpb, a, dev)
        for e in range(train_epochs):
            train.train_epoch(st, e)
        if params is not None:
            st.model.load_state_dict(params, strict=True)
        eg = build_partition_eval_graph(st.part, p.node_dict, st.boundary, comm)
        ev = ParallelEvaluator(a, eg, st.feat, st.labels, p.node_dict["val_mask"].to(dev),
                               p.node_dict["test_mask"].to(dev), comm)
        logits = ev.logits(st.model)
        va, te = ev._acc(logits, ev.val_mask), ev._acc(logits, ev.test_mask)
        sd = {k: v.detach().cpu().clone() for k, v in st.model.state_dict().items()}
        return p.node_dict["_ID"][:p.graph.n_in].cpu(), logits.cpu(), va, te, sd
    return run_threads(len(parts), fn, device=str(dev))


def _accuracy_agrees(acc, full, labels, mask, tol):
    """The accuracies are equal, except that a node may flip when its top two whole-graph logits lie within ``tol``."""
    from bns_gcn_b200.evaluate import calc_acc
    want = calc_acc(full[mask], labels[mask])
    if acc == want:
        return True
    if labels.dim() > 1:                      # multi-label: an entry may flip when its logit lies within tol of 0
        return bool((full[mask].abs() <= tol * full.abs().max()).any())
    top2 = full[mask].topk(2, dim=1).values
    close = int(((top2[:, 0] - top2[:, 1]) <= tol * full.abs().max()).sum())
    return abs(acc - want) <= close / max(int(mask.sum()), 1) + 1e-12


MODELS = {
    "graphsage": dict(model="graphsage"),
    "graphsage-linear": dict(model="graphsage", n_linear=1),
    "gcn": dict(model="gcn"),
    # SyncBatchNorm normalises by the whole training set's size: every node a training node, as under --inductive;
    # validation and test nodes are then drawn among them (evaluated nodes may be training nodes)
    "gcn-batchnorm": dict(model="gcn", norm="batch", graph=dict(train=1.0), redraw_masks=True),
    # multi-label (micro-F1 from the summed TP / FP / FN counts)
    "graphsage-multilabel": dict(model="graphsage", shape="tiny-ml", multilabel=True),
    "gat-1head": dict(model="gat", heads=1),
    "gat-2heads": dict(model="gat", heads=2),
}


@pytest.mark.parametrize("method", ["random", "metis"])
@pytest.mark.parametrize("n_parts", [1, 2, 3, 4])
@pytest.mark.parametrize("case", sorted(MODELS))
def test_partition_logits_equal_the_whole_graph_evaluation(built, case, n_parts, method):
    """Each rank's logits == the whole-graph evaluation's rows of its nodes (1e-4), after one training epoch, on
    ``tiny`` (closing width 5); the summed accuracies equal the whole graph's up to ties within the tolerance."""
    from bns_gcn_b200 import train
    from bns_gcn_b200.data import make_graph, partition_graph
    from tests.harness import make_args
    dev = torch.device("cuda:0")
    kw = dict(MODELS[case])
    fg = make_graph(kw.pop("shape", "tiny"), seed=5, **kw.pop("graph", {}))
    if kw.pop("redraw_masks", False):
        u = torch.rand(fg.n_nodes, generator=torch.Generator().manual_seed(11))
        fg.val_mask, fg.test_mask = u < 0.3, u >= 0.3
    parts = partition_graph(fg, n_parts, method, seed=0)
    args = make_args(n_partitions=n_parts, sampling_rate=0.5, dropout=0.3, eval=True, **kw)
    res = _parallel(parts, args, dev)
    sd = res[0][4]
    for r in range(1, n_parts):
        assert all(torch.equal(sd[k], res[r][4][k]) for k in sd)          # the weights are replicated
    g, _ = _whole_graph(fg, n_parts, method, dev)
    a = argparse.Namespace(**vars(args))
    a.n_feat, a.n_class, a.n_train = fg.n_feat, fg.n_class, int(fg.train_mask.sum())
    from bns_gcn_b200.helper.utils import get_layer_size
    net = train.create_model(get_layer_size(fg.n_feat, a.n_hidden, fg.n_class, a.n_layers), a)
    net.load_state_dict(sd, strict=True)
    net.to(dev).eval()
    with torch.no_grad():
        full = net(_full_handle(g, dev), g.feat.to(dev)).cpu()
    assert torch.isfinite(full).all()
    for gid, logits, _, _, _ in res:
        assert logits.shape == (gid.numel(), fg.n_class)
        assert _rel(logits, full[gid]) <= TOL, (case, n_parts, method)
    for k, mask in ((2, g.val_mask), (3, g.test_mask)):
        assert len({r[k] for r in res}) == 1                               # every rank reports the same accuracy
        assert mask.any()
        assert _accuracy_agrees(res[0][k], full, g.label, mask, TOL), (res[0][k], k)


@pytest.mark.parametrize("n_parts", [2, 4])
@pytest.mark.parametrize("model", ["graphsage", "gcn", "gat"])
def test_partition_evaluation_reproduces_the_reference_golden(built, model, n_parts):
    """tests/golden/ref_<model>_eval_p2.pt: the reference's whole-graph evaluation logits of its trained model.  Its
    parameters, loaded by name, give the same logits through the partition-parallel path at 2 and 4 partitions."""
    from bns_gcn_b200.data import make_graph, partition_graph
    from tests.harness import make_args
    dev = torch.device("cuda:0")
    gold = torch.load(os.path.join(GOLD, f"ref_{model}_eval_p2.pt"))
    cfg, r0 = gold["config"], gold["ranks"][0]
    fg = make_graph(cfg["shape"], seed=0)
    params = dict(zip(r0["param_names"], r0["params"]))
    parts = partition_graph(fg, n_parts, "random", seed=0)
    args = make_args(model=model, n_layers=cfg["n_layers"], n_hidden=cfg["n_hidden"], heads=cfg.get("heads", 1),
                     n_partitions=n_parts, eval=True)
    res = _parallel(parts, args, dev, train_epochs=0, params=params)
    _, orig = _whole_graph(fg, n_parts, "random", dev)
    want = r0["eval_logits"]
    got = torch.empty_like(want)
    for gid, logits, _, _, _ in res:
        got[orig[gid]] = logits
    assert _rel(got, want) <= TOL


# ---- the driver -----------------------------------------------------------------------------------------------------

def _run_driver(tmp_path, monkeypatch, model, inductive, n_parts=2):
    from bns_gcn_b200 import train
    from bns_gcn_b200.data import make_graph, partition_graph
    from bns_gcn_b200.helper.comm import run_threads
    from tests.harness import make_args
    monkeypatch.chdir(tmp_path)
    fg = make_graph("tiny", seed=0)
    parts = partition_graph(fg, n_parts, "random", seed=0, inductive=inductive)
    args = make_args(dataset="tiny", model=model, heads=2, sampling_rate=0.5, n_hidden=16, n_partitions=n_parts,
                     n_epochs=4, log_every=2, eval=True, parallel_eval=True, inductive=inductive,
                     graph_name="tiny-2-random-vol-" + ("induc" if inductive else "trans"))

    def no_whole_graph(*a, **k):
        raise AssertionError("the whole graph must not be built under --parallel-eval")
    monkeypatch.setattr("bns_gcn_b200.data.make_graph", no_whole_graph)

    def fn(comm, r):
        a = argparse.Namespace(**vars(args))
        p = parts[r]
        a.n_feat, a.n_class, a.n_train = p.meta["n_feat"], p.meta["n_class"], p.meta["n_train"]
        st, _ = train.run(p.graph, p.node_dict, p.gpb, a, "cuda:0")
        return st.model
    return args, run_threads(n_parts, fn, device="cuda:0")


@pytest.mark.parametrize("model", ["gat", "graphsage"])
def test_run_with_parallel_eval_writes_checkpoints_and_results(built, tmp_path, monkeypatch, capsys, model):
    """train.run --eval --parallel-eval at 2 partitions: the checkpoints, result lines and final checkpoint of the
    whole-graph evaluation, without the whole graph (make_graph raises); every rank ran the evaluation."""
    from bns_gcn_b200.evaluate import checkpoint_path, load_checkpoint, result_file_name
    args, models = _run_driver(tmp_path, monkeypatch, model, False)
    with open(result_file_name(args)) as f:
        lines = f.read().strip().splitlines()
    assert len(lines) == 2, lines
    assert all(ln.startswith("Epoch") and "Validation Accuracy" in ln and "Test Accuracy" in ln for ln in lines), lines
    for e in (1, 3):
        assert os.path.exists(checkpoint_path(args, e))
    assert os.path.exists(checkpoint_path(args))
    load_checkpoint(models[0], checkpoint_path(args, 3))
    sd = torch.load(checkpoint_path(args, 3))
    assert list(sd.keys()) == [k for k, _ in models[0].named_parameters()]
    assert all(k.startswith(("layers.", "norm.")) for k in sd)
    out = capsys.readouterr().out
    assert out.count("Test Result | Accuracy") == 1 and out.count("model saved") == 1


def test_run_with_parallel_eval_refuses_inductive(built, tmp_path, monkeypatch):
    with pytest.raises(ValueError, match="--parallel-eval"):
        _run_driver(tmp_path, monkeypatch, "graphsage", True)


# ---- the bench shape ------------------------------------------------------------------------------------------------

def test_reddit_shape_partition_logits_equal_the_whole_graph(built):
    """The Reddit shape at 4 in-process ranks: 3-layer GraphSAGE, hidden 256, --use-pp, after one training epoch at
    the bench configuration (sampling rate 0.1) -- each rank's logits within 1e-4 of the whole-graph evaluation."""
    free, _ = torch.cuda.mem_get_info(0)
    if free / 2 ** 30 < 40:
        pytest.skip("needs ~40 GB of free device memory (full-size graph + 4 in-process ranks)")
    from bns_gcn_b200 import train
    from bns_gcn_b200.data import make_graph, partition_graph
    from bns_gcn_b200.helper.utils import get_layer_size
    from tests.harness import make_args
    dev = torch.device("cuda:0")
    fg = make_graph("reddit", seed=0)
    parts = partition_graph(fg, 4, "random", seed=0, device=dev)
    args = make_args(dataset="reddit", model="graphsage", n_layers=3, n_hidden=256, sampling_rate=0.1, dropout=0.5,
                     n_partitions=4, eval=True, backend="p2p")
    res = _parallel(parts, args, dev)
    g, _ = _whole_graph(fg, 4, "random", dev)
    a = argparse.Namespace(**vars(args))
    a.n_feat, a.n_class, a.n_train = fg.n_feat, fg.n_class, int(fg.train_mask.sum())
    net = train.create_model(get_layer_size(fg.n_feat, 256, fg.n_class, 3), a)
    net.load_state_dict(res[0][4], strict=True)
    net.to(dev).eval()
    with torch.no_grad():
        full = net(_full_handle(g, dev), g.feat.to(dev)).cpu()
    for gid, logits, _, _, _ in res:
        assert _rel(logits, full[gid]) <= TOL
