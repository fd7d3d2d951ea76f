"""SyncBatchNorm (``--norm batch``): ``bns_bn_colsums_f32`` (modes 0 and 1), ``bns_bn_apply_f32`` and ``bns_bn_bwd_f32``
against float64 restatements of the reference's conventions (oracle/bns_oracle.py ``_SyncBNFunc``): the one-pass
variance ``(S2 - mean S1) / n``, the running statistics moved by ``momentum`` with that biased variance, and
``dx = (w / n) rstd (n dy - d bias - x_hat d weight)``.

Per-element bounds, as in tests/test_layernorm_dropout_gpu.py, from the magnitudes that enter each element, with the
conditioning factor ``kappa = mean(x^2) / (var + eps)`` that the one-pass variance passes on to rstd.  The inputs keep
|mean| / std <= 3, so kappa stays below 10: this is the reference's formula, and the tests do not argue with it.
Widths 4 .. 1024 (44: 256 threads do not divide into 11 float4 columns), rows from 0 to the benchmark's 232,965,
around the 4 blocks per SM of the column sums, strided operands, one batch split over three ranks (one of them
empty), the ``SyncBatchNorm`` module at three in-process ranks over three steps, the running statistics of a
``--norm batch`` training run against the oracle's, and argument rejection."""
import argparse

import pytest
import torch

from tests import layer_reference as R

pytestmark = pytest.mark.gpu

EPS, MOMENTUM = 1e-5, 0.1
WIDTHS = (4, 44, 128, 256, 1024)
ROWS = ("0", "1", "5", "4sm-1", "4sm+1", "bench")


def _dev():
    return torch.device("cuda:0")


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _n_rows(tag):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return {"0": 0, "1": 1, "5": 5, "4sm-1": 4 * sms - 1, "4sm+1": 4 * sms + 1, "bench": 232_965}[tag]


def _strided(n, F, pad, fill=float("nan")):
    return torch.full((n, F + pad), fill, device=_dev())[:, :F]


# ---- launches ---------------------------------------------------------------------------------------------------------
def colsums(mode, a, x=None, mean=None, rstd=None):
    from bns_gcn_b200._lib import check, lib
    n, F = a.shape
    out = torch.full((2 * F,), float("nan"), device=_dev())
    ws = torch.empty(lib.bns_bn_workspace_bytes(F), dtype=torch.uint8, device=_dev())
    check(lib.bns_bn_colsums_f32(mode, a.data_ptr(), a.stride(0), None if x is None else x.data_ptr(),
                                 0 if x is None else x.stride(0), n, F, None if mean is None else mean.data_ptr(),
                                 None if rstd is None else rstd.data_ptr(), out.data_ptr(), ws.data_ptr(), ws.numel(),
                                 _stream()), "bns_bn_colsums_f32")
    return out


def apply(x, sums, whole, w, b, rm, rv, y):
    from bns_gcn_b200._lib import check, lib
    n, F = x.shape
    mean, rstd = torch.full((F,), float("nan"), device=_dev()), torch.full((F,), float("nan"), device=_dev())
    check(lib.bns_bn_apply_f32(x.data_ptr(), x.stride(0), n, F, sums.data_ptr(), float(whole), EPS, w.data_ptr(),
                               b.data_ptr(), MOMENTUM, None if rm is None else rm.data_ptr(),
                               None if rv is None else rv.data_ptr(), y.data_ptr(), y.stride(0), mean.data_ptr(),
                               rstd.data_ptr(), _stream()), "bns_bn_apply_f32")
    return mean, rstd


def bwd(dy, x, mean, rstd, w, sums, whole, dx):
    from bns_gcn_b200._lib import check, lib
    n, F = x.shape
    check(lib.bns_bn_bwd_f32(dy.data_ptr(), dy.stride(0), x.data_ptr(), x.stride(0), n, F, mean.data_ptr(),
                             rstd.data_ptr(), w.data_ptr(), sums.data_ptr(), float(whole), dx.data_ptr(), dx.stride(0),
                             _stream()), "bns_bn_bwd_f32")


# ---- float64 reference ------------------------------------------------------------------------------------------------
def reference(x, dy, w, b, rm, rv, n=None):
    """Float64 batch norm of the reference over the rows of ``x`` (``n`` = whole_size, default the row count): values
    and bounds of the sums, the statistics, y, the running statistics after one step, d bias / d weight and dx."""
    xd, dyd, wd, bd = x.double(), dy.double(), w.double(), b.double()
    n = xd.shape[0] if n is None else n
    s1, s2 = xd.sum(0), (xd * xd).sum(0)
    a1, a2 = xd.abs().sum(0), (xd * xd).sum(0)
    mu = s1 / n
    var = (s2 - mu * s1) / n
    rstd = 1.0 / torch.sqrt(var + EPS)
    m1 = a1 / n
    kappa = (a2 / n) / (var + EPS)                      # how much the one-pass variance amplifies rounding
    xh = (xd - mu) * rstd
    a = xh.abs() * (1 + kappa) + rstd * m1              # the scale of x_hat's own rounding
    out = {"sums": (torch.cat([s1, s2]), torch.cat([a1, a2])),
           "mean": (mu, m1), "rstd": (rstd, rstd * kappa),
           "y": (xh * wd + bd, wd.abs() * a + bd.abs()),
           "running_mean": (rm.double() * (1 - MOMENTUM) + mu * MOMENTUM, rm.double().abs() * (1 - MOMENTUM) + m1 * MOMENTUM),
           "running_var": (rv.double() * (1 - MOMENTUM) + var * MOMENTUM,
                           rv.double().abs() * (1 - MOMENTUM) + (a2 / n + mu.abs() * m1) * MOMENTUM)}
    d1, d2 = dyd.sum(0), (dyd * xh).sum(0)
    ad = dyd.abs()
    out["dsums"] = (torch.cat([d1, d2]), torch.cat([ad.sum(0), (ad * a).sum(0)]))
    out["dx"] = ((wd / n) * rstd * (n * dyd - d1 - xh * d2),
                 wd.abs() * rstd * (1 + kappa) * (ad + ad.sum(0) / n + xh.abs() * (ad * a).sum(0) / n
                                                  + a * (ad * xh.abs()).sum(0) / n))
    return out


def _inputs(n, F, seed):
    dev = _dev()
    g = torch.Generator(device=dev).manual_seed(seed)
    col_scale = 10.0 ** (torch.rand(F, generator=g, device=dev) * 4 - 2)
    col_mean = (torch.rand(F, generator=g, device=dev) * 6 - 3) * col_scale         # |mean| / std <= 3
    x = torch.randn(n, F, generator=g, device=dev) * col_scale + col_mean
    dy = torch.randn(n, F, generator=g, device=dev)
    w = torch.randn(F, generator=g, device=dev)
    b = torch.randn(F, generator=g, device=dev) * 0.3
    rm = torch.randn(F, generator=g, device=dev)
    rv = torch.rand(F, generator=g, device=dev) + 0.5
    return x, dy, w, b, rm, rv


def _run_split(x, dy, w, b, rm, rv, sizes):
    """One batch over ``len(sizes)`` ranks: mode-0 sums per slice, added; apply per slice with whole_size = the total;
    the same for the backward.  Operands strided, outputs NaN-filled.  Every rank moves its own running statistics."""
    n, F = x.shape
    bounds = [0]
    for s in sizes:
        bounds.append(bounds[-1] + s)
    xs, dys, ys, dxs = [], [], [], []
    for r0, r1 in zip(bounds[:-1], bounds[1:]):
        xi, dyi = _strided(r1 - r0, F, 4, 0.0), _strided(r1 - r0, F, 8, 0.0)
        xi.copy_(x[r0:r1])
        dyi.copy_(dy[r0:r1])
        xs.append(xi)
        dys.append(dyi)
        ys.append(_strided(r1 - r0, F, 4))
        dxs.append(_strided(r1 - r0, F, 4))
    part = [colsums(0, xi) for xi in xs]
    for p_, xi in zip(part, xs):
        if xi.shape[0] == 0:
            assert bool((p_ == 0).all()), "colsums of 0 rows must write zeros"
    sums = torch.stack(part).sum(0)
    rms, rvs = [rm.clone() for _ in sizes], [rv.clone() for _ in sizes]
    stats = [apply(xi, sums, n, w, b, rmi, rvi, yi) for xi, rmi, rvi, yi in zip(xs, rms, rvs, ys)]
    dpart = [colsums(1, dyi, xi, mu, rs) for dyi, xi, (mu, rs) in zip(dys, xs, stats)]
    dsums = torch.stack(dpart).sum(0)
    for dyi, xi, (mu, rs), dxi in zip(dys, xs, stats, dxs):
        bwd(dyi, xi, mu, rs, w, dsums, n, dxi)
    torch.cuda.synchronize()
    for t in ys + dxs:
        full = t.as_strided((t.shape[0], t.stride(0)), (t.stride(0), 1))
        assert bool(torch.isfinite(full[:, :F]).all()) and bool(torch.isnan(full[:, F:]).all())
    return {"sums": sums, "mean": stats[0][0], "rstd": stats[0][1], "y": torch.cat(ys), "dsums": dsums,
            "dx": torch.cat(dxs), "rms": rms, "rvs": rvs, "stats": stats}


def _check(label, got, ref):
    worst = {}
    for k in ("sums", "mean", "rstd", "y", "dsums", "dx"):
        worst[k] = R.assert_close(f"{label} {k}", got[k], *ref[k])
    for i, (rmi, rvi) in enumerate(zip(got["rms"], got["rvs"])):
        worst["running_mean"] = R.assert_close(f"{label} rank {i} running_mean", rmi, *ref["running_mean"])
        worst["running_var"] = R.assert_close(f"{label} rank {i} running_var", rvi, *ref["running_var"])
    for mu, rs in got["stats"][1:]:
        assert torch.equal(mu, got["mean"]) and torch.equal(rs, got["rstd"]), "ranks disagree on the statistics"
    return worst


@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("F", WIDTHS)
def test_sync_bn_kernels_against_float64(built, F, rows):
    """One rank: both column-sum modes, apply with running statistics, backward.  0 rows: zero sums, and apply still
    moves the running statistics (from the sums the other ranks contributed)."""
    n = _n_rows(rows)
    x, dy, w, b, rm, rv = _inputs(max(n, 3), F, seed=F * 13 + n)
    if n == 0:
        empty = _strided(0, F, 4)
        s = colsums(0, empty)
        torch.cuda.synchronize()
        assert bool((s == 0).all())
        other = colsums(0, x)                                      # what the other ranks contributed
        rm1, rv1 = rm.clone(), rv.clone()
        mu, rs = apply(empty, other, x.shape[0], w, b, rm1, rv1, _strided(0, F, 4))
        bwd(empty, empty, mu, rs, w, colsums(1, dy, x, mu, rs), x.shape[0], _strided(0, F, 4))
        ref = reference(x, dy, w, b, rm, rv)
        R.assert_close(f"F={F} n=0 running_mean", rm1, *ref["running_mean"])
        R.assert_close(f"F={F} n=0 running_var", rv1, *ref["running_var"])
        R.assert_close(f"F={F} n=0 mean", mu, *ref["mean"])
        return
    if n == 1:
        # one row has no spread (var = 0, |mean| / std infinite), outside what the one-pass variance can serve: it
        # runs as one rank's slice of a 1,000-row batch
        x, dy, w, b, rm, rv = _inputs(1000, F, seed=F * 13 + n)
        got = _run_split(x, dy, w, b, rm, rv, [1, 999])
        _check(f"F={F} n=1 of 1000", got, reference(x, dy, w, b, rm, rv))
        return
    x, dy = x[:n], dy[:n]
    got = _run_split(x, dy, w, b, rm, rv, [n])
    _check(f"F={F} n={n}", got, reference(x, dy, w, b, rm, rv))
    # apply without running statistics leaves everything else as it was
    y2 = torch.empty(n, F, device=_dev())
    mu2, rs2 = apply(x.contiguous(), got["sums"], n, w, b, None, None, y2)
    assert torch.equal(mu2, got["mean"]) and torch.equal(rs2, got["rstd"]) and torch.equal(y2, got["y"])


@pytest.mark.parametrize("F", [44, 256])
def test_sync_bn_across_ranks_equals_one_batch(built, F):
    """Three unequal slices, one of them empty: summed mode-0 / mode-1 sums, apply and backward per slice with
    whole_size = the total equal one float64 batch norm over the whole batch."""
    n = 3001
    x, dy, w, b, rm, rv = _inputs(n, F, seed=F)
    got = _run_split(x, dy, w, b, rm, rv, [1900, 0, 1101])
    _check(f"F={F} split 1900/0/1101", got, reference(x, dy, w, b, rm, rv))


def test_sync_bn_module_three_ranks(built):
    """module.sync_bn.SyncBatchNorm at three in-process ranks (700 / 5 / 1300 rows, width 256), three training steps
    with a plain SGD step on weight / bias in between: y, dx, d weight, d bias, the running statistics and the
    evaluation-mode output on them, against float64 after every step."""
    from bns_gcn_b200.helper.comm import run_threads
    from bns_gcn_b200.module.sync_bn import SyncBatchNorm
    F, sizes, steps, lr = 256, (700, 5, 1300), 3, 0.05
    total = sum(sizes)
    data = [_inputs(total, F, seed=100 + s)[:2] for s in range(steps)]
    lo = [sum(sizes[:r]) for r in range(len(sizes))]
    w0, b0 = _inputs(4, F, seed=7)[2:4]

    def fn(comm, r):
        bn = SyncBatchNorm(F, total).to(_dev())
        with torch.no_grad():
            bn.weight.copy_(w0)
            bn.bias.copy_(b0)
        rec = []
        for s in range(steps):
            x = data[s][0][lo[r]:lo[r] + sizes[r]].clone().requires_grad_(True)
            dy = data[s][1][lo[r]:lo[r] + sizes[r]]
            w_used, b_used = bn.weight.detach().clone(), bn.bias.detach().clone()
            bn.train()
            y = bn(x)
            y.backward(dy)
            bn.eval()
            with torch.no_grad():
                y_eval = bn(x.detach())
            rec.append({k: v.detach().clone() for k, v in dict(
                w=w_used, b=b_used, y=y, dx=x.grad, dw=bn.weight.grad, db=bn.bias.grad, rm=bn.running_mean,
                rv=bn.running_var, y_eval=y_eval).items()})
            with torch.no_grad():
                bn.weight -= lr * bn.weight.grad / total
                bn.bias -= lr * bn.bias.grad / total
            bn.weight.grad = bn.bias.grad = None
        return rec
    torch.cuda.synchronize()
    out = run_threads(len(sizes), fn, device="cuda:0")
    rm, rv = torch.zeros(F, device=_dev()), torch.ones(F, device=_dev())
    for s in range(steps):
        w, b = out[0][s]["w"], out[0][s]["b"]
        for r in range(len(sizes)):
            assert torch.equal(out[r][s]["w"], w) and torch.equal(out[r][s]["b"], b)
            assert torch.equal(out[r][s]["rm"], out[0][s]["rm"]) and torch.equal(out[r][s]["rv"], out[0][s]["rv"])
        x, dy = data[s]
        # each step starts from the module's own float32 weights and running statistics of the step before
        ref = reference(x, dy, w, b, rm, rv)
        rm_ref, brm = ref["running_mean"]
        rv_ref, brv = ref["running_var"]
        scale = w.double() / torch.sqrt(rv_ref + EPS)
        for r in range(len(sizes)):
            o, sl = out[r][s], slice(lo[r], lo[r] + sizes[r])
            lab = f"step {s} rank {r}"
            R.assert_close(f"{lab} y", o["y"], ref["y"][0][sl], ref["y"][1][sl])
            R.assert_close(f"{lab} dx", o["dx"], ref["dx"][0][sl], ref["dx"][1][sl])
            R.assert_close(f"{lab} d bias", o["db"], ref["dsums"][0][:F], ref["dsums"][1][:F])
            R.assert_close(f"{lab} d weight", o["dw"], ref["dsums"][0][F:], ref["dsums"][1][F:])
            R.assert_close(f"{lab} running_mean", o["rm"], rm_ref, brm)
            R.assert_close(f"{lab} running_var", o["rv"], rv_ref, brv)
            xs = x[sl].double()
            want = (xs - rm_ref) * scale + b.double()
            bound = (xs.abs() + rm_ref.abs() + brm) * scale.abs() * (1 + brv / rv_ref) + b.double().abs()
            R.assert_close(f"{lab} eval y", o["y_eval"], want, bound)
        rm, rv = out[0][s]["rm"], out[0][s]["rv"]


def _run_product_bn(parts, args, device, n_epochs):
    """``tests.harness.run_product``, recording per epoch the biases in front of each batch norm and, at the end, the
    running statistics."""
    from bns_gcn_b200 import train
    from bns_gcn_b200.helper.comm import run_threads

    def fn(comm, r):
        p = parts[r]
        a = argparse.Namespace(**vars(args))
        a.n_feat, a.n_class, a.n_train = p.meta["n_feat"], p.meta["n_class"], p.meta["n_train"]
        st = train.setup(p.graph, p.node_dict, p.gpb, a, device)
        sel_log, biases = [], []
        for e in range(n_epochs):
            biases.append(_pre_norm_biases(st.model))
            train.train_epoch(st, e)
            sel_log.append([None if s is None else s.cpu().clone() for s in st.selected])
        torch.cuda.synchronize()
        return {"selected": sel_log, "biases": biases, "running": _running(st.model)}
    return run_threads(len(parts), fn, device=device)


def _run_oracle_bn(parts, args, n_epochs, selected_per_epoch):
    from oracle import bns_oracle as O

    def fn(comm, r):
        p = parts[r]
        rk = O.OracleRank(O.RankInput.from_partition(p), comm, model=args.model, n_layers=args.n_layers,
                          n_hidden=args.n_hidden, sampling_rate=args.sampling_rate, use_pp=args.use_pp,
                          dropout=args.dropout, norm=args.norm, lr=args.lr, weight_decay=args.weight_decay,
                          seed=args.seed, n_linear=args.n_linear)
        biases = []
        for e in range(n_epochs):
            biases.append(_pre_norm_biases(rk.net))
            rk.epoch(selected=selected_per_epoch[e][r])
        return {"biases": biases, "running": _running(rk.net)}
    return O.run_threads(len(parts), fn)


def _pre_norm_biases(net):
    """The summed biases of the layer in front of each norm (parameters 1 | 3 + 5 of the 3-layer GraphSAGE)."""
    ps = [q.detach().double().cpu() for q in net.parameters()]
    return [ps[1], ps[3] + ps[5]]


def _running(net):
    return [(m.running_mean.detach().double().cpu(), m.running_var.detach().double().cpu()) for m in net.norm]


def test_running_statistics_match_the_oracle(built):
    """The ``sync-bn`` parity configuration (tiny shape, 3 partitions, sampling 0.5, every node a training node),
    3 epochs: running_var, and running_mean less the momentum-weighted history of the bias in front of the norm, equal
    the oracle's ``SyncBNRef`` buffers within 1e-5.  (That bias has a true gradient of 0 -- the normalisation removes
    any shift -- so each implementation's Adam walks it on its own rounding noise; running_mean carries it along.)"""
    from bns_gcn_b200.data import make_graph, partition_graph
    from tests.harness import make_args
    n_parts, n_epochs = 3, 3
    fg = make_graph("tiny", seed=0, train=1.0)
    parts = partition_graph(fg, n_parts, "random", seed=0)
    args = make_args(dataset="tiny", sampling_rate=0.5, n_partitions=n_parts, norm="batch")
    prod = _run_product_bn(parts, args, "cuda:0", n_epochs)
    selected = [[prod[r]["selected"][e] for r in range(n_parts)] for e in range(n_epochs)]
    orc = _run_oracle_bn(parts, args, n_epochs, selected)
    for r in range(n_parts):
        for i in range(2):
            rel = {}
            for name, res in (("prod", prod[r]), ("oracle", orc[r])):
                shift = sum(MOMENTUM * (1 - MOMENTUM) ** (n_epochs - 1 - e) * res["biases"][e][i] for e in range(n_epochs))
                rel[name] = (res["running"][i][0] - shift, res["running"][i][1])
            for k, name in enumerate(("running_mean - bias history", "running_var")):
                a, b = rel["prod"][k], rel["oracle"][k]
                err = ((a - b).norm() / b.norm()).item()
                print(f"[running] rank {r} norm {i} {name}: {err:.3g}")
                assert err < 1e-5, (r, i, name, err)


def test_sync_bn_entry_points_reject_bad_arguments(built):
    """F % 4 != 0, F > 1024, only one running statistic, an unaligned matrix: BNS_E_INVALID naming the entry point; a
    short workspace: BNS_E_WORKSPACE."""
    from bns_gcn_b200._lib import lib
    dev = _dev()
    LD, n = 1040, 3
    x, dy, y, dx = (torch.zeros(n, LD, device=dev) for _ in range(4))
    sums, w, b, rm, rv, mean, rstd = (torch.zeros(2 * LD, device=dev) for _ in range(7))
    ws = torch.empty(lib.bns_bn_workspace_bytes(1024), dtype=torch.uint8, device=dev)
    st = _stream()

    def cs(F=256, xo=0, wsb=None):
        return lib.bns_bn_colsums_f32(0, x.data_ptr() + xo, LD, None, 0, n, F, None, None, sums.data_ptr(), ws.data_ptr(),
                                      ws.numel() if wsb is None else wsb, st)

    def ap(F=256, xo=0, one_stat=False):
        return lib.bns_bn_apply_f32(x.data_ptr() + xo, LD, n, F, sums.data_ptr(), float(n), EPS, w.data_ptr(),
                                    b.data_ptr(), MOMENTUM, rm.data_ptr(), None if one_stat else rv.data_ptr(),
                                    y.data_ptr(), LD, mean.data_ptr(), rstd.data_ptr(), st)

    def bw(F=256, xo=0):
        return lib.bns_bn_bwd_f32(dy.data_ptr(), LD, x.data_ptr() + xo, LD, n, F, mean.data_ptr(), rstd.data_ptr(),
                                  w.data_ptr(), sums.data_ptr(), float(n), dx.data_ptr(), LD, st)

    names = {cs: b"bns_bn_colsums_f32", ap: b"bns_bn_apply_f32", bw: b"bns_bn_bwd_f32"}
    bad = {cs: [dict(F=6), dict(F=1028), dict(xo=4)], ap: [dict(F=6), dict(F=1028), dict(xo=4), dict(one_stat=True)],
           bw: [dict(F=6), dict(F=1028), dict(xo=4)]}
    for fn, cases in bad.items():
        assert fn() == 0, names[fn]
        for kw in cases:
            assert fn(**kw) == -1 and names[fn] in lib.bns_last_error(), (names[fn], kw)
    need = lib.bns_bn_workspace_bytes(256)
    assert cs(wsb=need - 16) == -3 and b"bns_bn_colsums_f32" in lib.bns_last_error()
    torch.cuda.synchronize()
