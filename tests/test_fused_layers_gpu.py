"""The fused training layers of ``fused.py`` against a float64 restatement (tests/layer_reference.py), element by
element, through ``GraphSAGELayer`` / ``GCNLayer.forward(..., fused=(arena, p, seed, holder))`` in training mode.

Every forward output, ``d h_u`` and every parameter gradient slot of the ``ParamArena`` is checked; the arena's gradient
buffer is filled with NaN before each backward, so a slot the backward does not write fails, and pad rows / entries
must come out exactly 0.  The widths are the benchmark's (precomputed 1204 -> 256, 256 -> 256, 256 -> 41 classes padded
to 44 at a 48-float stride) and those of the other dataset shapes (100 -> 47, 256 -> 100, 128 -> 172).  Both branches
of each layer (aggregate first, and transform first for a layer that narrows) run at 256 -> 41 and must agree.  The
partition has rows of 3,000+ entries, empty rows, halo-only rows, a chunk size of 64 so that long rows span many chunks,
and the halo variants: a 10 % and a 50 % sample through the epoch's compaction, the slot-map fallback, nothing
received, no halo matrix, and 2 source-row blocks forced on the inner passes.  Also: ``PPLinearFn``'s dropout against
its replayed mask, the halo pass waiting for the exchange's ``ready`` event, the halo rows of the input gradient handed
to the exchange only once final, and bit-identical repeats."""
import functools
import types

import pytest
import torch

from tests import layer_reference as R

pytestmark = pytest.mark.gpu

N_IN, N_HALO, CHUNK = 3000, 2000, 64
HEAVY = {0: 3100, 1234: 3600, N_IN - 1: 4200}       # rows of 3,000+ inner entries (columns repeat: n_in = 3000)
SLEEP_CYCLES = 20_000_000                           # ~10 ms of torch.cuda._sleep on an H100


def _dev():
    return torch.device("cuda:0")


@functools.lru_cache(maxsize=None)
def _host_graph():
    """CSR of the inner (n_in x n_in) and halo (n_in x n_halo) matrices, ~31 entries per row on average."""
    gen = torch.Generator().manual_seed(0)
    r = torch.rand(N_IN, generator=gen)
    many = torch.rand(N_IN, generator=gen) < 0.1                    # rows longer than one chunk
    deg_in = torch.poisson(torch.where(many, 80.0, 14.0), generator=gen).long()
    deg_out = torch.poisson(torch.where(many, 25.0, 5.0), generator=gen).long()
    deg_in[r < 0.06] = 0                                            # halo-only rows ...
    deg_out[r < 0.03] = 0                                           # ... and rows without any entry
    for row, d in HEAVY.items():
        deg_in[row], deg_out[row] = d, 300
    ip_in, ip_out = (torch.cat([torch.zeros(1, dtype=torch.int64), d.cumsum(0)]) for d in (deg_in, deg_out))
    ix_in = torch.randint(0, N_IN, (int(ip_in[-1]),), generator=gen)
    ix_out = torch.randint(0, N_HALO, (int(ip_out[-1]),), generator=gen)
    return ip_in, ix_in, ip_out, ix_out, gen


@functools.lru_cache(maxsize=None)
def _case(kind, variant):
    """The partition graph of ``kind`` ("sage" or "gcn": GCN's compaction carries the halo column scale) in one halo
    ``variant``, its norms, and the reference's entry lists: destination row ``v``, row of ``h_u`` ``u``, and static
    source id ``c`` (inner node, or ``n_in`` + halo node) of every live entry."""
    from bns_gcn_b200 import ops
    from bns_gcn_b200.graph import PartitionGraph
    dev = _dev()
    ip_in, ix_in, ip_out, ix_out, _ = _host_graph()
    gen = torch.Generator().manual_seed(17)
    deg = (ip_in[1:] - ip_in[:-1]) + (ip_out[1:] - ip_out[:-1])
    if kind == "sage":
        in_norm = deg.clamp(min=1).float() * (0.75 + 0.5 * torch.rand(N_IN, generator=gen))
        out_norm = None
    else:
        in_norm = deg.clamp(min=1).float().sqrt() * (0.75 + 0.5 * torch.rand(N_IN, generator=gen))
        out_norm = torch.randint(1, 60, (N_IN + N_HALO,), generator=gen).float().sqrt()
    with_halo = variant != "no-halo-matrix"
    frac = {"sampled10": 0.1, "nothing-received": 0.0, "no-halo-matrix": 0.0}.get(variant, 0.5)
    n_slab = int(frac * N_HALO)
    slot = torch.full((N_HALO,), -1, dtype=torch.int32)
    slot[torch.randperm(N_HALO, generator=gen)[:n_slab]] = torch.randperm(n_slab, generator=gen).int()

    a_in = ops.DeviceGraph.from_csr(ip_in.to(dev), ix_in.int().to(dev), N_IN, CHUNK)
    a_out = ops.DeviceGraph.from_csr(ip_out.to(dev), ix_out.int().to(dev), N_HALO, CHUNK) if with_halo else None
    assert a_in.n_split_rows > 200 and (a_out is None or a_out.n_split_rows >= 3)
    g = PartitionGraph(N_IN, N_HALO if with_halo else 0, a_in, a_out, dev)
    in_norm = in_norm.to(dev)
    out_norm = out_norm.to(dev) if out_norm is not None else None
    if with_halo:
        g.slot.copy_(slot.to(dev))
        if kind == "gcn" and variant != "colmap-unweighted":
            g.halo_col_scale = g.recip(out_norm)[N_IN:]
        g.refresh_compaction()
        if variant == "colmap":
            g.compact = None
        else:
            assert (g.compact.cw is not None) == (g.halo_col_scale is not None)
    g.n_u = N_IN + n_slab

    rows_in = torch.repeat_interleave(torch.arange(N_IN), ip_in[1:] - ip_in[:-1])
    v, u, c = [rows_in], [ix_in], [ix_in]
    if n_slab:
        rows_out = torch.repeat_interleave(torch.arange(N_IN), ip_out[1:] - ip_out[:-1])
        x = slot[ix_out].long()
        live = x >= 0
        v.append(rows_out[live])
        u.append(N_IN + x[live])
        c.append(N_IN + ix_out[live])
        if g.compact is not None:
            assert int(g.compact.chunk_cnt.sum()) == int(live.sum())
    return types.SimpleNamespace(kind=kind, variant=variant, g=g, n_in=N_IN, n_u=N_IN + n_slab,
                                 v=torch.cat(v).to(dev), u=torch.cat(u).to(dev), c=torch.cat(c).to(dev),
                                 in_norm=in_norm, out_norm=out_norm)


def _layer(kind, fin, fout, pp=False):
    """A real layer on the device, its parameters moved into a ``ParamArena`` (pad rows 0)."""
    from bns_gcn_b200 import fused
    from bns_gcn_b200.module.layer import GCNLayer, GraphSAGELayer
    torch.manual_seed(fin * 1000 + fout)
    layer = (GraphSAGELayer if kind == "sage" else GCNLayer)(fin, fout, use_pp=pp).to(_dev())
    return layer, fused.ParamArena(layer)


def _inputs(case, fin, fout, seed=0):
    """``h_u [n_u, fin]`` and ``dout [n_in, ceil4(fout)]`` with pad columns exactly 0 (as bns_xent_f32 writes them)."""
    gen = torch.Generator().manual_seed(seed)
    h_u = torch.randn(case.n_u, fin, generator=gen)
    dout = torch.zeros(case.n_in, (fout + 3) // 4 * 4)
    dout[:, :fout] = torch.randn(case.n_in, fout, generator=gen)
    return h_u.to(_dev()), dout.to(_dev())


def _step(case, layer, arena, feat, dout):
    """One training step of the layer: ``(padded output, d h_u, {parameter name: padded gradient slot})``."""
    from bns_gcn_b200 import fused
    holder = fused.Transient()
    arena.flat_g.fill_(float("nan"))
    norms = (case.in_norm,) if case.kind == "sage" else (case.in_norm, case.out_norm)
    layer(case.g, feat, *norms, fused=(arena, 0.0, 0, holder))
    holder.value.backward(dout)
    torch.cuda.synchronize()
    grads = {n: arena.grad_padded(p).clone() for n, p in layer.named_parameters()}
    return holder.value.detach().clone(), feat.grad.clone(), grads


def _leaf(t):
    return t.detach().clone().requires_grad_(True)


def _reference(case, layer, arena, h_u, dout):
    """Float64 values and bounds of ``[out, d h_u, d param ...]`` in ``layer.named_parameters()`` order."""
    n_in, v, u = case.n_in, case.v, case.u
    rs = case.g.recip(case.in_norm).double().unsqueeze(1)
    params = [arena.padded(p) for _, p in layer.named_parameters()]
    if case.kind == "sage":
        def fn(h, w1, b1, w2, b2):
            return h[:n_in] @ w1.t() + b1 + (R.aggregate(h, v, u, n_in) * rs) @ w2.t() + b2
    else:
        cs = case.g.recip(case.out_norm).double()[case.c]

        def fn(h, w, b):
            return (R.aggregate(h, v, u, n_in, cs) * rs) @ w.t() + b
    return R.reference(fn, [h_u] + params, dout)


def _check(label, case, layer, arena, h_u, dout, got):
    out, du, grads = got
    want, bound = _reference(case, layer, arena, h_u, dout)
    names = [n for n, _ in layer.named_parameters()]
    R.assert_close(f"{label} out", out, want[0], bound[0])
    R.assert_close(f"{label} d h_u", du, want[1], bound[1])
    for name, w, b in zip(names, want[2:], bound[2:]):
        R.assert_close(f"{label} d {name}", grads[name], w, b)
    fout = layer.linear.out_features if hasattr(layer, "linear") else layer.linear2.out_features
    assert torch.all(out[:, fout:] == 0), f"{label}: pad columns of the output are not 0"
    for name, p in layer.named_parameters():
        assert torch.all(grads[name][p.shape[0]:] == 0), f"{label}: pad of the gradient of {name} is not 0"


SAGE_SHAPES = [(256, 256), (256, 41), (100, 47), (256, 100), (128, 172)]
HALO_VARIANTS = ["sampled10", "colmap", "nothing-received", "no-halo-matrix", "sampled50-2blocks"]
CASES = ([("sage", fin, fout, "sampled50", True) for fin, fout in SAGE_SHAPES]
         + [("gcn", 256, fout, "sampled50", True) for fout in (256, 41)]
         # the aggregate-first branch at the width that otherwise transforms first
         + [(kind, 256, 41, "sampled50", False) for kind in ("sage", "gcn")]
         + [(kind, 256, fout, variant, True) for kind in ("sage", "gcn") for fout in (256, 41) for variant in HALO_VARIANTS]
         # GCN: a compaction without weights while the layer has a halo column scale takes the slot-map path
         + [("gcn", 256, fout, "colmap-unweighted", True) for fout in (256, 41)])


def _setup(monkeypatch, variant, transform_first):
    from bns_gcn_b200.module import layer as layer_mod
    monkeypatch.setattr(layer_mod, "AGGREGATE_AFTER_TRANSFORM", transform_first)
    if variant.endswith("-2blocks"):
        monkeypatch.setenv("BNS_SPMM_COLBLOCKS", "2")
        variant = variant[:-len("-2blocks")]
    else:
        monkeypatch.delenv("BNS_SPMM_COLBLOCKS", raising=False)
    return variant


@pytest.mark.parametrize("kind,fin,fout,variant,transform_first", CASES)
def test_layer_matches_float64(built, monkeypatch, kind, fin, fout, variant, transform_first):
    """Forward, d h_u and every parameter gradient against float64; a second identical step is bit-identical."""
    case = _case(kind, _setup(monkeypatch, variant, transform_first))
    layer, arena = _layer(kind, fin, fout)
    h_u, dout = _inputs(case, fin, fout)
    got = _step(case, layer, arena, _leaf(h_u), dout)
    branch = "transform-first" if transform_first and fout < fin else "aggregate-first"
    _check(f"{kind} {fin}->{fout} {variant} {branch}", case, layer, arena, h_u, dout, got)
    again = _step(case, layer, arena, _leaf(h_u), dout)
    assert torch.equal(got[0], again[0]) and torch.equal(got[1], again[1])
    for name in got[2]:
        assert torch.equal(got[2][name], again[2][name]), name


@pytest.mark.parametrize("kind", ["sage", "gcn"])
def test_both_branches_agree(built, monkeypatch, kind):
    """At 256 -> 41 the transform-first and aggregate-first branches compute the same thing to within rounding."""
    from bns_gcn_b200.module import layer as layer_mod
    case = _case(kind, "sampled50")
    layer, arena = _layer(kind, 256, 41)
    h_u, dout = _inputs(case, 256, 41, seed=5)
    runs = {}
    for flag in (True, False):
        monkeypatch.setattr(layer_mod, "AGGREGATE_AFTER_TRANSFORM", flag)
        runs[flag] = _step(case, layer, arena, _leaf(h_u), dout)
    _, bound = _reference(case, layer, arena, h_u, dout)
    (o1, d1, g1), (o2, d2, g2) = runs[True], runs[False]
    R.assert_close(f"{kind} branches out", o1, o2.double(), bound[0])
    R.assert_close(f"{kind} branches d h_u", d1, d2.double(), bound[1])
    for (name, _), b in zip(layer.named_parameters(), bound[2:]):
        R.assert_close(f"{kind} branches d {name}", g1[name], g2[name].double(), b)


@pytest.mark.parametrize("p", [0.0, 0.5])
@pytest.mark.parametrize("kind,n_feat", [("sage", 602), ("gcn", 604)])
def test_pp_linear_dropout(built, kind, n_feat, p):
    """Layer 0 with precomputed input (``PPLinearFn``): ``(x m / (1 - p)) W^T + b`` and ``dx = (dy W) m / (1 - p)`` with
    the mask ``m`` replayed by ``fused.dropout`` on ones.  The RNG offset moves on between forward and backward (the
    next epoch's): the backward must still use the forward's mask.  GraphSAGE's input is ``[x | mean]``, 1204 wide on
    the Reddit shape; GCN's is the 602-wide ``x`` there, which the fused step does not take (``train._fused_eligible``
    needs a multiple of 4), so GCN runs at 604."""
    from bns_gcn_b200 import fused, ops
    dev = _dev()
    layer, arena = _layer(kind, n_feat, 256, pp=True)
    k = layer.linear.in_features
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(N_IN, k, generator=gen).to(dev)
    dy = torch.randn(N_IN, 256, generator=gen).to(dev)
    seed = 104729
    ops.RNG.update(seed=11, offset=17, offset_dev=None)
    try:
        keep = torch.ones_like(x)
        if p > 0:
            keep = (fused.dropout(torch.ones_like(x), p, seed) != 0).float()
            rate = keep.mean().item()
            assert abs(rate - (1 - p)) <= 0.01 * (1 - p), rate
        feat = _leaf(x)
        arena.flat_g.fill_(float("nan"))
        norms = (None,) if kind == "sage" else (None, None)
        out = layer(None, feat, *norms, fused=(arena, p, seed, None))
        ops.RNG.update(offset=18)
        out.backward(dy)
        torch.cuda.synchronize()
        assert ops.RNG["offset"] == 18, "the backward did not put the RNG offset back"
    finally:
        ops.RNG.update(seed=0, offset=0, offset_dev=None)
    W, b = arena.padded(layer.linear.weight), arena.padded(layer.linear.bias)
    m = keep.double() / (1.0 - p)
    want, bound = R.reference(lambda xx, w, bb: (xx * m) @ w.t() + bb, [x, W, b], dy)
    label = f"{kind} pp {k}->256 p={p}"
    R.assert_close(f"{label} out", out, want[0], bound[0])
    R.assert_close(f"{label} dx", feat.grad, want[1], bound[1])
    R.assert_close(f"{label} d linear.weight", arena.grad_padded(layer.linear.weight), want[2], bound[2])
    R.assert_close(f"{label} d linear.bias", arena.grad_padded(layer.linear.bias), want[3], bound[3])


@pytest.mark.parametrize("transform_first", [True, False], ids=["transform-first", "aggregate-first"])
@pytest.mark.parametrize("kind", ["sage", "gcn"])
def test_halo_pass_waits_for_ready(built, monkeypatch, kind, transform_first):
    """The halo rows of ``h_u`` are NaN until a side stream, after ~10 ms of sleep, copies the true rows in and
    records the event the layer gets as ``ready``; the layer runs on the main stream and must see the true rows."""
    case = _case(kind, _setup(monkeypatch, "sampled50", transform_first))
    layer, arena = _layer(kind, 256, 41)
    h_u, dout = _inputs(case, 256, 41, seed=7)
    _step(case, layer, arena, _leaf(h_u), dout)          # warm-up: every lazy buffer and derived weight exists
    n_in = case.n_in
    feat = h_u.clone()
    feat[n_in:] = float("nan")
    feat.requires_grad_(True)
    side, ready = torch.cuda.Stream(), torch.cuda.Event()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        torch.cuda._sleep(SLEEP_CYCLES)
        with torch.no_grad():
            feat[n_in:].copy_(h_u[n_in:])
        ready.record(side)
    feat._bns_ready = ready
    got = _step(case, layer, arena, feat, dout)
    _check(f"{kind} ready {'transform-first' if transform_first else 'aggregate-first'}", case, layer, arena, h_u,
           dout, got)


class _Exchange:
    """Stands in for ``feature_buffer.Buffer``: keeps a copy of the halo rows of the gradient it is handed."""

    def __init__(self, n_in):
        self.n_in, self.calls = n_in, []

    def begin_backward(self, layer, grad):
        self.calls.append((layer, grad[self.n_in:].clone()))


@pytest.mark.parametrize("transform_first", [True, False], ids=["transform-first", "aggregate-first"])
def test_exchange_gets_final_halo_gradient(built, monkeypatch, transform_first):
    """``SageConvFn.backward`` hands ``d h_u`` to ``begin_backward`` once its halo rows are final: the copy taken at
    that point equals the returned gradient's halo rows.  Freed device blocks are filled with NaN first, so rows read
    before they are written cannot match by chance."""
    case = _case("sage", _setup(monkeypatch, "sampled50", transform_first))
    layer, arena = _layer("sage", 256, 41)
    h_u, dout = _inputs(case, 256, 41, seed=9)
    ex = _Exchange(case.n_in)
    feat = _leaf(h_u)
    feat._bns_exchange = (ex, 2)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    poison = [torch.full((case.n_u, 256), float("nan"), device=_dev()) for _ in range(6)]
    del poison
    got = _step(case, layer, arena, feat, dout)
    assert len(ex.calls) == 1 and ex.calls[0][0] == 2
    halo = ex.calls[0][1]
    assert halo.shape == (case.n_u - case.n_in, 256)
    assert torch.equal(halo, got[1][case.n_in:])
    _check(f"sage exchange {'transform-first' if transform_first else 'aggregate-first'}", case, layer, arena, h_u,
           dout, got)
