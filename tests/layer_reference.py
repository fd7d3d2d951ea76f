"""Float64 restatement of the fused training layers of ``fused.py`` (``PPLinearFn``, ``SageConvFn``, ``GcnConvFn``) and
of ``ops.spmm_auto``, over explicit entry lists, and the per-element comparison their tests use.

Entry ``k`` adds row ``u[k]`` of the source matrix to output row ``v[k]``, times ``w[k]`` when a per-entry weight is
given (GCN's column scale of the entry's source node).  A layer is written as a function of its differentiable inputs;
``reference`` runs it forward and backward in float64 autograd, once on the inputs and once on their absolute values.
Every layer here is linear in each input with non-negative scales, so the second run gives, for every output and
gradient element, the sum of the magnitudes of the products that make it up: the scale f32 rounding is relative to."""
import torch

# |got - ref| <= TOL * bound: one entry of a row of ~5,000 is 2e-4 of the bound.  Measured on an H100 80GB HBM3, the
# worst error is 0.074 x TOL x bound in the layer tests and 0.17 x in the SpMM tests (a row of 700 entries of one source
# row, whose rounding errors all have one sign).  The tests print their worst ratio per tensor (pytest -s shows them).
TOL = 2e-5


def aggregate(x, v, u, n_rows, w=None):
    """``out[v[k]] += w[k] * x[u[k]]`` in the precision of ``x``."""
    src = x[u] if w is None else x[u] * w.unsqueeze(1)
    return torch.zeros(n_rows, x.shape[1], dtype=x.dtype, device=x.device).index_add(0, v, src)


def _run(fn, inputs, dout):
    xs = [t.detach().double().requires_grad_(True) for t in inputs]
    out = fn(*xs)
    grads = torch.autograd.grad(out, xs, dout.detach().double())
    return [out.detach()] + [g.detach() for g in grads]


def reference(fn, inputs, dout):
    """``([out, d input_0, ...], [bounds of the same])`` of ``out = fn(*inputs)`` under the output gradient ``dout``.
    Constants ``fn`` closes over (row / column scales, dropout masks) must be non-negative."""
    return _run(fn, inputs, dout), _run(fn, [t.abs() for t in inputs], dout.abs())


def assert_close(label, got, want, bound, tol=TOL):
    """``|got - want| <= tol * bound + 1e-30`` element by element.  A failure names the tensor, how many elements and
    rows are out, and the worst element with its row and column.  Returns the worst ratio of error to ``tol * bound``,
    printed with ``label``."""
    got = got.detach().double()
    assert got.shape == want.shape, f"{label}: shape {tuple(got.shape)} != {tuple(want.shape)}"
    err = (got - want).abs()
    lim = tol * bound + 1e-30
    ratio = torch.nan_to_num(err / lim, nan=float("inf"))
    worst = int(torch.argmax(ratio))
    idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(worst), ratio.shape))
    bad = ~(err <= lim)
    if bool(bad.any()):
        rows = torch.unique(torch.nonzero(bad)[:, 0]).tolist()
        raise AssertionError(
            f"{label}: {int(bad.sum())} of {bad.numel()} elements exceed {tol:g} x bound, in {len(rows)} rows "
            f"(first: {rows[:8]}); worst at {idx}: got {got[idx].item()!r}, want {want[idx].item()!r}, "
            f"bound {bound[idx].item()!r}")
    r = ratio.view(-1)[worst].item() if ratio.numel() else 0.0
    print(f"[ratio] {label}: {r:.3g}")
    return r
