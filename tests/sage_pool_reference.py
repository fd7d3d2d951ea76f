"""Restatement of GraphSAGE's max-pooling layer (``SAGEConv(in, out, 'pool')``) over explicit entry lists, with the
winner rule computed explicitly: entry ``k`` sends row ``u[k]`` to row ``v[k]``, the entries are listed in the walk
order of the product's kernels (inner entries in CSR order, then the sampled halo entries in ``a_out``'s order), and
the winner of ``(v, f)`` is the first listed entry whose value equals the maximum.  The gradient of ``m[v, f]`` goes to
that entry's source only (torch's ``amax`` backward would split ties evenly).  The kernels' tests compare
``graph.SageMax``, ``graph.sage_max_infer`` and ``sage_max_infer_block`` with it in float64; the oracle's
``graphsage-pool`` kind (tests/sage_pool_oracle.py) runs ``MaxByWinner`` in float32."""
import torch


def max_first(z, u, v, n_rows):
    """``m [n_rows, F]`` (0 for a row without entries) and ``first [n_rows, F]``: the index into the entry list of
    each column's winner, -1 for a row without entries."""
    nnz, F = u.numel(), z.shape[1]
    zk = z[u]
    idx = v.unsqueeze(1).expand(-1, F)
    m = torch.full((n_rows, F), float("-inf"), dtype=z.dtype).scatter_reduce(0, idx, zk, "amax")
    order = torch.arange(nnz).unsqueeze(1).expand(-1, F)
    first = torch.full((n_rows, F), nnz, dtype=torch.int64).scatter_reduce(
        0, idx, torch.where(zk == m[v], order, torch.full_like(order, nnz)), "amin")
    empty = first == nnz
    return torch.where(empty, torch.zeros_like(m), m), torch.where(empty, torch.full_like(first, -1), first)


class MaxByWinner(torch.autograd.Function):
    """``m = max over the entries u -> v of z[u]`` per column; the backward adds ``d m[v, f]`` to the winner's source
    only."""

    @staticmethod
    def forward(ctx, z, u, v, n_rows):
        m, first = max_first(z.detach(), u, v, n_rows)
        ctx.save_for_backward(u, first)
        ctx.n_u = z.shape[0]
        return m

    @staticmethod
    def backward(ctx, dm):
        u, first = ctx.saved_tensors
        rows, cols = torch.nonzero(first >= 0, as_tuple=True)
        dz = torch.zeros(ctx.n_u, dm.shape[1], dtype=dm.dtype)
        dz.index_put_((u[first[rows, cols]], cols), dm[rows, cols], accumulate=True)
        return dz, None, None, None


def sage_max_reference(z, u, v, pos, n_rows):
    """float64 ``m [n_rows, F]`` and ``win [n_rows, F]``: the winners' positions ``pos[first]`` (-1 for a row without
    entries)."""
    m, first = max_first(z.double(), u, v, n_rows)
    win = torch.where(first >= 0, pos[first.clamp(min=0)], torch.full_like(first, -1))
    return m, win


def sage_max_backward_reference(y, dm, u, v, n_rows):
    """float64 ``d y = relu'(y) * (d m sent to the winners)`` for ``z = relu(y)``."""
    z = torch.relu(y.double())
    _, first = max_first(z, u, v, n_rows)
    rows, cols = torch.nonzero(first >= 0, as_tuple=True)
    dz = torch.zeros_like(z)
    dz.index_put_((u[first[rows, cols]], cols), dm.double()[rows, cols], accumulate=True)
    return dz * (z > 0)


def sage_pool_layer_reference(x, u, v, n_in, w_pool, b_pool, w_self, w_neigh, bias):
    """The layer without dropout: ``rst = x[:n_in] w_self^T + max(relu(x w_pool^T + b_pool)) w_neigh^T + bias``, in the
    dtype of its arguments, differentiable through ``MaxByWinner``."""
    z = torch.relu(x @ w_pool.t() + b_pool)
    m = MaxByWinner.apply(z, u, v, n_in)
    return x[:n_in] @ w_self.t() + m @ w_neigh.t() + bias
