"""Float64 restatement of GAT's training attention -- the ``u_add_v``, ``leaky_relu``, ``edge_softmax``, ``attn_drop``
and ``u_mul_e`` + ``sum`` of ``dgl.nn.GATConv`` -- over explicit entry lists.  The attention kernels' tests compare
``graph.GatAttention`` with it."""
import torch
import torch.nn.functional as F


def gat_attention_reference(ft, el, er, u, v, n_rows, H, Fo, d, slope=0.2, keep=None, p=0.0):
    """Entry ``k`` sends ``ft[u[k]]`` to row ``v[k]``.  Per head

        a = edge_softmax(leaky_relu(el[u] + er[v]))   (times keep / (1 - p) when a keep mask [nnz, H] is given)
        rst[r] = sum over the entries k of row r of a[k] * ft[u[k]]

    and the gradients of ``<rst, d>`` with respect to ``ft``, ``el`` and ``er``, all in float64 on the CPU.  The scores
    and the softmax go through autograd, so the LeakyReLU at 0 and the softmax follow torch.  The rest is linear in
    ``ft`` and is written out one head at a time (``rst = A ft``, ``d ft = A^T d``, ``d a[k] = <d[v[k]], ft[u[k]]>``):
    nothing of shape ``[nnz, H, Fo]`` is held, so H * Fo = 1024 stays small.

    Returns ``(rst [n_rows, H * Fo], d_ft, d_el, d_er, e, a_da)``: ``e [nnz, H]`` the scores after the LeakyReLU,
    ``a_da [nnz, H]`` the products ``a[k] * d a[k]`` whose row sums the softmax backward subtracts (the size of the
    terms that cancel in d er)."""
    ft, d = ft.double().view(-1, H, Fo), d.double().view(-1, H, Fo)
    elr, err = el.double().clone().requires_grad_(True), er.double().clone().requires_grad_(True)
    e = F.leaky_relu(elr[u] + err[v], slope)
    m = torch.full((n_rows, H), float("-inf"), dtype=torch.float64)
    m = m.scatter_reduce(0, v.unsqueeze(1).expand(-1, H), e.detach(), "amax")
    ex = torch.exp(e - m[v])
    den = torch.zeros(n_rows, H, dtype=torch.float64).index_add(0, v, ex)
    a = ex / den[v]
    if keep is not None:
        a = a * keep.double() / (1.0 - p)
    rst, d_ft, d_a = [], [], []
    with torch.no_grad():
        ad = a.detach()
        for h in range(H):
            fh, dh = ft[:, h], d[:, h]
            rst.append(torch.zeros(n_rows, Fo, dtype=torch.float64).index_add(0, v, ad[:, h:h + 1] * fh[u]))
            d_ft.append(torch.zeros(ft.shape[0], Fo, dtype=torch.float64).index_add(0, u, ad[:, h:h + 1] * dh[v]))
            d_a.append((dh[v] * fh[u]).sum(1))
    d_a = torch.stack(d_a, 1)
    (a * d_a).sum().backward()
    return (torch.stack(rst, 1).reshape(n_rows, H * Fo), torch.stack(d_ft, 1).reshape(-1, H * Fo), elr.grad, err.grad,
            e.detach(), ad * d_a)
