"""Float64 restatement of GATv2's attention -- the score ``attn . leaky_relu(z_src[u] + z_dst[v])``, ``edge_softmax``,
``attn_drop`` and the weighted sum of ``dgl.nn.GATv2Conv`` -- over explicit entry lists.  The GATv2 kernels' tests
compare ``graph.Gatv2Attention``, ``graph.gatv2_infer`` and ``graph.gatv2_infer_block`` with it."""
import torch
import torch.nn.functional as F


def gatv2_scores_reference(zs, zd, attn, u, v, H, Fp, slope=0.2):
    """``s [nnz, H]`` in float64 (no gradient)."""
    zs, zd, at = zs.double().view(-1, H, Fp), zd.double().view(-1, H, Fp), attn.double().reshape(1, H, Fp)
    out = torch.empty(u.numel(), H, dtype=torch.float64)
    for k0 in range(0, u.numel(), 4096):
        sl = slice(k0, k0 + 4096)
        out[sl] = (F.leaky_relu(zs[u[sl]] + zd[v[sl]], slope) * at).sum(-1)
    return out


def gatv2_attention_reference(zs, zd, attn, u, v, n_rows, H, Fp, d, slope=0.2, keep=None, p=0.0):
    """Entry ``k`` sends ``zs[u[k]]`` to row ``v[k]``.  Per head

        s = sum_f attn * leaky_relu(zs[u] + zd[v]),  a = edge_softmax(s)  (times keep / (1 - p) with a mask [nnz, H])
        rst[r] = sum over the entries k of row r of a[k] * zs[u[k]]

    and the gradients of ``<rst, d>`` with respect to ``zs``, ``zd`` and ``attn``, all in float64 through autograd.
    Returns ``(rst [n_rows, H * Fp], d_zs, d_zd, d_attn [H * Fp], s [nnz, H])``."""
    zsr = zs.double().clone().requires_grad_(True)
    zdr = zd.double().clone().requires_grad_(True)
    atr = attn.double().reshape(1, H, Fp).clone().requires_grad_(True)
    zs3, zd3 = zsr.view(-1, H, Fp), zdr.view(-1, H, Fp)
    s = (F.leaky_relu(zs3[u] + zd3[v], slope) * atr).sum(-1)                       # [nnz, H]
    m = torch.full((n_rows, H), float("-inf"), dtype=torch.float64)
    m = m.scatter_reduce(0, v.unsqueeze(1).expand(-1, H), s.detach(), "amax")
    ex = torch.exp(s - m[v])
    den = torch.zeros(n_rows, H, dtype=torch.float64).index_add(0, v, ex)
    a = ex / den[v]
    if keep is not None:
        a = a * keep.double() / (1.0 - p)
    rst = torch.zeros(n_rows, H, Fp, dtype=torch.float64).index_add(0, v, a.unsqueeze(2) * zs3[u])
    (rst * d.double().view(n_rows, H, Fp)).sum().backward()
    return (rst.detach().reshape(n_rows, H * Fp), zsr.grad, zdr.grad, atr.grad.reshape(-1), s.detach())


def gatv2_infer_reference(indptr, indices, zs, zd, attn, H, Fp, slope=0.2):
    """The evaluation forward on a CSR graph (rows without entries give 0), float64."""
    n_rows = indptr.numel() - 1
    v = torch.repeat_interleave(torch.arange(n_rows), indptr[1:] - indptr[:-1])
    u = indices.long()
    s = gatv2_scores_reference(zs, zd, attn, u, v, H, Fp, slope)
    m = torch.full((n_rows, H), float("-inf"), dtype=torch.float64).scatter_reduce(
        0, v.unsqueeze(1).expand(-1, H), s, "amax")
    ex = torch.exp(s - m[v])
    den = torch.zeros(n_rows, H, dtype=torch.float64).index_add(0, v, ex)
    a = ex / den[v]
    zs3 = zs.double().view(-1, H, Fp)
    rst = torch.zeros(n_rows, H, Fp, dtype=torch.float64).index_add(0, v, a.unsqueeze(2) * zs3[u])
    return rst.reshape(n_rows, H * Fp)
