"""Float64 restatement of the graph transformer layer's attention -- the score ``<q_v, k_u> * scale``, ``edge_softmax``,
``attn_drop`` and the weighted sum of the value rows -- over explicit entry lists, and of the whole layer.  The kernels'
tests compare ``graph.TconvAttention``, ``graph.tconv_infer`` and ``graph.tconv_infer_block`` with it; the oracle's
``transformer`` kind (tests/transformer_oracle.py) is checked against ``transformer_layer_reference``."""
import torch


def tconv_scores_reference(q, k, src, dst, H, Fp, scale):
    """``s [nnz, H]`` in float64 (no gradient)."""
    q3, k3 = q.double().view(-1, H, Fp), k.double().view(-1, H, Fp)
    out = torch.empty(src.numel(), H, dtype=torch.float64)
    for k0 in range(0, src.numel(), 4096):
        sl = slice(k0, k0 + 4096)
        out[sl] = (q3[dst[sl]] * k3[src[sl]]).sum(-1) * scale
    return out


def _softmax_sum(s, val3, src, dst, n_rows, H, keep=None, p=0.0):
    m = torch.full((n_rows, H), float("-inf"), dtype=torch.float64)
    m = m.scatter_reduce(0, dst.unsqueeze(1).expand(-1, H), s.detach(), "amax")
    ex = torch.exp(s - m[dst])
    den = torch.zeros(n_rows, H, dtype=torch.float64).index_add(0, dst, ex)
    a = ex / den[dst]
    if keep is not None:
        a = a * keep.double() / (1.0 - p)
    return torch.zeros(n_rows, H, val3.shape[-1], dtype=torch.float64).index_add(0, dst, a.unsqueeze(2) * val3[src])


def tconv_attention_reference(q, k, val, src, dst, n_rows, H, Fp, d, scale, keep=None, p=0.0):
    """Entry ``e`` sends ``val[src[e]]`` to row ``dst[e]``.  Per head

        s = scale * <q[dst], k[src]>,  a = edge_softmax(s)  (times keep / (1 - p) with a mask [nnz, H])
        rst[r] = sum over the entries e of row r of a[e] * val[src[e]]

    and the gradients of ``<rst, d>`` with respect to ``q``, ``k`` and ``val``, all in float64 through autograd.
    Returns ``(rst [n_rows, H * Fp], d_q, d_k, d_val, s [nnz, H])``."""
    qr, kr, vr = (t.double().clone().requires_grad_(True) for t in (q, k, val))
    q3, k3, v3 = qr.view(-1, H, Fp), kr.view(-1, H, Fp), vr.view(-1, H, Fp)
    s = (q3[dst] * k3[src]).sum(-1) * scale                                    # [nnz, H]
    rst = _softmax_sum(s, v3, src, dst, n_rows, H, keep, p)
    (rst * d.double().view(n_rows, H, Fp)).sum().backward()
    return rst.detach().reshape(n_rows, H * Fp), qr.grad, kr.grad, vr.grad, s.detach()


def tconv_infer_reference(indptr, indices, q, k, val, H, Fp, scale):
    """The evaluation forward on a CSR graph (rows without entries give 0), float64."""
    n_rows = indptr.numel() - 1
    dst = torch.repeat_interleave(torch.arange(n_rows), indptr[1:] - indptr[:-1])
    src = indices.long()
    s = tconv_scores_reference(q, k, src, dst, H, Fp, scale)
    rst = _softmax_sum(s, val.double().view(-1, H, Fp), src, dst, n_rows, H)
    return rst.reshape(n_rows, H * Fp)


def transformer_layer_reference(x_src, src, dst, n_dst, wq, bq, wk, bk, wv, bv, ws, bs, H, C):
    """The layer without dropout, in the dtype of its arguments: ``[n_dst, H, C]`` =
    attention over ``(q = x_dst wq^T + bq, k = x_src wk^T + bk, v = x_src wv^T + bv)`` with scale ``1/sqrt(C)``, plus
    ``x_dst ws^T + bs`` on every head, ``x_dst = x_src[:n_dst]``."""
    x_dst = x_src[:n_dst]
    q3 = (x_dst @ wq.t() + bq).view(-1, H, C)
    k3 = (x_src @ wk.t() + bk).view(-1, H, C)
    v3 = (x_src @ wv.t() + bv).view(-1, H, C)
    s = (q3[dst] * k3[src]).sum(-1) / C ** 0.5
    m = torch.full((n_dst, H), float("-inf"), dtype=s.dtype)
    m = m.scatter_reduce(0, dst.unsqueeze(1).expand(-1, H), s.detach(), "amax")
    ex = torch.exp(s - m[dst])
    den = torch.zeros(n_dst, H, dtype=s.dtype).index_add(0, dst, ex)
    a = ex / den[dst]
    rst = torch.zeros(n_dst, H, C, dtype=s.dtype).index_add(0, dst, a.unsqueeze(2) * v3[src])
    return rst + (x_dst @ ws.t() + bs).unsqueeze(1)
