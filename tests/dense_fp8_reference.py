"""The product of ``bns_dense_tn_fp8`` (``--dense-dtype fp8``) restated on the host in float64:

  C[m, n] = (sum_k qa[m, k] qb[n, k]) * sa[m] * sb[n]  (+ bias[n]) (+ addend[m, n])  (* row_scale[m])

with the operands as fp8 rows (``tests/fp8_reference.py``: e4m3 codes, one power-of-two scale per row), and the bound
every GEMM test holds the kernel to: the same sum over the magnitudes of its terms."""
import torch


def tn(qa, sa, qb, sb, bias=None, addend=None, row_scale=None):
    """``(ref, bound)`` in float64 for codes ``qa [M, K]``, ``qb [N, K]`` (``float8_e4m3fn``) and scales ``sa [M]``,
    ``sb [N]``; the epilogue terms are f32 tensors or ``None``."""
    a, b = qa.double(), qb.double()
    s = sa.double()[:, None] * sb.double()[None, :]
    ref, bnd = (a @ b.t()) * s, (a.abs() @ b.abs().t()) * s.abs()
    if bias is not None:
        ref = ref + bias.double()
        bnd = bnd + bias.double().abs()
    if addend is not None:
        ref = ref + addend.double()
        bnd = bnd + addend.double().abs()
    if row_scale is not None:
        rs = row_scale.double()[:, None]
        ref, bnd = ref * rs, bnd * rs.abs()
    return ref, bnd
