"""Dense layers of the path (K8, module/layer.py:30, 38, 83, 92 of the reference are plain ``nn.Linear`` in fp32).

The reference runs them as true-fp32 cuBLAS SGEMMs (torch 1.12: ``allow_tf32=False`` for matmul).  The fp32
SIMT pipe (67 TFLOP/s on the H100 SXM data sheet) is far below the tensor cores, while one TF32 tensor-core
pass would miss the 1e-4 parity bar (10-bit mantissa).  ``linear()`` therefore uses the error-compensated **3xTF32**
scheme: split every f32 operand into ``hi = tf32(x)`` and ``lo = x - hi`` (exact in f32) and accumulate
``hi*hi + hi*lo + lo*hi`` on the tensor cores with f32 accumulation; the dropped ``lo*lo`` term is 2^-22 relative.

``MODE`` (env BNS_DENSE): "tc" (default) -- the hand-written wgmma kernels of csrc/dense_tc.cuh: 3xTF32 with the
operand split fused into the TMA -> shared memory -> wgmma pipeline (forward, input gradient, split-K weight gradient);
operands whose rows are not 16-byte multiples fall back to fp32 cuBLAS | "fp32" (cuBLAS SIMT, the literal reference
precision) | "auto" (library-composed 3xtf32 where K >= 512) | "3xtf32" | "bf16x3".
``tools/check_dense_tc.py perf`` times the Reddit-shape layer GEMMs against cuBLAS.  On the previous GPU the
library-composed 3xtf32 (three cuBLAS TF32 GEMMs + a split pass) was slower than fp32 cuBLAS except at K >= 512, and
bf16x3 always slower.
"""
import os

import torch
import torch.nn.functional as F

import threading

# torch.backends.cuda.matmul.allow_tf32 is process-global and read at enqueue time.  Ranks that are threads of one
# process (tests, smoke) must not see each other's setting: every GEMM of this module is enqueued under this lock,
# fp32 ones included (forward AND backward -- hence the custom fp32 Function below instead of F.linear).
_GEMM_LOCK = threading.RLock()

MODE = os.environ.get("BNS_DENSE", "tc")
# bench.py sets this to a list to collect (start_event, end_event, useful_flops, algorithmic_bytes) per wgmma GEMM
PROFILE = None
MIN_K_3X = 512       # "auto": 3xTF32 only where the GEMM is big enough to repay the split pass (layer 0: K = 2 * n_feat)


def _split(t: torch.Tensor):
    """hi = t rounded to TF32 (10 explicit mantissa bits, round-to-nearest on the 13 dropped bits), lo = t - hi.
    One fused pass (``bns_split_tf32_f32``) on CUDA; torch ops elsewhere (CPU checks)."""
    t = t.contiguous()
    if t.is_cuda and t.numel() % 4 == 0:
        from .._lib import check, lib
        hi, lo = torch.empty_like(t), torch.empty_like(t)
        with torch.cuda.device(t.device):
            check(lib.bns_split_tf32_f32(t.data_ptr(), t.numel(), hi.data_ptr(), lo.data_ptr(),
                                         torch.cuda.current_stream().cuda_stream), "bns_split_tf32_f32")
        return hi, lo
    bits = t.view(torch.int32)
    hi = ((bits + 0x1000) & -0x2000).view(torch.float32)
    return hi, t - hi


def _mm3(a2, b2, trans_a=False, trans_b=False) -> torch.Tensor:
    """op(a) @ op(b) with 3xTF32 error compensation; ``a2`` / ``b2`` are (hi, lo) pairs."""
    (ah, al), (bh, bl) = a2, b2
    if trans_a:
        ah, al = ah.t(), al.t()
    if trans_b:
        bh, bl = bh.t(), bl.t()
    with _GEMM_LOCK:
        prev = torch.backends.cuda.matmul.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = True
        try:
            out = torch.mm(al, bh)          # small terms first, then the dominant one: better rounding
            out.addmm_(ah, bl)
            out.addmm_(ah, bh)
        finally:
            torch.backends.cuda.matmul.allow_tf32 = prev
    return out


class _Linear3x(torch.autograd.Function):

    @staticmethod
    def forward(ctx, x, weight, bias):
        x2, w2 = _split(x), _split(weight)
        ctx.x2, ctx.w2, ctx.has_bias = x2, w2, bias is not None
        y = _mm3(x2, w2, trans_b=True)
        if bias is not None:
            y += bias
        return y

    @staticmethod
    def backward(ctx, dy):
        d2 = _split(dy)
        dx = _mm3(d2, ctx.w2) if ctx.needs_input_grad[0] else None
        dw = _mm3(d2, ctx.x2, trans_a=True) if ctx.needs_input_grad[1] else None
        db = dy.sum(0) if ctx.has_bias and ctx.needs_input_grad[2] else None
        ctx.x2 = ctx.w2 = None
        return dx, dw, db


# ---- bf16x3: x = b0 + b1 + b2 (24 mantissa bits), six bf16 tensor-core GEMMs, f32 accumulation ----------------------
_PAIRS = ((2, 0), (0, 2), (1, 1), (1, 0), (0, 1), (0, 0))          # small terms first


def _split3(t: torch.Tensor):
    from .._lib import check, lib
    t = t.contiguous()
    n = t.numel()
    if n % 4:
        raise RuntimeError("bf16x3 split needs a multiple of 4 elements")
    outs = [torch.empty(t.shape, dtype=torch.bfloat16, device=t.device) for _ in range(3)]
    with torch.cuda.device(t.device):
        check(lib.bns_split_bf16x3_f32(t.data_ptr(), n, outs[0].data_ptr(), outs[1].data_ptr(), outs[2].data_ptr(),
                                       torch.cuda.current_stream().cuda_stream), "bns_split_bf16x3_f32")
    return outs


def _mm6(a3, b3, trans_a=False, trans_b=False):
    """sum over i + j <= 2 of  op(a_i) @ op(b_j)  in f32."""
    acc = None
    for i, j in _PAIRS:
        a = a3[i].t() if trans_a else a3[i]
        b = b3[j].t() if trans_b else b3[j]
        acc = torch.mm(a, b, out_dtype=torch.float32) if acc is None else torch.addmm(acc, a, b, out_dtype=torch.float32)
    return acc


class _LinearBf16x3(torch.autograd.Function):

    @staticmethod
    def forward(ctx, x, weight, bias):
        x3, w3 = _split3(x), _split3(weight)
        ctx.x3, ctx.w3, ctx.has_bias = x3, w3, bias is not None
        y = _mm6(x3, w3, trans_b=True)                      # [M,K] @ [N,K]^T
        if bias is not None:
            y += bias
        return y

    @staticmethod
    def backward(ctx, dy):
        d3 = _split3(dy)
        dx = _mm6(d3, ctx.w3) if ctx.needs_input_grad[0] else None                # [M,N] @ [N,K]
        dw = _mm6(d3, ctx.x3, trans_a=True) if ctx.needs_input_grad[1] else None  # [M,N]^T @ [M,K]
        db = dy.sum(0) if ctx.has_bias and ctx.needs_input_grad[2] else None
        ctx.x3 = ctx.w3 = None
        return dx, dw, db


class _LinearFp32(torch.autograd.Function):
    """Plain f32 cuBLAS (the reference's precision), enqueued under ``_GEMM_LOCK`` in both directions."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        ctx.save_for_backward(x, weight)
        ctx.has_bias = bias is not None
        with _GEMM_LOCK:
            return F.linear(x, weight, bias)

    @staticmethod
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        with _GEMM_LOCK:
            dx = dy.mm(weight) if ctx.needs_input_grad[0] else None
            dw = dy.t().mm(x) if ctx.needs_input_grad[1] else None
        db = dy.sum(0) if ctx.has_bias and ctx.needs_input_grad[2] else None
        return dx, dw, db


# ---- "tc": hand-written wgmma kernels (csrc/dense_tc.cuh), 3xTF32 with the split fused into the pipeline ---------
def _tc_operand(t: torch.Tensor) -> bool:
    return (t.is_cuda and t.dtype == torch.float32 and t.dim() == 2 and t.stride(1) == 1 and t.stride(0) % 4 == 0
            and t.stride(0) >= t.shape[1] and t.data_ptr() % 16 == 0 and t.shape[0] > 0 and t.shape[1] > 0)


def tc_eligible(x: torch.Tensor, weight: torch.Tensor, bias=None) -> bool:
    """Shapes the wgmma kernels take: 16-byte aligned rows everywhere the forward AND both gradients touch."""
    return (_tc_operand(x) and _tc_operand(weight) and x.shape[1] == weight.shape[1] and weight.shape[0] % 4 == 0
            and weight.shape[1] % 4 == 0
            and (bias is None or (bias.is_cuda and bias.dtype == torch.float32 and bias.is_contiguous()
                                  and bias.data_ptr() % 16 == 0)))


def tc_mm_tn(a: torch.Tensor, b: torch.Tensor, bias=None, addend=None, row_scale=None, out=None,
             bf16: bool = False) -> torch.Tensor:
    """``(a @ b.T (+ bias) (+ addend)) (* row_scale[:, None])``: a [M, K], b [N, K], addend [M, >= N]
    (``bns_dense_tn_3xtf32``).  ``out`` may alias ``addend`` (in-place accumulation into a gradient buffer).
    ``bf16``: the products of ``bns_dense_tn_bf16`` instead -- a and b rounded to bf16 inside the kernel, f32 sums and
    epilogue (``--dense-dtype bf16``)."""
    from .._lib import check, lib
    fn_name = "bns_dense_tn_bf16" if bf16 else "bns_dense_tn_3xtf32"
    M, K = a.shape
    N = b.shape[0]
    if out is None:
        out = torch.empty((M, N), dtype=torch.float32, device=a.device)
    prof = PROFILE
    if prof is not None:
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record(torch.cuda.current_stream(a.device))
    with torch.cuda.device(a.device):
        check(getattr(lib, fn_name)(a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0),
                                    None if bias is None else bias.data_ptr(),
                                    None if addend is None else addend.data_ptr(),
                                    0 if addend is None else addend.stride(0),
                                    None if row_scale is None else row_scale.data_ptr(), out.data_ptr(), out.stride(0), M, N, K,
                                    torch.cuda.current_stream().cuda_stream), fn_name)
    if prof is not None:
        ev1.record(torch.cuda.current_stream(a.device))
        prof.append((ev0, ev1, 2.0 * M * N * K, 4.0 * (M * K + N * K + M * N * (2 if addend is not None else 1))))
    return out


def tc_mm_tn_fp8(a, b, bias=None, addend=None, row_scale=None, out=None) -> torch.Tensor:
    """``tc_mm_tn`` on fp8 rows (``ops.Fp8Rows``, a [M, K], b [N, K]; ``bns_dense_tn_fp8``, ``--dense-dtype fp8``):
    ``(sum_k qa qb) * a.scale[:, None] * b.scale[None, :]``, the sums of each 128-code block promoted to f32, then the
    same f32 epilogue (bias, addend -- which ``out`` may alias --, row_scale)."""
    from .. import ops
    from .._lib import check, lib
    ops._table(a, "a")
    ops._table(b, "b")
    M, K = a.shape
    N = b.shape[0]
    if b.shape[1] != K:
        raise ValueError(f"tc_mm_tn_fp8: a has {K} columns, b {b.shape[1]}")
    if out is None:
        out = torch.empty((M, N), dtype=torch.float32, device=a.device)
    prof = PROFILE
    if prof is not None:
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record(torch.cuda.current_stream(a.device))
    with torch.cuda.device(a.device):
        check(lib.bns_dense_tn_fp8(a.codes.data_ptr(), a.codes.stride(0), a.scale.data_ptr(), b.codes.data_ptr(),
                                   b.codes.stride(0), b.scale.data_ptr(), None if bias is None else bias.data_ptr(),
                                   None if addend is None else addend.data_ptr(), 0 if addend is None else addend.stride(0),
                                   None if row_scale is None else row_scale.data_ptr(), out.data_ptr(), out.stride(0), M, N,
                                   K, torch.cuda.current_stream().cuda_stream), "bns_dense_tn_fp8")
    if prof is not None:
        ev1.record(torch.cuda.current_stream(a.device))
        prof.append((ev0, ev1, 2.0 * M * N * K, M * K + N * K + 4.0 * (M + N + M * N * (2 if addend is not None else 1))))
    return out


_WS = {}


def _workspace(kind: str, nbytes: int, device) -> torch.Tensor:
    """Scratch reused across calls, one per (kind, device, stream): ranks that are threads of one process run on their
    own streams and must not share it; consecutive calls on one stream are ordered."""
    key = (kind, device, torch.cuda.current_stream(device).cuda_stream)
    ws = _WS.get(key)
    if ws is None or ws.numel() < nbytes:
        ws = _WS[key] = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=device)
    return ws


def colsum(x: torch.Tensor, out=None, out2=None) -> torch.Tensor:
    """``x.sum(0)`` of a 2-D f32 CUDA matrix (bias gradients): ``bns_colsum_f32`` where the rows are 16-byte
    multiples, torch otherwise.  ``out`` / ``out2``: destinations (e.g. gradient slots of the parameter arena)."""
    if not (_tc_operand(x) and x.shape[1] % 4 == 0 and x.shape[1] <= 1024):
        r = x.sum(0)
        if out is not None:
            out.copy_(r)
        if out2 is not None:
            out2.copy_(r)
        return r if out is None else out
    from .._lib import check, lib
    rows, cols = x.shape
    if out is None:
        out = torch.empty(cols, dtype=torch.float32, device=x.device)
    nbytes = lib.bns_colsum_workspace_bytes(cols)
    ws = _workspace("colsum", nbytes, x.device)
    with torch.cuda.device(x.device):
        check(lib.bns_colsum_f32(x.data_ptr(), x.stride(0), rows, cols, out.data_ptr(),
                                 None if out2 is None else out2.data_ptr(), ws.data_ptr(), nbytes,
                                 torch.cuda.current_stream().cuda_stream), "bns_colsum_f32")
    return out


def tc_mm_nt(a: torch.Tensor, b: torch.Tensor, out=None, bf16: bool = False) -> torch.Tensor:
    """``a.T @ b``: a [R, N1], b [R, N2] -> [N1, N2], contraction over the rows (``bns_dense_nt_3xtf32``).  ``bf16``:
    ``bns_dense_nt_bf16`` (operands rounded to bf16 inside the kernel, same split-K plan and workspace)."""
    from .._lib import check, lib
    fn_name = "bns_dense_nt_bf16" if bf16 else "bns_dense_nt_3xtf32"
    R, N1 = a.shape
    N2 = b.shape[1]
    if out is None:
        out = torch.empty((N1, N2), dtype=torch.float32, device=a.device)
    nbytes = lib.bns_dense_nt_workspace_bytes(R, N1, N2)
    ws = _workspace("mm_nt", nbytes, a.device)
    prof = PROFILE
    if prof is not None:
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record(torch.cuda.current_stream(a.device))
    with torch.cuda.device(a.device):
        check(getattr(lib, fn_name)(a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0), out.data_ptr(), out.stride(0),
                                    R, N1, N2, ws.data_ptr(), nbytes, torch.cuda.current_stream().cuda_stream), fn_name)
    if prof is not None:
        ev1.record(torch.cuda.current_stream(a.device))
        prof.append((ev0, ev1, 2.0 * R * N1 * N2, 4.0 * (R * N1 + R * N2 + N1 * N2)))
    return out


class _LinearTc(torch.autograd.Function):
    """``x @ W^T + b (+ addend)``; the addend (the other branch of ``linear1(feat) + linear2(ah)``) rides in the
    epilogue and simply receives ``dY`` in backward."""

    @staticmethod
    def forward(ctx, x, weight, bias, addend):
        ctx.save_for_backward(x, weight)
        ctx.has_bias = bias is not None
        return tc_mm_tn(x, weight, bias, addend)

    @staticmethod
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        dy = dy.contiguous()
        dx = tc_mm_tn(dy, weight.t().contiguous()) if ctx.needs_input_grad[0] else None     # dY @ W
        dw = tc_mm_nt(dy, x) if ctx.needs_input_grad[1] else None                            # dY^T @ X
        db = colsum(dy) if ctx.has_bias and ctx.needs_input_grad[2] else None
        da = dy if ctx.needs_input_grad[3] else None
        return dx, dw, db, da


def linear(x: torch.Tensor, weight: torch.Tensor, bias=None, addend=None) -> torch.Tensor:
    """Drop-in for ``F.linear`` on 2-D f32 CUDA inputs; ``addend`` ([M, >= out_features], extra columns ignored) is
    added to the result -- inside the GEMM epilogue in "tc" mode (when it has exactly the padded output width)."""
    n = weight.shape[0]
    if addend is not None:
        y = _linear(x, weight, bias, addend)
        return y if y is not None else _linear(x, weight, bias, None) + addend[:, :n]
    return _linear(x, weight, bias, None)


def _linear(x, weight, bias, addend):
    """Returns None when ``addend`` was given but cannot be fused (the caller adds it)."""
    ok = x.is_cuda and x.dtype == torch.float32 and x.dim() == 2
    if MODE == "tc" and ok:
        n = weight.shape[0]
        pad = (-n) % 4
        add_ok = addend is None or (_tc_operand(addend) and addend.shape[0] == x.shape[0] and addend.shape[1] == n + pad)
        if pad == 0:
            if add_ok and tc_eligible(x, weight, bias):
                return _LinearTc.apply(x, weight, bias, addend)
        elif add_ok and weight.dim() == 2 and weight.is_cuda and weight.dtype == torch.float32:
            # e.g. 41 classes: run 44 output columns (zero rows of W) so that every row stays 16-byte aligned for TMA
            # and slice; autograd pads dY / slices dW accordingly
            w = F.pad(weight, (0, 0, 0, pad))
            b = F.pad(bias, (0, pad)) if bias is not None else None
            if tc_eligible(x, w, b):
                return _LinearTc.apply(x, w, b, addend)[:, :n]
        if addend is not None:
            return None
        return _LinearFp32.apply(x, weight, bias)        # shapes TMA cannot address (rows not 16-byte multiples)
    if addend is not None:
        return None
    if MODE == "bf16x3" and ok and x.numel() % 4 == 0 and weight.numel() % 4 == 0 and weight.shape[0] % 4 == 0:
        return _LinearBf16x3.apply(x, weight, bias)
    if ok and (MODE == "3xtf32" or (MODE == "auto" and x.shape[1] >= MIN_K_3X)):
        return _Linear3x.apply(x, weight, bias)
    if ok:
        return _LinearFp32.apply(x, weight, bias)
    return F.linear(x, weight, bias)
