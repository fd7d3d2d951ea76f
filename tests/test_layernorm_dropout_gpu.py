"""LayerNorm -> ReLU -> dropout (``bns_ln_relu_dropout_{fwd,bwd}_f32``) and layer 0's input dropout (``bns_dropout_f32``)
against a float64 restatement, element by element, with the dropout mask replayed from the counter layout that
``drop_mask4`` documents: Philox4x32-10 with key ``(seed_lo, seed_hi)`` and counter ``(row_lo, row_hi ^ (vec << 8),
offset_lo, offset_hi)``, ``vec`` the float4 column index; element ``4 vec + i`` is kept when ``float32(r_i) 2^-32 >= p``.

The widths launch every ``NV`` of the kernel (1, 2, 4 with and without an empty slot, 8), partial and full.  The row
counts give every warp at most one row, one more row than warps, about two rows, and the benchmark's 232,965 rows (about
55 rows per warp, so the per-warp ``dgamma`` / ``dbeta`` sums run over many rows).  Each matrix holds a constant row, a
row whose mean is 3000 standard deviations from 0 (a one-pass variance fails there, the kernel's two-pass one does not)
and rows whose pre-activations straddle 0.  Operands are strided and the outputs NaN-filled first.  Also: the masks
against the numpy replay of ``oracle.philox`` at seeds and offsets above 2^32 and at the graph-replay offset wrap,
independence of the model's dropout streams, argument rejection, and a CUDA-graph-replayed epoch at dropout 0.5."""
import contextlib
import io

import numpy as np
import pytest
import torch

from tests import layer_reference as R

pytestmark = pytest.mark.gpu

EPS = 1e-5
MASK32 = 0xFFFFFFFF
WIDTHS = (4, 44, 128, 132, 256, 300, 384, 388, 512, 600, 1024)
BENCH_ROWS = 232_965                    # inner nodes of the benchmark's single partition (Reddit shape)
ROWS = ("1", "7", "32sm", "32sm+1", "64sm+5", "bench")


def _dev():
    return torch.device("cuda:0")


def _n_rows(tag):
    """Row counts relative to the kernel's grid: ``ln_grid`` caps it at 4 blocks of 8 warps per SM."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return {"1": 1, "7": 7, "32sm": 32 * sms, "32sm+1": 32 * sms + 1, "64sm+5": 64 * sms + 5, "bench": BENCH_ROWS}[tag]


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ---- the mask ---------------------------------------------------------------------------------------------------------
def _mulhilo(m, c):
    """``(hi, lo)`` of the 64-bit product of the constant ``m`` and ``c`` (int64 tensor of uint32 values), in 16-bit
    halves so that no int64 product overflows."""
    t1, t2 = m * (c & 0xFFFF), m * (c >> 16)
    s = t1 + ((t2 & 0xFFFF) << 16)
    return (t2 >> 16) + (s >> 32), s & MASK32


def philox_torch(c0, c1, c2, c3, k0, k1):
    """``oracle.philox.philox4x32_10`` on int64 GPU tensors (a test below pins the two to each other)."""
    k0, k1 = k0 & MASK32, k1 & MASK32
    for _ in range(10):
        hi0, lo0 = _mulhilo(0xD2511F53, c0)
        hi1, lo1 = _mulhilo(0xCD9E8D57, c2)
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0, k1 = (k0 + 0x9E3779B9) & MASK32, (k1 + 0xBB67AE85) & MASK32
    return c0, c1, c2, c3


def keep_mask(seed, offset, r0, r1, F, p):
    """bool ``[r1 - r0, F]``: the keep mask of rows ``r0 .. r1 - 1`` (GPU restatement of the layout)."""
    nv = (F + 3) // 4
    rows = torch.arange(r0, r1, dtype=torch.int64, device=_dev())[:, None].expand(-1, nv)
    vec = torch.arange(nv, dtype=torch.int64, device=_dev())[None, :]
    off = torch.full_like(rows, offset & MASK32)
    r = philox_torch(rows & MASK32, (rows >> 32) ^ ((vec << 8) & MASK32), off, torch.full_like(rows, offset >> 32),
                     seed & MASK32, seed >> 32)
    u = torch.stack(r, -1).to(torch.float32) * 2.0 ** -32
    return (u >= float(np.float32(p))).reshape(r1 - r0, 4 * nv)[:, :F]


def keep_mask_np(seed, offset, n, F, p):
    """The same mask from ``oracle.philox.philox4x32_10`` (numpy), as a bool tensor on the CPU."""
    from oracle.philox import philox4x32_10
    nv = (F + 3) // 4
    rows = np.broadcast_to(np.arange(n, dtype=np.uint64)[:, None], (n, nv))
    vec = np.broadcast_to(np.arange(nv, dtype=np.uint64)[None, :], (n, nv))
    m = np.uint64(MASK32)
    r = philox4x32_10((rows & m).astype(np.uint32), ((rows >> np.uint64(32)) ^ ((vec << np.uint64(8)) & m)).astype(np.uint32),
                      np.full((n, nv), offset & MASK32, dtype=np.uint32), np.full((n, nv), offset >> 32, dtype=np.uint32),
                      seed & MASK32, seed >> 32)
    u = np.stack(r, -1).astype(np.float32) * np.float32(2.0 ** -32)
    return torch.from_numpy((u >= np.float32(p)).reshape(n, 4 * nv)[:, :F].copy())


def _keep_scale(p):
    """``1.f / (1.f - p)`` as the kernels compute it."""
    return float(np.float32(1.0) / (np.float32(1.0) - np.float32(p)))


# ---- launches ---------------------------------------------------------------------------------------------------------
def ln_fwd(x, gamma, beta, p, seed, offset, offset_dev=None, y=None):
    from bns_gcn_b200._lib import check, lib
    n, F = x.shape
    y = torch.empty_like(x) if y is None else y
    mean = torch.empty(max(n, 1), device=x.device)
    rstd = torch.empty(max(n, 1), device=x.device)
    check(lib.bns_ln_relu_dropout_fwd_f32(x.data_ptr(), x.stride(0), n, F, gamma.data_ptr(), beta.data_ptr(), EPS, p,
                                          seed, offset, None if offset_dev is None else offset_dev.data_ptr(),
                                          y.data_ptr(), y.stride(0), mean.data_ptr(), rstd.data_ptr(), _stream()),
          "bns_ln_relu_dropout_fwd_f32")
    return y, mean, rstd


def ln_bwd(dy, x, gamma, beta, mean, rstd, p, seed, offset, offset_dev=None, dx=None):
    from bns_gcn_b200._lib import check, lib
    n, F = x.shape
    dx = torch.empty_like(x) if dx is None else dx
    dgamma = torch.full((F,), float("nan"), device=x.device)
    dbeta = torch.full((F,), float("nan"), device=x.device)
    ws = torch.empty(lib.bns_ln_bwd_workspace_bytes(F), dtype=torch.uint8, device=x.device)
    check(lib.bns_ln_relu_dropout_bwd_f32(dy.data_ptr(), dy.stride(0), x.data_ptr(), x.stride(0), n, F, gamma.data_ptr(),
                                          beta.data_ptr(), mean.data_ptr(), rstd.data_ptr(), EPS, p, seed, offset,
                                          None if offset_dev is None else offset_dev.data_ptr(), dx.data_ptr(),
                                          dx.stride(0), dgamma.data_ptr(), dbeta.data_ptr(), ws.data_ptr(), ws.numel(),
                                          _stream()), "bns_ln_relu_dropout_bwd_f32")
    return dx, dgamma, dbeta


def _strided(n, F, pad, fill=float("nan")):
    """``[n, F]`` view of an ``[n, F + pad]`` buffer filled with ``fill``."""
    return torch.full((n, F + pad), fill, device=_dev())[:, :F]


# ---- inputs -----------------------------------------------------------------------------------------------------------
def _inputs(n, F, seed, pad=0):
    """x (random rows of scales 1e-2 .. 1e2 and means up to 3 scales, plus the crafted rows), gamma, beta, dy.  Half
    of beta is ``-gamma * u`` for a standardised vector ``u``: rows that are affine images of ``u`` then have
    pre-activations at rounding distance from 0 in those columns, on either side."""
    dev = _dev()
    g = torch.Generator(device=dev).manual_seed(seed)
    scale = 10.0 ** (torch.rand(n, 1, generator=g, device=dev) * 4 - 2)
    x = (torch.randn(n, F, generator=g, device=dev) + (torch.rand(n, 1, generator=g, device=dev) * 6 - 3)) * scale
    gamma = (torch.rand(F, generator=g, device=dev) + 0.5) * torch.sign(torch.randn(F, generator=g, device=dev))
    u = torch.randn(F, generator=g, device=dev, dtype=torch.float64)
    u = ((u - u.mean()) / (u - u.mean()).pow(2).mean().sqrt()).float()
    beta = torch.randn(F, generator=g, device=dev) * 0.3
    beta[0::2] = -(gamma * u)[0::2]
    if n >= 7:
        for r in sorted({1, n // 2, n - 2}):
            x[r] = 0.3                                                          # var = 0: z = beta
        for r in sorted({2, n // 3, n - 1}):
            x[r] = 3000.0 + torch.randn(F, generator=g, device=dev)             # |mean| / std = 3000
        for k, r in enumerate(sorted({3, 4, 5, n // 5, n - 3})):
            x[r] = u * (0.5 + k) + (k - 2) * 1.7                                # z straddles 0 in the even columns
    dy = torch.randn(n, F, generator=g, device=dev)
    if pad:
        xs, dys = _strided(n, F, pad, 0.0), _strided(n, F, pad, 0.0)
        xs.copy_(x)
        dys.copy_(dy)
        x, dy = xs, dys
    return x, gamma, beta, dy


# ---- the float64 reference and the check ------------------------------------------------------------------------------
def _close(worst, label, name, got, want, bound):
    with contextlib.redirect_stdout(io.StringIO()):
        r = R.assert_close(f"{label} {name}", got, want, bound)
    worst[name] = max(worst.get(name, 0.0), r)


def check_ln(x, gamma, beta, dy, p, seed, offset, label, y=None, dx=None, offset_dev=None, mask_offset=None):
    """Run forward and backward, compare every element with float64.  The backward reference takes the kernel's own
    ReLU active set: where ``|z| <= TOL * bound`` either side is right, and every entry whose side differs from the
    reference's must lie there.  Returns the outputs and the worst ratio per tensor."""
    n, F = x.shape
    y, mean, rstd = ln_fwd(x, gamma, beta, p, seed, offset, offset_dev, y)
    dx, dgamma, dbeta = ln_bwd(dy, x, gamma, beta, mean, rstd, p, seed, offset, offset_dev, dx)
    moff = offset if mask_offset is None else mask_offset
    s = _keep_scale(p)
    gd, bd = gamma.double(), beta.double()
    sums = torch.zeros(4, F, dtype=torch.float64, device=x.device)       # dgamma, its bound, dbeta, its bound
    worst, flips = {}, 0
    chunk = max(1, (1 << 22) // F)
    for r0 in range(0, n, chunk):
        r1 = min(n, r0 + chunk)
        xd = x[r0:r1].double()
        xc = xd - xd.mean(1, keepdim=True)
        rs = ((xc * xc).mean(1, keepdim=True) + EPS).rsqrt()
        xh = xc * rs
        z = xh * gd + bd
        a = xh.abs() + rs * xd.abs().mean(1, keepdim=True)                  # the scale of x_hat's own rounding
        bz = gd.abs() * a + bd.abs()
        keep = keep_mask(seed, moff, r0, r1, F, p) if p > 0 else torch.ones_like(z, dtype=torch.bool)
        yk = y[r0:r1]
        act = (yk != 0) | ((z > 0) & ~keep)
        flip = (act != (z > 0)) & keep
        assert bool((z[flip].abs() <= R.TOL * bz[flip]).all()), \
            f"{label}: a ReLU side differs from float64 at |z| = {z[flip].abs().max().item()!r}, beyond the margin"
        flips += int(flip.sum())
        m = (act & keep).double() * s
        lab = f"{label} rows {r0}:{r1}"
        _close(worst, lab, "y", yk, z * m, bz * keep.double() * s)
        g = dy[r0:r1].double() * m
        gz = g * gd
        agz = gz.abs()
        want = rs * (gz - gz.mean(1, keepdim=True) - xh * (gz * xh).mean(1, keepdim=True))
        bound = rs * (agz + agz.mean(1, keepdim=True) + xh.abs() * (agz * a).mean(1, keepdim=True)
                      + a * (agz * xh.abs()).mean(1, keepdim=True))
        _close(worst, lab, "dx", dx[r0:r1], want, bound)
        sums += torch.stack([(g * xh).sum(0), (g.abs() * a).sum(0), g.sum(0), g.abs().sum(0)])
    _close(worst, label, "dgamma", dgamma, sums[0], sums[1])
    _close(worst, label, "dbeta", dbeta, sums[2], sums[3])
    for k, v in worst.items():
        print(f"[ratio] {label} {k}: {v:.3g}")
    print(f"[kinks] {label}: {flips} entries on the other side of the ReLU, all within the margin")
    return (y, dx, dgamma, dbeta), worst


def _outputs_written(label, t, F):
    """Columns ``< F`` finite, the padding past ``F`` still NaN."""
    full = t.as_strided((t.shape[0], t.stride(0)), (t.stride(0), 1))
    assert bool(torch.isfinite(full[:, :F]).all()), f"{label}: a written element is not finite"
    assert bool(torch.isnan(full[:, F:]).all()), f"{label}: a column past F was written"


# ---- tests ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", ROWS)
@pytest.mark.parametrize("F", WIDTHS)
def test_layernorm_relu_dropout_against_float64(built, F, rows):
    """Every width class at every row count, p = 0.5 (the benchmark's).  Below the benchmark's row count x / dy are
    strided (leading dimension F + 4) and y / dx too (F + 8), NaN-filled: the padding must stay NaN.  At 232,965 rows
    the operands are contiguous, as in the benchmark."""
    n = _n_rows(rows)
    pad = 0 if rows == "bench" else 4
    x, gamma, beta, dy = _inputs(n, F, seed=F * 7 + n, pad=pad)
    y = torch.full((n, F), float("nan"), device=_dev()) if pad == 0 else _strided(n, F, 8)
    dx = torch.full((n, F), float("nan"), device=_dev()) if pad == 0 else _strided(n, F, 8)
    (y, dx, dgamma, dbeta), _ = check_ln(x, gamma, beta, dy, 0.5, 0x1234, 3, f"F={F} n={n}", y=y, dx=dx)
    _outputs_written(f"F={F} n={n} y", y, F)
    _outputs_written(f"F={F} n={n} dx", dx, F)
    assert bool(torch.isfinite(dgamma).all() and torch.isfinite(dbeta).all())


@pytest.mark.parametrize("p", [0.0, 0.1, 0.5, 0.9])
@pytest.mark.parametrize("F", [128, 600])
def test_layernorm_dropout_rates_and_determinism(built, F, p):
    """p = 0, 0.1, 0.5, 0.9 at 64 SMs + 5 rows; the keep rate is 1 - p; a second backward is bit-identical."""
    n = _n_rows("64sm+5")
    x, gamma, beta, dy = _inputs(n, F, seed=11 + F, pad=4)
    (y, dx, dgamma, dbeta), _ = check_ln(x, gamma, beta, dy, p, 77, 5, f"F={F} p={p}")
    if p > 0:
        rate = keep_mask(77, 5, 0, n, F, p).float().mean().item()
        assert abs(rate - (1 - p)) < 0.005, rate
    y2, mean, rstd = ln_fwd(x, gamma, beta, p, 77, 5)
    dx2, dgamma2, dbeta2 = ln_bwd(dy, x, gamma, beta, mean, rstd, p, 77, 5)
    assert torch.equal(y2, y) and torch.equal(dx2, dx)
    assert torch.equal(dgamma2, dgamma) and torch.equal(dbeta2, dbeta)


def test_layernorm_zero_rows_is_a_no_op(built):
    """n = 0: the forward writes nothing; the backward writes dgamma = dbeta = 0 and leaves dx alone."""
    F = 256
    x, gamma, beta, dy = _inputs(4, F, seed=1)
    y = torch.full_like(x, float("nan"))
    mean, rstd = torch.full((4,), -7.0, device=_dev()), torch.full((4,), -7.0, device=_dev())
    from bns_gcn_b200._lib import check, lib
    check(lib.bns_ln_relu_dropout_fwd_f32(x.data_ptr(), F, 0, F, gamma.data_ptr(), beta.data_ptr(), EPS, 0.5, 1, 0, None,
                                          y.data_ptr(), F, mean.data_ptr(), rstd.data_ptr(), _stream()), "fwd")
    dx = torch.full_like(x, float("nan"))
    dgamma, dbeta = torch.full((F,), float("nan"), device=_dev()), torch.full((F,), float("nan"), device=_dev())
    ws = torch.empty(lib.bns_ln_bwd_workspace_bytes(F), dtype=torch.uint8, device=_dev())
    check(lib.bns_ln_relu_dropout_bwd_f32(dy.data_ptr(), F, x.data_ptr(), F, 0, F, gamma.data_ptr(), beta.data_ptr(),
                                          mean.data_ptr(), rstd.data_ptr(), EPS, 0.5, 1, 0, None, dx.data_ptr(), F,
                                          dgamma.data_ptr(), dbeta.data_ptr(), ws.data_ptr(), ws.numel(), _stream()),
          "bwd")
    torch.cuda.synchronize()
    assert bool(torch.isnan(y).all() and torch.isnan(dx).all())
    assert bool((mean == -7).all() and (rstd == -7).all())
    assert bool((dgamma == 0).all() and (dbeta == 0).all())


def test_torch_philox_equals_oracle_philox(built):
    """The GPU restatement the big references use is the numpy one of oracle/philox.py, bit for bit."""
    from oracle.philox import philox4x32_10
    rng = np.random.default_rng(0)
    c = rng.integers(0, 2 ** 32, size=(4, 100_000), dtype=np.uint64).astype(np.uint32)
    for k0, k1 in [(0, 0), (MASK32, MASK32), (0x12345678, 0x9ABCDEF0)]:
        want = philox4x32_10(*c, k0, k1)
        got = philox_torch(*(torch.from_numpy(ci.astype(np.int64)).to(_dev()) for ci in c), k0, k1)
        for w, g in zip(want, got):
            assert np.array_equal(w.astype(np.int64), g.cpu().numpy())
    for seed, off, F in [(3, 9, 600), (2 ** 40 + 3, 2 ** 33 + 1, 1204)]:
        assert torch.equal(keep_mask(seed, off, 0, 50, F, 0.3).cpu(), keep_mask_np(seed, off, 50, F, 0.3))


# (seed, offset, offset_dev, effective offset): seeds at and above 2^32, offsets across 2^32, the graph-replay wrap
MASK_CASES = [
    (2 ** 32, 7, None, 7),
    (2 ** 63 + 0x5DEECE66D, 2 ** 32 + 5, None, 2 ** 32 + 5),
    (123, 2 ** 32 - 1, 2, 2 ** 32 + 1),
    (2 ** 32 + 9, 2 ** 64 - 1, 1, 0),
    (2 ** 32 + 9, 2 ** 64 - 1, 3, 2),
]


@pytest.mark.parametrize("seed,offset,dev_add,eff", MASK_CASES)
def test_masks_equal_numpy_replay(built, seed, offset, dev_add, eff):
    """The forward's mask (gamma = 0, beta = 1: z = 1 everywhere, so y != 0 is the mask) and bns_dropout_f32's mask
    (dropout of ones) equal the numpy replay exactly, as does the forward / backward at that offset against float64.
    ``offset = 2**64 - 1`` with ``*offset_dev = e + 1`` is epoch ``e`` of a replayed CUDA graph."""
    from bns_gcn_b200._lib import check, lib
    dev = _dev()
    off_dev = None if dev_add is None else torch.tensor([dev_add], dtype=torch.int64, device=dev)
    p = 0.5
    for F, n in [(600, 300), (132, 700)]:
        want = keep_mask_np(seed, eff, n, F, p)
        x = torch.randn(n, F, device=dev)
        y, _, _ = ln_fwd(x, torch.zeros(F, device=dev), torch.ones(F, device=dev), p, seed, offset, off_dev)
        assert torch.equal((y != 0).cpu(), want), ("ln", F)
        y_imm, _, _ = ln_fwd(x, torch.zeros(F, device=dev), torch.ones(F, device=dev), p, seed, eff)
        assert torch.equal(y, y_imm)
        d = torch.empty(n, F, device=dev)
        check(lib.bns_dropout_f32(torch.ones(n, F, device=dev).data_ptr(), F, n, F, p, seed, offset,
                                  None if off_dev is None else off_dev.data_ptr(), d.data_ptr(), F, _stream()), "drop")
        assert torch.equal((d != 0).cpu(), want), ("dropout", F)
    x, gamma, beta, dy = _inputs(n, F, seed=5)
    check_ln(x, gamma, beta, dy, p, seed, offset, f"seed={seed:#x} offset={offset:#x}+{dev_add}", offset_dev=off_dev,
             mask_offset=eff)


@pytest.mark.parametrize("F", [1204, 604])
def test_dropout_f32_against_replay(built, F):
    """``bns_dropout_f32`` (layer 0's input dropout): strided operands, y = x * mask * (1 / (1 - p)) exactly (one
    multiply), the padding untouched; through ``fused.DropoutFn`` the backward applies the same mask to dy even after
    the RNG offset has moved on."""
    from bns_gcn_b200 import fused, ops
    from bns_gcn_b200._lib import check, lib
    dev = _dev()
    n, p, seed, off = _n_rows("32sm+1"), 0.5, 104729 + 3, 2 ** 32 + 17
    want = keep_mask_np(seed, off, n, F, p).to(dev)
    ks = torch.tensor(_keep_scale(p), dtype=torch.float32, device=dev)
    x = _strided(n, F, 8, 0.0)
    x.copy_(torch.randn(n, F, device=dev))
    y = _strided(n, F, 4)
    check(lib.bns_dropout_f32(x.data_ptr(), x.stride(0), n, F, p, seed, off, None, y.data_ptr(), y.stride(0),
                              _stream()), "bns_dropout_f32")
    _outputs_written(f"dropout F={F}", y, F)
    assert torch.equal(y, torch.where(want, x * ks, torch.zeros_like(x)))
    ops.RNG.update(seed=0, offset=off, offset_dev=None)
    try:
        xl = x.contiguous().requires_grad_(True)
        yl = fused.DropoutFn.apply(xl, p, seed)
        ops.RNG.update(offset=off + 1)
        dy = torch.randn(n, F, device=dev)
        yl.backward(dy)
    finally:
        ops.RNG.update(seed=0, offset=0, offset_dev=None)
    assert torch.equal(yl.detach(), torch.where(want, x * ks, torch.zeros_like(x)))
    assert torch.equal(xl.grad, torch.where(want, dy * ks, torch.zeros_like(dy)))


def test_model_dropout_streams_are_independent(built, monkeypatch):
    """The benchmark's model (3-layer GraphSAGE, --use-pp, LayerNorm, dropout 0.5) at 8 ranks for 3 epochs: every
    forward draws its masks from (model seed * 1000003 + rank + salt, epoch), with salt 104729 (i + 1) for layer 0's
    input and 7919 (i + 1) for the LayerNorm after layer i.  Any two of the 72 streams agree on 50 % +- 0.5 % of a
    common [20000, 256] region at p = 0.5."""
    import threading
    from bns_gcn_b200 import train
    from bns_gcn_b200._lib import lib
    from bns_gcn_b200.data import make_graph, partition_graph
    from bns_gcn_b200.helper.comm import run_threads
    from tests.harness import make_args
    P, E, SEED = 8, 3, 5
    tls, calls = threading.local(), []
    for name, pos in (("bns_ln_relu_dropout_fwd_f32", 7), ("bns_dropout_f32", 4)):
        fn = getattr(lib, name)

        def rec(*a, fn=fn, name=name, pos=pos):
            if getattr(tls, "fwd", False) and a[pos] > 0:
                calls.append((tls.rank, tls.epoch, name, a[pos + 1], a[pos + 2], a[pos + 3]))
            return fn(*a)
        monkeypatch.setattr(lib, name, rec)
    fg = make_graph("small", seed=0)
    parts = partition_graph(fg, P, "random", seed=0)
    args = make_args(dataset="small", n_hidden=16, sampling_rate=0.5, dropout=0.5, seed=SEED, n_partitions=P)

    def fn(comm, r):
        import argparse
        pt = parts[r]
        a = argparse.Namespace(**vars(args))
        a.n_feat, a.n_class, a.n_train = pt.meta["n_feat"], pt.meta["n_class"], pt.meta["n_train"]
        st = train.setup(pt.graph, pt.node_dict, pt.gpb, a, "cuda:0")
        assert st.arena is not None, "the fused training step was not taken"
        st.model.register_forward_pre_hook(lambda *_: setattr(tls, "fwd", True))
        st.model.register_forward_hook(lambda *_: setattr(tls, "fwd", False))
        tls.rank = r
        for e in range(E):
            tls.epoch = e
            train.train_epoch(st, e)
    run_threads(P, fn, device="cuda:0")
    want = set()
    for r in range(P):
        for e in range(E):
            base = SEED * 1000003 + r
            want |= {(r, e, "bns_dropout_f32", base + 104729, e, None),
                     (r, e, "bns_ln_relu_dropout_fwd_f32", base + 7919, e, None),
                     (r, e, "bns_ln_relu_dropout_fwd_f32", base + 7919 * 2, e, None)}
    assert len(calls) == len(want) == P * E * 3 and set(calls) == want, sorted(set(calls) ^ want)[:6]
    signs = torch.stack([keep_mask(c[3], c[4], 0, 20000, 256, 0.5).reshape(-1).float() * 2 - 1 for c in calls])
    agree = ((signs @ signs.t()) / signs.shape[1] + 1) / 2
    off_diag = agree[~torch.eye(len(calls), dtype=torch.bool, device=agree.device)]
    print(f"[streams] {len(calls)} streams, pairwise agreement {off_diag.min().item():.4f} .. {off_diag.max().item():.4f}")
    assert bool(((off_diag - 0.5).abs() <= 0.005).all())


def test_layernorm_entry_points_reject_bad_arguments(built):
    """p = 1, leading dimensions below F, F = 1028, F = 6 and misaligned x / gamma / dx are answered with BNS_E_INVALID
    and a message naming the entry point, before anything is launched."""
    from bns_gcn_b200._lib import lib
    dev = _dev()
    LD, n = 1040, 2
    x, dy, y, dx = (torch.zeros(n, LD, device=dev) for _ in range(4))
    gamma, beta, mean, rstd, dg, db = (torch.zeros(LD, device=dev) for _ in range(6))
    ws = torch.empty(lib.bns_ln_bwd_workspace_bytes(1024), dtype=torch.uint8, device=dev)

    def fwd(F=256, p=0.5, ldx=LD, xo=0, go=0):
        return lib.bns_ln_relu_dropout_fwd_f32(x.data_ptr() + xo, ldx, n, F, gamma.data_ptr() + go, beta.data_ptr(),
                                               EPS, p, 1, 0, None, y.data_ptr(), LD, mean.data_ptr(), rstd.data_ptr(),
                                               _stream())

    def bwd(F=256, p=0.5, ldx=LD, lddx=LD, xo=0, go=0, dxo=0):
        return lib.bns_ln_relu_dropout_bwd_f32(dy.data_ptr(), LD, x.data_ptr() + xo, ldx, n, F, gamma.data_ptr() + go,
                                               beta.data_ptr(), mean.data_ptr(), rstd.data_ptr(), EPS, p, 1, 0, None,
                                               dx.data_ptr() + dxo, lddx, dg.data_ptr(), db.data_ptr(), ws.data_ptr(),
                                               ws.numel(), _stream())

    bad = {fwd: [dict(p=1.0), dict(ldx=252), dict(F=1028), dict(F=6), dict(xo=4), dict(go=4)],
           bwd: [dict(p=1.0), dict(ldx=252), dict(lddx=252), dict(F=1028), dict(F=6), dict(xo=4), dict(go=4),
                 dict(dxo=4)]}
    for fn, cases in bad.items():
        name = {fwd: b"bns_ln_relu_dropout_fwd_f32", bwd: b"bns_ln_relu_dropout_bwd_f32"}[fn]
        assert fn() == 0, name
        for kw in cases:
            assert fn(**kw) == -1 and name in lib.bns_last_error(), (name, kw)
    torch.cuda.synchronize()


def test_cuda_graph_epoch_with_dropout_equals_eager(built):
    """train.GraphedEpoch with the benchmark's model (3-layer GraphSAGE, hidden 256, --use-pp, LayerNorm, dropout 0.5,
    fused step) on the 6,000-row partition of the ``small`` shape: 2 eager epochs, then 3 replays, whose masks take their
    offset from ``2**64 - 1 + epoch_dev``, against 5 eager epochs."""
    from tests.harness import make_args
    from bns_gcn_b200 import train
    from bns_gcn_b200.data import make_graph, partition_graph
    from bns_gcn_b200.helper import context as ctx
    dev = _dev()
    fg = make_graph("small", seed=0)
    part = partition_graph(fg, 1, "random", seed=0)[0]

    def fresh():
        ctx.reset()
        a = make_args(dataset="small", model="graphsage", n_hidden=256, dropout=0.5)
        a.n_feat, a.n_class, a.n_train = part.meta["n_feat"], part.meta["n_class"], part.meta["n_train"]
        st = train.setup(part.graph, part.node_dict, part.gpb, a, dev)
        assert st.arena is not None and st.model.dropout.p == 0.5
        return st
    prev = torch.autograd.is_multithreading_enabled()
    torch.autograd.set_multithreading_enabled(False)
    prev_stream = torch.cuda.current_stream(dev)
    torch.cuda.set_stream(torch.cuda.Stream(dev))
    try:
        st = fresh()
        eager = [train.train_epoch(st, e).item() for e in range(5)]
        w_eager = [p.detach().clone() for p in st.model.parameters()]
        st = fresh()
        ge = train.GraphedEpoch(st, warmup=2)
        replay = [ge().item() for _ in range(3)]
        w_graph = [p.detach().clone() for p in st.model.parameters()]
    finally:
        torch.cuda.synchronize(dev)
        torch.cuda.set_stream(prev_stream)
        torch.autograd.set_multithreading_enabled(prev)
        ctx.reset()
    same = replay == eager[2:] and all(torch.equal(a, b) for a, b in zip(w_graph, w_eager))
    print(f"[graph] losses eager {eager[2:]} replay {replay}; bit-identical: {same}")
    for a_, b_ in zip(replay, eager[2:]):
        assert abs(a_ - b_) <= 1e-6 * abs(b_), (replay, eager)
    for a_, b_ in zip(w_graph, w_eager):
        assert ((a_ - b_).norm() / b_.norm()).item() <= 1e-6
