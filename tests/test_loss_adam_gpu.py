"""The loss kernel (``bns_xent_f32`` through ``fused.softmax_xent``: sum-reduced cross-entropy and BCE-with-logits
over the masked rows, and d(logits)) and the fused Adam step (``bns_adam_step_f32`` through ``fused.FusedAdam``)
against float64, element by element, with ``layer_reference.assert_close``.

Cross-entropy, per masked row with maximum ``m``, softmax sum ``s = sum_c exp(x_c - m)`` and label ``y``:
  d(logits)  ref = (p_c - [c == y]) * scale,  bound = (p_c + [c == y]) * |scale|.  The kernel forms ``p_c`` as
             ``expf(x_c - m) / s`` (a few roundings relative to ``p_c``: ``x_c - m`` is exact wherever ``exp`` does not
             underflow) and subtracts 1 at the label, where the difference cancels: its rounding is relative to
             ``p_c + 1``.
  loss       ref = sum_rows (m + log s - x_y),  bound = sum_rows (|m| + log s + |x_y|).  The kernel rounds ``m + log s``
             and then subtracts ``x_y``: each step's error is relative to the magnitudes it adds; ``log s >= 0``
             carries the error of ``s`` (relative to ``s``, absolute in ``log s``); the sums over the rows of a warp,
             the warps of a block and the blocks add terms that are all ``>= 0``.
BCE-with-logits, per masked element with target ``t``:
  d(logits)  ref = (sigmoid(x) - t) * scale, bound = (sigmoid(x) + |t|) * |scale| (the same cancellation as above).
  loss       ref = sum (max(x, 0) - x t + log1p(exp(-|x|))), bound = sum (max(x, 0) + |x t| + log1p(exp(-|x|))):
             the three terms are each rounded relative to their own magnitude, then added.
Unmasked rows and the pad columns must be exactly 0.  Logits are views into wider NaN-filled buffers (pad columns
included): a read outside the ``n_class`` real columns turns the result NaN.

Adam: each step is restated in float64 from the kernel's own f32 state before that step, so error cannot compound.
The restatement uses the f32 values of lr, beta1, beta2, eps and weight_decay that the C ABI receives (torch.optim.Adam
uses the double ones; for beta2 = 0.999, the f32 ``1 - beta2`` is 1.3e-5 relative away from torch's 0.001, a
difference of the call's arguments that ``test_kernels_gpu`` compares with torch itself):
  exp_avg     bound = |m| + (1 - b1) (|g| + wd |p| + |m|)
  exp_avg_sq  bound = b2 v + (1 - b2) (|g| + wd |p|)^2                  (no cancellation: every term is >= 0)
  param       bound = lr / bc1 * bound(exp_avg) / denom + |p'| 2^-23 / TOL
where ``denom = sqrt(v') / sqrt(bc2) + eps``: the update is relative to the exp_avg it divides, and the last term is
one ulp of ``p' = p - update`` in f32, expressed in units of ``TOL``.  The kernel rounds ``p'`` once (half an ulp);
where the update is far below an ulp of ``p`` that rounding is the whole error, which a bound of half an ulp would
meet with a ratio of 1.  Measured on an H100 80GB HBM3 at 700 W: ratio 0.997 against half an ulp."""
import contextlib
import io

import numpy as np
import pytest
import torch

from tests import layer_reference as R

pytestmark = pytest.mark.gpu

BENCH_ROWS = 232_965            # inner nodes of the benchmark's single partition (Reddit shape)


def _dev():
    return torch.device("cuda:0")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _ceil4(n):
    return (n + 3) // 4 * 4


def _gen(seed):
    return torch.Generator(device=_dev()).manual_seed(seed)


def _close(worst, key, label, got, want, bound):
    with contextlib.redirect_stdout(io.StringIO()):
        r = R.assert_close(label, got, want, bound)
    worst[key] = max(worst.get(key, 0.0), r)


def _report(worst):
    for k, v in worst.items():
        print(f"[ratio] {k}: {v:.3g}")


def _mask(kind, n, g):
    if kind == "absent":
        return None
    if kind == "all":
        return torch.ones(n, dtype=torch.bool, device=_dev())
    if kind == "none":
        return torch.zeros(n, dtype=torch.bool, device=_dev())
    return torch.rand(n, generator=g, device=_dev()) < 0.6


def _logits(n, C, mag, g):
    """``[n, ceil4(C)]`` view of a NaN-filled ``[n + 2, ceil4(C) + 4]`` buffer; columns ``[C, ceil4(C))`` stay NaN."""
    buf = torch.full((n + 2, _ceil4(C) + 4), float("nan"), device=_dev())
    x = buf[:n, :_ceil4(C)]
    x[:, :C] = torch.randn(n, C, generator=g, device=_dev()) * mag
    return x


# ---- cross-entropy ------------------------------------------------------------------------------------------------
def _xent_case(fused, worst, key, n, C, mag, mask_kind, seed, scale=1.0 / 777.0):
    g = _gen(seed)
    x = _logits(n, C, mag, g)
    lbuf = torch.randint(0, C, (n + 4,), generator=g, device=_dev())
    labels = lbuf[:n]
    if n >= 3:
        x[0, :C] = x[0, 0].item()                              # all logits equal
        labels[1] = torch.argmax(x[1, :C])                     # label at the row maximum
        labels[2] = torch.argmin(x[2, :C])                     # label at the row minimum
    mask = _mask(mask_kind, n, g)
    loss, dl = fused.softmax_xent(x, C, labels, mask, scale)
    label = f"xent (rows, C, |x|, mask) = ({n}, {C}, {mag:g}, {mask_kind})"
    on = torch.ones(n, dtype=torch.bool, device=_dev()) if mask is None else mask
    assert dl.shape == x.shape
    assert bool((dl[~on] == 0).all()) and bool((dl[:, C:] == 0).all()), f"{label}: pad or unmasked entry not 0"
    xd = x[on, :C].double()
    lab = labels[on]
    m = xd.max(1).values
    s = torch.exp(xd - m[:, None]).sum(1)
    logp = xd - m[:, None] - torch.log(s)[:, None]
    p = torch.exp(logp)
    hot = torch.nn.functional.one_hot(lab, C).double()
    if p.numel():
        _close(worst, key + " dlogits", label, dl[on, :C], (p - hot) * scale, (p + hot) * abs(scale))
    xl = xd.gather(1, lab[:, None])[:, 0]
    want = -logp.gather(1, lab[:, None])[:, 0].sum()
    bound = (m.abs() + torch.log(s) + xl.abs()).sum()
    _close(worst, key + " loss", label, loss.reshape(1), want.reshape(1), bound.reshape(1))
    if mask_kind == "none" or n == 0:
        assert loss.item() == 0.0 and bool((dl == 0).all()), label
    return loss


def test_xent_sweep(built):
    """rows x classes x logit magnitude, the mask cycling through absent / all / none / 60 %.  The benchmark's row
    count makes every warp walk about 55 rows (the grid is capped at 4 blocks of 8 warps per SM)."""
    from bns_gcn_b200 import fused
    assert _sms() * 4 * 8 < BENCH_ROWS, "the grid cap is not reached: one row per warp"
    worst = {}
    i = 0
    for n in (0, 1, 33, 4096, BENCH_ROWS):
        for C in (1, 2, 41, 47, 100):
            for mag in (1.0, 80.0, 1e4):
                _xent_case(fused, worst, "xent", n, C, mag, ("absent", "all", "none", "60%")[i % 4], seed=i)
                i += 1
    for kind in ("absent", "all", "none", "60%"):
        _xent_case(fused, worst, "xent", BENCH_ROWS, 41, 3.0, kind, seed=100 + i)
        i += 1
    _report(worst)


def test_xent_ticket_rearms_across_launch_sizes(built):
    """A small, a large and a small launch back to back on one stream: the completion ticket re-arms each time, and
    each loss is bit-identical when repeated."""
    from bns_gcn_b200 import fused
    worst = {}
    runs = [(64, 41), (BENCH_ROWS, 41), (64, 41), (BENCH_ROWS, 41), (64, 41)]
    losses = [_xent_case(fused, worst, "xent sequence", n, C, 3.0, "60%", seed=n) for n, C in runs]
    bits = [np.float32(l.item()).view(np.uint32) for l in losses]
    assert bits[0] == bits[2] == bits[4] and bits[1] == bits[3], [l.item() for l in losses]
    _report(worst)


# ---- BCE with logits ----------------------------------------------------------------------------------------------
def _bce_case(fused, worst, n, mask_kind, seed, scale=0.5):
    C = 100
    g = _gen(seed)
    x = _logits(n, C, 1.0, g)
    x[:, :C] = (torch.rand(n, C, generator=g, device=_dev()) * 2 - 1) * 100   # logits up to +-100
    tbuf = torch.full((n + 2, C + 4), float("nan"), device=_dev())
    t = tbuf[:n, :C]
    t.copy_((torch.rand(n, C, generator=g, device=_dev()) < 0.04).float())     # sparse multi-label targets (Yelp-like)
    mask = _mask(mask_kind, n, g)
    loss, dl = fused.softmax_xent(x, C, t, mask, scale)
    label = f"bce (rows, C, mask) = ({n}, {C}, {mask_kind})"
    on = torch.ones(n, dtype=torch.bool, device=_dev()) if mask is None else mask
    assert bool((dl[~on] == 0).all()), f"{label}: unmasked entry not 0"
    xd, td = x[on, :C].double(), t[on].double()
    sig = torch.sigmoid(xd)
    if sig.numel():
        _close(worst, "bce dlogits", label, dl[on, :C], (sig - td) * scale, (sig + td.abs()) * abs(scale))
    soft = torch.log1p(torch.exp(-xd.abs()))
    want = (xd.clamp_min(0) - xd * td + soft).sum()
    bound = (xd.clamp_min(0) + (xd * td).abs() + soft).sum()
    _close(worst, "bce loss", label, loss.reshape(1), want.reshape(1), bound.reshape(1))
    if mask_kind == "none":
        assert loss.item() == 0.0 and bool((dl == 0).all()), label


def test_bce(built):
    from bns_gcn_b200 import fused
    worst = {}
    i = 0
    for n in (1, 33, 4096, BENCH_ROWS):
        for kind in ("absent", "all", "none", "60%"):
            _bce_case(fused, worst, n, kind, seed=i)
            i += 1
    _report(worst)


# ---- Adam ---------------------------------------------------------------------------------------------------------
def _f32(v):
    return float(np.float32(v))


def test_adam_step_against_float64(built):
    """One step at a time over an arena of more than 1.1 M floats (beyond one float4 per thread of the capped grid, so
    the grid-stride loop runs), gradients of magnitude 0, 1e-12, 1e-4, 1 and 1e3, weight decay 0 and 5e-4, step
    counters 0, 1, 2 (consecutive), 1000 and 2^31 + 5 (set in step_dev).  Padded slots stay 0 and step_dev advances
    by one per step."""
    from bns_gcn_b200 import fused
    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Linear(1204, 1001), torch.nn.Linear(1001, 41)).to(_dev())
    arena = fused.ParamArena(net)
    assert arena.total > _sms() * 8 * 256 * 4, "the arena fits one pass of the grid"
    real = torch.zeros(arena.total, dtype=torch.bool, device=_dev())
    for o, n, _ in arena.slots.values():
        real[o:o + n] = True
    lr, b1, b2, eps = 1e-2, 0.9, 0.999, 1e-8
    worst = {}
    for wd in (0.0, 5e-4):
        opt = fused.FusedAdam(arena, lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd)
        with torch.no_grad():
            arena.flat_p.zero_()
            arena.exp_avg.zero_()
            arena.exp_avg_sq.zero_()
            arena.flat_p[real] = torch.randn(int(real.sum()), device=_dev()) * 0.05
        L, B1, B2, E, W = (_f32(v) for v in (lr, b1, b2, eps, wd))
        for j, step in enumerate((0, 1, 2, 1000, 2 ** 31 + 5)):
            g = _gen(j + (100 if wd else 0))
            n = int(real.sum())
            mag = torch.tensor([0.0, 1e-12, 1e-4, 1.0, 1e3], device=_dev())[torch.randint(0, 5, (n,), generator=g,
                                                                                         device=_dev())]
            with torch.no_grad():
                arena.flat_g.zero_()
                arena.flat_g[real] = torch.randn(n, generator=g, device=_dev()) * mag
            if int(opt.step_dev.item()) != step:
                opt.step_dev.fill_(step)
            p, gr, m, v = (t.double().clone() for t in (arena.flat_p, arena.flat_g, arena.exp_avg, arena.exp_avg_sq))
            opt.step()
            assert int(opt.step_dev.item()) == step + 1
            t = step + 1
            grd = gr + W * p
            gmag = gr.abs() + W * p.abs()
            m1 = m + (1 - B1) * (grd - m)
            v1 = B2 * v + (1 - B2) * grd * grd
            bc1, bc2 = 1 - B1 ** t, 1 - B2 ** t
            denom = v1.sqrt() / bc2 ** 0.5 + E
            p1 = p - (L / bc1) * m1 / denom
            bm = m.abs() + (1 - B1) * (gmag + m.abs())
            bv = B2 * v + (1 - B2) * gmag * gmag
            bp = (L / bc1) * bm / denom + p1.abs() * (2.0 ** -23 / R.TOL)
            label = f"adam step {step} wd {wd:g}"
            _close(worst, "adam exp_avg", label, arena.exp_avg, m1, bm)
            _close(worst, "adam exp_avg_sq", label, arena.exp_avg_sq, v1, bv)
            _close(worst, "adam param", label, arena.flat_p, p1, bp)
            for name, tt in (("param", arena.flat_p), ("exp_avg", arena.exp_avg), ("exp_avg_sq", arena.exp_avg_sq)):
                assert bool((tt[~real] == 0).all()), f"{label}: a padded slot of {name} moved"
    _report(worst)
