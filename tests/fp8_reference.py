"""The fp8 gather-table format of ``--agg-dtype fp8``, restated on the host: the reference every fp8 test compares with.

For each row x of F columns, m = max |x_i|:
  * scale s = 2^e, e the smallest integer with m * 2^-e <= 448 (the largest finite e4m3), clamped to e >= -126 so that s
    is a normal f32; a row of zeros gets s = 1;
  * codes q_i = x_i * 2^-e (an f32 product, exact: a power of two, never above 448) rounded to nearest even e4m3 by
    torch's conversion (which keeps subnormal codes and maps -0.0 to 0x80);
  * a row holding NaN or +-Inf gets s = NaN and all-zero codes, so every sum that gathers it is NaN.
"""
import torch

E4M3_MAX = 448.0


def scale_exponents(x: torch.Tensor):
    """``(e, bad)`` per row of the f32 matrix ``x``: the exponent of the row's scale and whether the row is not finite."""
    a = x.double().abs()
    bad = ~torch.isfinite(a).all(1)
    m = torch.where(torch.isfinite(a), a, torch.zeros_like(a)).amax(1) if a.shape[1] else a.new_zeros(a.shape[0])
    mant, k = torch.frexp(m)                               # m = mant * 2^k, mant in [0.5, 1)
    e = torch.where(mant <= E4M3_MAX / 512.0, k - 9, k - 8).long()
    e = torch.where(m == 0, torch.zeros_like(e), e.clamp(min=-126))
    return e, bad


def quantize_rows(x: torch.Tensor):
    """``(codes [n, F] float8_e4m3fn, scale [n] f32)`` of the f32 matrix ``x`` (on any device)."""
    x = x.float()
    e, bad = scale_exponents(x)
    inv = torch.ldexp(torch.ones_like(e, dtype=torch.float32), -e)
    codes = torch.where(bad.unsqueeze(1), torch.zeros_like(x), x * inv.unsqueeze(1)).to(torch.float8_e4m3fn)
    scale = torch.ldexp(torch.ones_like(e, dtype=torch.float32), e)
    scale[bad] = float("nan")
    return codes, scale


def dequantize(codes: torch.Tensor, scale: torch.Tensor) -> torch.Tensor:
    """The f64 values a table stands for (exact: every code times a power of two is an f64)."""
    return codes.double() * scale.double().unsqueeze(1)
