"""Host restatement of the FP8 projections (include/lade_sm100.h, lade_gemm_fp8 / lade_quant_rows_fp8).

* ``quant_rows``: the e4m3 row quantiser, bit for bit: amax = max |x| (fp32), s = fp32(amax / 448) (1 when amax is 0 or
  not finite), q = e4m3(fp32(x / s)), round to nearest even, saturated to +-448.
* ``linear64``: the exact value of the FP8 linear from the dequantised operands, in float64.
* ``emulate_kernel``: the kernel's fp32 accumulation order: each 128-deep k-block summed exactly (the tensor cores'
  product of two e4m3 values is exact in fp32) then rounded once to fp32 -- the promotion -- and added into an fp32
  accumulator; K splits summed in split order; then the two scale multiplies and the rounding to T.
* ``bound``: the error bound the GPU result is held to against ``linear64``.
"""
import numpy as np
import torch

E4M3_MAX = 448.0
BK = 128


def row_scale(amax: torch.Tensor) -> torch.Tensor:
    """fp32 scales of fp32 row maxima."""
    amax = amax.float()
    ok = torch.isfinite(amax) & (amax > 0)
    return torch.where(ok, amax / torch.tensor(E4M3_MAX, dtype=torch.float32), torch.ones_like(amax))


def quant_rows(x: torch.Tensor):
    """(q uint8 [rows, cols], s float32 [rows]) of a [rows, cols] tensor (any float dtype: its values are used as is)."""
    xf = x.float()
    s = row_scale(xf.abs().amax(dim=1))
    y = (xf / s[:, None]).clamp(-E4M3_MAX, E4M3_MAX)
    q = y.to(torch.float8_e4m3fn).view(torch.uint8)
    return q, s


def dequant(q: torch.Tensor) -> torch.Tensor:
    """float64 values of e4m3 bytes."""
    return q.view(torch.float8_e4m3fn).to(torch.float64)


def linear64(qa, sa, qw, sw) -> torch.Tensor:
    """Exact (float64) c[r][n] = (sum_k a[r][k] w[n][k]) * sa[r] * sw[n]; the sums of e4m3 products are exact in
    float64 for K <= 2^20."""
    return (dequant(qa) @ dequant(qw).T) * sa.double()[:, None] * sw.double()[None, :]


def emulate_kernel(qa, sa, qw, sw, split_k: int = 1, out_dtype=torch.bfloat16, promote: bool = True,
                   drop_block: int = -1):
    """The kernel's rounding points in order (fp32 block sums, fp32 accumulation, split order, two scale multiplies,
    one rounding to T).  `promote=False` models a kernel that keeps one tensor-core accumulator over all of K at
    about 14 bits (the DeepSeek-V3 report's measurement of Hopper's fp8 accumulation): each block is added into the
    running sum rounded to 13 mantissa bits.  `drop_block` skips that k-block (a planted error)."""
    a, w = dequant(qa), dequant(qw)
    K = a.shape[1]
    nkb = K // BK
    per = nkb // split_k
    parts = []
    for p in range(split_k):
        acc = torch.zeros(a.shape[0], w.shape[0], dtype=torch.float32)
        for kb in range(p * per, (p + 1) * per):
            if kb == drop_block:
                continue
            blk = a[:, kb * BK:(kb + 1) * BK] @ w[:, kb * BK:(kb + 1) * BK].T        # exact in float64
            if promote:
                acc = acc + blk.float()
            else:
                acc = round_mantissa((acc.double() + blk), 13).float()
        parts.append(acc)
    tot = parts[0]
    for p in parts[1:]:
        tot = tot + p
    c = (tot * sa.float()[:, None]) * sw.float()[None, :]
    return c.to(out_dtype)


def round_mantissa(x: torch.Tensor, bits: int) -> torch.Tensor:
    """x rounded to `bits` explicit mantissa bits (round to nearest)."""
    m, e = torch.frexp(x)
    scale = 2.0 ** (bits + 1)
    return torch.ldexp(torch.round(m * scale) / scale, e)


def bound(qa, sa, qw, sw, out_dtype=torch.bfloat16, split_k: int = 8) -> torch.Tensor:
    """|c - linear64| <= bound, elementwise.  Inside a 128-deep block the tensor cores do not accumulate in full fp32:
    on the H100 the per-block error reaches about 2^-16 of sum |a w| (DESIGN.md §6), consistent with the ~14-bit
    accumulator the DeepSeek-V3 report describes; the bound allows one 14-bit rounding, 2^-13 * sum |a w| * sa * sw,
    plus the fp32 additions of the K / 128 promoted block sums and split_k partials, plus the final rounding to T
    (2^-8 (bf16) / 2^-11 (fp16) of the value)."""
    mag = (dequant(qa).abs() @ dequant(qw).abs().T) * sa.double()[:, None] * sw.double()[None, :]
    K = qa.shape[1]
    acc = (2.0 ** -13 + (K // BK + split_k + 2) * 2.0 ** -24) * mag
    ref = linear64(qa, sa, qw, sw).abs()
    rel = 2.0 ** -8 if out_dtype == torch.bfloat16 else 2.0 ** -11
    tiny = 2.0 ** -133 if out_dtype == torch.bfloat16 else 2.0 ** -24
    return acc * (1 + rel) + rel * (ref + acc) + tiny


def bits_equal(a: torch.Tensor, b: torch.Tensor) -> bool:
    return bool(torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8)))


def np_e4m3_table():
    """All 256 e4m3fn values (NaN at 0x7f / 0xff) as float64."""
    return torch.arange(256, dtype=torch.int32).to(torch.uint8).view(torch.float8_e4m3fn).to(torch.float64).numpy()


__all__ = ["quant_rows", "row_scale", "dequant", "linear64", "emulate_kernel", "bound", "bits_equal", "np_e4m3_table", "round_mantissa", "np"]
