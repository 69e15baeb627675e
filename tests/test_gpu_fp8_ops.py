"""The quantising glue kernels (lade_rmsnorm_quant_fp8 with and without the residual, lade_swiglu_quant_fp8,
lade_quant_rows_fp8), bf16 and fp16: the e4m3 bytes and the fp32 scales are bit-exact against the host quantiser
(tests/fp8_restatement.py) applied to the row the existing kernel (lade_rmsnorm / lade_swiglu) produces.  Zero rows,
one huge element, fp16 rows of +-60000, rows in the e4m3 subnormal range; widths 4096 .. 14336; 1 .. 1024 rows."""
import pytest
import torch

import fp8_restatement as F
from lookaheaddecoding_b200 import _cabi
from lookaheaddecoding_b200._cabi import check

pytestmark = pytest.mark.gpu
DTYPES = [torch.bfloat16, torch.float16]


def _sfx(dt):
    return "" if dt == torch.bfloat16 else "_f16"


def _rows(rows, cols, dt, kind, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(rows, cols, generator=g, device="cuda")
    if kind == "zero":
        x[::2] = 0
    elif kind == "huge":
        x[:, cols // 3] = 6e4 if dt == torch.float16 else 3e30
    elif kind == "big":
        x = torch.where(x > 0, 60000.0, -60000.0) * torch.rand(rows, cols, generator=g, device="cuda").clamp(min=0.5)
    elif kind == "tiny":
        x = x * 2.0 ** -12
    return x.to(dt).contiguous()


def _check(q, s, ref_rows):
    rq, rs = F.quant_rows(ref_rows.cpu())
    assert torch.equal(s.cpu(), rs), (s.cpu() - rs).abs().max()
    bad = (q.cpu() != rq).nonzero()
    assert bad.numel() == 0, f"{bad.shape[0]} bytes differ, first at {bad[0].tolist()}"


CASES = [(1, 4096, "randn"), (120, 4096, "zero"), (240, 5120, "huge"), (1024, 4096, "randn"), (120, 11008, "tiny"),
         (240, 13824, "randn"), (1, 14336, "big")]


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("rows,cols,kind", CASES)
def test_quant_rows_bit_exact(dt, rows, cols, kind):
    lib = _cabi.load()
    x = _rows(rows, cols, dt, kind, rows + cols)
    q = torch.empty(rows, cols, dtype=torch.uint8, device="cuda")
    s = torch.empty(rows, dtype=torch.float32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    check(getattr(lib, "lade_quant_rows_fp8" + _sfx(dt))(st, x.data_ptr(), q.data_ptr(), s.data_ptr(), rows, cols))
    torch.cuda.synchronize()
    _check(q, s, x)


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("residual", [False, True])
@pytest.mark.parametrize("rows,cols,kind", [c for c in CASES if c[1] <= 8192 or c[0] == 1])
def test_rmsnorm_quant_bit_exact(dt, residual, rows, cols, kind):
    lib = _cabi.load()
    if cols > 8192 * 3:
        pytest.skip("rmsnorm row limit")
    x = _rows(rows, cols, dt, kind, 7 * rows + cols)
    d = _rows(rows, cols, dt, "randn", rows + 3) if residual else None
    w = (torch.rand(cols, device="cuda") + 0.5).to(dt)
    st = torch.cuda.current_stream().cuda_stream
    h1, h2 = x.clone(), x.clone()
    out = torch.empty_like(x)
    sfx = _sfx(dt)
    dp = d.data_ptr() if residual else 0
    check(getattr(lib, "lade_rmsnorm" + sfx)(st, h1.data_ptr(), dp, w.data_ptr(), h1.data_ptr() if residual else 0,
                                             out.data_ptr(), rows, cols, 1e-5))
    q = torch.empty(rows, cols, dtype=torch.uint8, device="cuda")
    s = torch.empty(rows, dtype=torch.float32, device="cuda")
    check(getattr(lib, "lade_rmsnorm_quant_fp8" + sfx)(st, h2.data_ptr(), dp, w.data_ptr(), h2.data_ptr() if residual else 0,
                                                       q.data_ptr(), s.data_ptr(), rows, cols, 1e-5))
    torch.cuda.synchronize()
    assert F.bits_equal(h1, h2)                           # the residual sum is written back the same way
    _check(q, s, out)


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("rows,inter,kind", [(1, 11008, "randn"), (120, 11008, "zero"), (240, 13824, "randn"),
                                             (240, 14336, "tiny"), (1024, 4096, "huge")])
def test_swiglu_quant_bit_exact(dt, rows, inter, kind):
    lib = _cabi.load()
    gu = _rows(rows, 2 * inter, dt, kind, rows + inter)
    if kind == "huge" and dt == torch.bfloat16:
        gu[:, inter + 5] = 1e30                           # the up half: a huge product in one column
    st = torch.cuda.current_stream().cuda_stream
    out = torch.empty(rows, inter, dtype=dt, device="cuda")
    sfx = _sfx(dt)
    check(getattr(lib, "lade_swiglu" + sfx)(st, gu.data_ptr(), out.data_ptr(), rows, inter))
    q = torch.empty(rows, inter, dtype=torch.uint8, device="cuda")
    s = torch.empty(rows, dtype=torch.float32, device="cuda")
    check(getattr(lib, "lade_swiglu_quant_fp8" + sfx)(st, gu.data_ptr(), q.data_ptr(), s.data_ptr(), rows, inter))
    torch.cuda.synchronize()
    _check(q, s, out)
