"""lade_gemm_fp8 / _f16 against a float64 reference of the dequantised operands (tests/fp8_restatement.py `bound`),
exact integer probes of the accumulation, one-hot probes, NaN canaries and row independence.

The worst err / bound of every case is printed (DESIGN.md §6 records them)."""
import pytest
import torch

import fp8_restatement as F
from lookaheaddecoding_b200 import _cabi
from lookaheaddecoding_b200._cabi import LADE_EINVAL, check

pytestmark = pytest.mark.gpu
OUT = {torch.bfloat16: "lade_gemm_fp8", torch.float16: "lade_gemm_fp8_f16"}
# (N, K) of the 7B / 13B / Llama-3-8B projections: fused QKV, o, fused gate/up, down
SHAPES = [(12288, 4096), (4096, 4096), (22016, 4096), (4096, 11008), (15360, 5120), (5120, 5120), (27648, 5120),
          (5120, 13824), (6144, 4096), (28672, 4096), (4096, 14336)]


CANARY_ROWS = 16


def _gemm(qa, sa, qw, sw, m, dt=torch.bfloat16, tile=0, split=0, ldc=None):
    """One launch into a NaN-filled [m + CANARY_ROWS][ldc] buffer.  Rows >= m must stay NaN (the second 128-row block
    computes rows up to 255 whatever m is); a rejected call must leave the whole buffer NaN.  Returns (rc, c[:m])."""
    lib = _cabi.load()
    n, k = qw.shape
    ldc = ldc or n
    c = torch.full((m + CANARY_ROWS, ldc), float("nan"), dtype=dt, device="cuda")
    rc = getattr(lib, OUT[dt])(torch.cuda.current_stream().cuda_stream, qa.data_ptr(), sa.data_ptr(), qw.data_ptr(),
                               sw.data_ptr(), c.data_ptr(), m, qa.shape[0], n, k, ldc, tile, split)
    torch.cuda.synchronize()
    if rc == 0:
        assert torch.isnan(c[m:]).all(), f"canary below row {m} overwritten"
    else:
        assert torch.isnan(c).all(), "a rejected call wrote"
    return rc, c[:m]


def _operands(m, n, k, seed, a_rows=None):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(a_rows or m, k, generator=g, device="cuda").to(torch.bfloat16)
    w = (torch.randn(n, k, generator=g, device="cuda") * 0.02).to(torch.bfloat16)
    qa, sa = F.quant_rows(a.float().cpu())
    qw, sw = F.quant_rows(w.float().cpu())
    return qa.cuda(), sa.cuda(), qw.cuda(), sw.cuda()


def _check_bound(c, qa, sa, qw, sw, m, dt, what):
    qa, sa = qa[:m].cpu(), sa[:m].cpu()
    qw, sw = qw.cpu(), sw.cpu()
    ref = F.linear64(qa, sa, qw, sw)
    b = F.bound(qa, sa, qw, sw, out_dtype=dt)
    err = (c[:m, :qw.shape[0]].double().cpu() - ref).abs()
    ratio = float((err / b).max())
    print(f"{what}: worst err/bound {ratio:.3f}")
    assert ratio <= 1.0, what


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("m", [1, 8, 64, 65, 120, 128, 129, 240, 256, 1024])
def test_rows_against_float64(dt, m):
    n, k = 4096, 4096
    qa, sa, qw, sw = _operands(m, n, k, m)
    rc, c = _gemm(qa, sa, qw, sw, m, dt)
    assert rc == 0
    _check_bound(c, qa, sa, qw, sw, m, dt, f"m={m} {dt}")


@pytest.mark.parametrize("n,k", SHAPES)
def test_projection_shapes(n, k):
    for m in (120, 240):
        qa, sa, qw, sw = _operands(m, n, k, n + k)
        rc, c = _gemm(qa, sa, qw, sw, m)
        assert rc == 0
        _check_bound(c, qa, sa, qw, sw, m, torch.bfloat16, f"N={n} K={k} m={m}")


def test_forced_configurations():
    n, k = 1000 + 24, 2048         # a ragged last tile for every width
    qa, sa, qw, sw = _operands(240, n, k, 5)
    ok = 0
    for tile in (32, 64, 96, 128, 160):
        for split in (1, 2, 4, 8, 16):
            for m in (120, 240):
                rc, c = _gemm(qa, sa, qw, sw, m, tile=tile, split=split, ldc=n + 8)
                if tile > 128 or split > 8 or (k // 128) % split:
                    assert rc == LADE_EINVAL, (tile, split)
                if rc == LADE_EINVAL:          # also: a split whose partial tiles do not fit the ring it leaves
                    continue                   # (_gemm checked that nothing was written)
                assert rc == 0, (tile, split, m)
                _check_bound(c, qa, sa, qw, sw, m, torch.bfloat16, f"tile {tile} split {split} m {m}")
                assert torch.isnan(c[:, n:]).all(), "canary right of the last tile"
                ok += 1
    assert ok >= 20


def _int_operands(m, n, k):
    a = torch.zeros(m, k)
    w = torch.zeros(n, k)
    a[:, :128], w[:, :128] = 15.0, 15.0           # block 0: 28800
    a[:, 128], w[:, 128] = 1.0, 1.0               # block 1: 1      -> 28801 (15 bits)
    a[:, 256:384], w[:, 256:384] = 15.0, -15.0    # block 2: -28800 -> 1
    w[1::2, 128] = 3.0                            # odd columns: 3
    q = lambda x: x.to(torch.float8_e4m3fn).view(torch.uint8).cuda()
    return q(a), torch.ones(m, device="cuda"), q(w), torch.ones(n, device="cuda")


@pytest.mark.parametrize("split", [1, 2, 4])
def test_integer_probe_cross_block_sums_are_exact(split):
    """Running sums that need 15 bits across k-blocks come out exact: the promotion into fp32 works."""
    qa, sa, qw, sw = _int_operands(130, 64, 1024)
    rc, c = _gemm(qa, sa, qw, sw, 130, tile=64, split=split)
    assert rc == 0
    want = torch.ones(130, 64)
    want[:, 1::2] = 3.0
    assert torch.equal(c.float().cpu(), want)


def test_integer_probe_within_block_measurement():
    """Within one 128-deep block the tensor cores do not accumulate in fp32: the block sum 2^15 - 255 = 32513 (15
    significant bits) comes out as 32512 on the H100 (about 14 bits kept, DESIGN.md §6.4); the next block's -32768 is
    added exactly after the promotion, so the result is -256 where the exact value is -255."""
    k = 128 * 8
    a = torch.zeros(1, k)
    w = torch.zeros(8, k)
    a[0, :128] = 16.0
    w[:, :128] = 16.0                      # 128 * 256 = 32768 = 2^15
    a[0, 127], w[:, 127] = 1.0, 1.0        # ... + 1 - 256 = 2^15 - 255 in block 0 (needs 15 bits)
    a[0, 128:256] = 16.0
    w[:, 128:256] = -16.0                  # block 1: -32768
    q = lambda x: x.to(torch.float8_e4m3fn).view(torch.uint8).cuda()
    qa, qw = q(a), q(w)
    one = torch.ones(8, device="cuda")
    rc, c = _gemm(qa, one[:1], qw, one, 1, dt=torch.float16)
    exact = F.linear64(qa.cpu(), one[:1].cpu(), qw.cpu(), one.cpu())
    print(f"within-block probe: exact {exact[0, 0].item()} kernel {c[0, 0].item()}")
    assert rc == 0
    assert exact[0].tolist() == [-255.0] * 8
    assert c[0].float().cpu().tolist() == [-256.0] * 8


def test_one_hot_and_nan_rows():
    m, n, k = 129, 256, 512
    a = torch.zeros(m, k)
    w = torch.zeros(n, k)
    for r in range(m):
        a[r, (r * 7) % k] = 1.0 + (r % 7) / 8
    for j in range(n):
        w[j, (j * 7) % k] = 1.0
    q = lambda x: x.to(torch.float8_e4m3fn).view(torch.uint8).cuda()
    qa = torch.full((m + 40, k), 0x7F, dtype=torch.uint8, device="cuda")      # rows >= m: NaN
    qa[:m] = q(a)
    sa = torch.full((m + 40,), float("nan"), device="cuda")
    sa[:m] = 2.0
    sw = torch.full((n,), 0.5, device="cuda")
    rc, c = _gemm(qa, sa, q(w), sw, m, ldc=n + 16)
    assert rc == 0
    want = (a @ w.T)
    assert torch.equal(c[:, :n].float().cpu(), want)
    assert torch.isnan(c[:, n:]).all()


def test_row_independence():
    """Row r's output bits do not depend on how many rows the launch carries (m = 1 .. 1024, chunked above 256)."""
    n, k = 4096, 4096
    qa, sa, qw, sw = _operands(1024, n, k, 11)
    _, full = _gemm(qa, sa, qw, sw, 1024)
    for m in (1, 120, 128, 240, 256):
        _, c = _gemm(qa, sa, qw, sw, m)
        assert F.bits_equal(c, full[:m]), m
    # the same row at different positions / chunks
    rep = qa[:1].repeat(1024, 1).contiguous()
    srep = sa[:1].repeat(1024).contiguous()
    _, c = _gemm(rep, srep, qw, sw, 1024)
    assert F.bits_equal(c, full[:1].expand(1024, -1).contiguous())
