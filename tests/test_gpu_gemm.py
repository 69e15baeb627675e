"""wgmma weight-streaming projection GEMM (lade_gemm_bf16) vs torch: C = A . W^T, bf16 in/out, fp32 accumulate.

The reference computes these with nn.Linear (modeling_llama.py:447-449,541,378,1608).  Accumulation order differs
from cuBLAS, so results may differ by one bf16 ulp on a small fraction of elements; the test bounds both the
fraction and the magnitude against an fp32 matmul of the same bf16 inputs.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _lib():
    from lookaheaddecoding_b200 import _cabi
    return _cabi.load(), _cabi.check, _cabi


def _run(lib, a, w, m, n, k, ldc=None, tile_n=0, split_k=0, c=None):
    ldc = ldc or n
    if c is None:
        c = torch.full((a.shape[0], ldc), float("nan"), dtype=torch.bfloat16, device="cuda")
    rc = lib.lade_gemm_bf16(torch.cuda.current_stream().cuda_stream, a.data_ptr(), w.data_ptr(), c.data_ptr(), m,
                            a.shape[0], n, k, ldc, tile_n, split_k)
    return rc, c


def _check(c, a, w, m, n):
    ref32 = a[:m].float() @ w.float().t()
    ref = ref32.to(torch.bfloat16)
    got = c[:m, :n]
    assert torch.isfinite(got.float()).all()
    # bf16 has 8 bits of mantissa: one ulp is 2^-8 relative
    err = (got.float() - ref32).abs()
    tol = ref32.abs() * 2 ** -7 + 1e-2 * ref32.abs().mean()
    assert (err <= tol).all(), f"max err {err.max().item()}"
    assert (got != ref).float().mean() < 0.02


SHAPES = [
    # (m, n, k, tile_n, split_k)
    (120, 768, 256, 0, 0),        # tiny-model qkv
    (1, 256, 256, 0, 0),
    (34, 512, 512, 32, 1),
    (128, 4096, 4096, 0, 0),      # o_proj (7B): auto = tile 128, split 4
    (120, 12288, 4096, 0, 0),     # fused qkv (7B): auto = tile 192, split 2
    (120, 22016, 4096, 0, 0),     # fused gate/up (7B): ragged last tile
    (120, 4096, 11008, 0, 0),     # down_proj (7B): split 4, 43 k-blocks each
    (76, 32000, 4096, 0, 0),      # lm_head rows
    (120, 1000, 1024, 96, 1),     # n not a multiple of the tile
    (120, 1000, 1024, 64, 2),
    (97, 2048, 2048, 256, 8),     # widest tile, deepest split
    (120, 5120, 5120, 160, 1),
    # tuning knobs: tile_n | pipeline depth cap << 16 | no-prefill << 20
    (120, 12288, 4096, 192 | (3 << 16), 2),
    (120, 22016, 4096, 160 | (1 << 20), 1),
    (76, 32000, 4096, 224 | (2 << 16) | (1 << 20), 1),
    (120, 4096, 11008, 128 | (3 << 16), 4),
]


@pytest.mark.parametrize("m,n,k,tile_n,split_k", SHAPES)
def test_gemm_matches_fp32_reference(m, n, k, tile_n, split_k):
    lib, check, _ = _lib()
    torch.manual_seed(m * 7 + n)
    a = torch.randn(128, k, device="cuda").to(torch.bfloat16)
    w = (torch.randn(n, k, device="cuda") * 0.05).to(torch.bfloat16)
    rc, c = _run(lib, a, w, m, n, k, tile_n=tile_n, split_k=split_k)
    check(rc)
    torch.cuda.synchronize()
    _check(c, a, w, m, n)
    # rows >= m are never written
    if m < 128:
        assert torch.isnan(c[m:].float()).all()


def test_gemm_short_a_buffer_and_strided_output():
    """A buffer with exactly m rows (TMA zero-fills the rest of the box) and an output slice with ldc > n."""
    lib, check, _ = _lib()
    torch.manual_seed(3)
    m, n, k = 45, 512, 1024
    a = torch.randn(m, k, device="cuda").to(torch.bfloat16)
    w = (torch.randn(n, k, device="cuda") * 0.05).to(torch.bfloat16)
    big = torch.full((m, 3 * n), float("nan"), dtype=torch.bfloat16, device="cuda")
    view = big[:, n:]
    rc = lib.lade_gemm_bf16(torch.cuda.current_stream().cuda_stream, a.data_ptr(), w.data_ptr(), view.data_ptr(), m, m, n, k,
                            3 * n, 0, 0)
    check(rc)
    torch.cuda.synchronize()
    _check(big[:, n:2 * n], a, w, m, n)
    assert torch.isnan(big[:, :n].float()).all() and torch.isnan(big[:, 2 * n:].float()).all()


def test_gemm_deterministic_and_graph_capturable():
    lib, check, _ = _lib()
    torch.manual_seed(5)
    m, n, k = 120, 4096, 4096
    a = torch.randn(128, k, device="cuda").to(torch.bfloat16)
    w = (torch.randn(n, k, device="cuda") * 0.05).to(torch.bfloat16)
    rc, c1 = _run(lib, a, w, m, n, k)
    check(rc)
    c2 = torch.zeros_like(c1)
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            check(lib.lade_gemm_bf16(s.cuda_stream, a.data_ptr(), w.data_ptr(), c2.data_ptr(), m, 128, n, k, n, 0, 0))
    torch.cuda.current_stream().wait_stream(s)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(c1[:m], c2[:m])


def test_gemm_rejects_unsupported_shapes():
    lib, _, cabi = _lib()
    a = torch.zeros(256, 688, dtype=torch.bfloat16, device="cuda")
    w = torch.zeros(64, 688, dtype=torch.bfloat16, device="cuda")
    c = torch.zeros(256, 64, dtype=torch.bfloat16, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    assert lib.lade_gemm_bf16(st, a.data_ptr(), w.data_ptr(), c.data_ptr(), 120, 256, 64, 688, 64, 0, 0) == cabi.LADE_EUNSUPPORTED
    a2 = torch.zeros(256, 512, dtype=torch.bfloat16, device="cuda")
    w2 = torch.zeros(64, 512, dtype=torch.bfloat16, device="cuda")
    assert lib.lade_gemm_bf16(st, a2.data_ptr(), w2.data_ptr(), c.data_ptr(), 129, 256, 64, 512, 64, 0, 0) == cabi.LADE_EUNSUPPORTED
