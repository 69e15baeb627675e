"""CPU checks of the FP8 projection restatement (tests/fp8_restatement.py) the GPU tests hold the kernels to.

* the row quantiser against an independent nearest-even search over the 256 e4m3 codes: ties, saturation, subnormals,
  +-0; the scale rule (amax / 448, 1 for an all-zero row);
* the kernel's fp32 accumulation order (per-128 block promotion, split partials in split order) stays within the bound
  the GPU GEMM is held to on randn, all-positive, one-huge-element, cancelling and wide-range data;
* planted errors break the bound or an exact probe: a dropped k-block, scales swapped between rows and columns,
  quantising the fp32 norm output instead of the one rounded to the model dtype, a missing promotion (a ~14-bit
  running accumulator).
"""
import numpy as np
import pytest
import torch

import fp8_restatement as F


def _nearest_even_e4m3(y: np.ndarray) -> np.ndarray:
    tab = F.np_e4m3_table()
    codes = np.array([c for c in range(256) if np.isfinite(tab[c])])
    vals = tab[codes]
    y = np.clip(y, -448.0, 448.0)
    out = np.empty(y.shape, dtype=np.uint8)
    for i, v in enumerate(y.ravel()):
        d = np.abs(vals - v)
        best = np.flatnonzero(d == d.min())
        if len(best) > 1:                                  # tie: the even code (mantissa LSB 0); +-0: keep the sign
            best = [b for b in best if codes[b] % 2 == 0] or best
            best = [b for b in best if (codes[b] >= 128) == bool(np.signbit(v))] or best   # +-0: the sign of v
        out.ravel()[i] = codes[best[0]]
    return out


def test_quantiser_matches_nearest_even_search():
    g = torch.Generator().manual_seed(0)
    tab = F.np_e4m3_table()
    fin = np.sort(np.unique(tab[np.isfinite(tab)]))
    mids = (fin[1:] + fin[:-1]) / 2                         # exact ties between neighbours
    rows = [
        torch.tensor(np.concatenate([[448.0], mids[:127]])),                 # amax 448: s = 1, ties as they are
        torch.tensor(np.concatenate([[448.0], mids[127:], np.zeros(254 - len(mids))])),
        torch.tensor([448.0, 2.0 ** -9, -2.0 ** -9, 3 * 2.0 ** -10, 2.0 ** -7, 0.0, -0.0, 1e-30] + [0.0] * 120),  # subnormals, +-0
        torch.randn(128, generator=g) * 3,
        torch.zeros(128),
    ]
    x = torch.stack([r.float() for r in rows])
    q, s = F.quant_rows(x)
    assert s[4].item() == 1.0 and s[0].item() == 1.0
    ref_s = (x.abs().amax(1) / 448.0)
    assert torch.equal(s[:4], ref_s[:4])
    y = (x / s[:, None]).numpy().astype(np.float64)
    assert np.array_equal(q.numpy(), _nearest_even_e4m3(y))
    assert q[2, 6].item() == 0x80 and q[2, 5].item() == 0                   # -0 keeps its sign
    # saturation: a quotient that rounds past 448 stays 448
    q2, _ = F.quant_rows(torch.tensor([[448.0, -447.9, 430.0]]))
    assert F.dequant(q2)[0].tolist() == [448.0, -448.0, 416.0]


def _data(kind, m, n, k, g):
    if kind == "randn":
        a, w = torch.randn(m, k, generator=g), torch.randn(n, k, generator=g) * 0.02
    elif kind == "positive":
        a, w = torch.rand(m, k, generator=g), torch.rand(n, k, generator=g)
    elif kind == "huge":
        a, w = torch.randn(m, k, generator=g), torch.randn(n, k, generator=g)
        a[:, 7] = 3e4
    elif kind == "cancel":
        a = torch.randn(m, k // 2, generator=g)
        a = torch.cat([a, a], 1)
        w = torch.randn(n, k // 2, generator=g)
        w = torch.cat([w, -w], 1)
    else:   # wide range
        a = torch.randn(m, k, generator=g) * torch.exp2(torch.randint(-20, 20, (m, k), generator=g).float())
        w = torch.randn(n, k, generator=g) * torch.exp2(torch.randint(-10, 10, (n, k), generator=g).float())
    return a.to(torch.bfloat16), w.to(torch.bfloat16)


@pytest.mark.parametrize("kind", ["randn", "positive", "huge", "cancel", "wide"])
@pytest.mark.parametrize("split_k", [1, 2, 8])
def test_emulated_kernel_within_bound(kind, split_k):
    g = torch.Generator().manual_seed(hash(kind) % 1000 + split_k)
    a, w = _data(kind, 8, 64, 2048, g)
    qa, sa = F.quant_rows(a)
    qw, sw = F.quant_rows(w)
    c = F.emulate_kernel(qa, sa, qw, sw, split_k=split_k).double()
    ref = F.linear64(qa, sa, qw, sw)
    b = F.bound(qa, sa, qw, sw)
    assert ((c - ref).abs() <= b).all(), float(((c - ref).abs() / b).max())


def _probe_operands(k=1024):
    """Integer e4m3 operands whose running sum needs 15 bits while every block sum needs at most 9: exact in fp32."""
    a = torch.zeros(2, k)
    w = torch.zeros(4, k)
    a[:, :128], w[:, :128] = 15.0, 15.0           # block 0: 28800
    a[:, 128], w[:, 128] = 1.0, 1.0               # block 1: 1      -> 28801
    a[:, 256:384], w[:, 256:384] = 15.0, -15.0    # block 2: -28800 -> 1
    qa = a.to(torch.float8_e4m3fn).view(torch.uint8)
    qw = w.to(torch.float8_e4m3fn).view(torch.uint8)
    return qa, torch.ones(2), qw, torch.ones(4)


def test_planted_errors_are_caught():
    g = torch.Generator().manual_seed(3)
    a, w = _data("positive", 8, 64, 1024, g)
    qa, sa = F.quant_rows(a)
    qw, sw = F.quant_rows(w)
    ref, b = F.linear64(qa, sa, qw, sw), F.bound(qa, sa, qw, sw)
    over = lambda c: bool(((c.double() - ref).abs() > b).any())
    assert not over(F.emulate_kernel(qa, sa, qw, sw))
    assert over(F.emulate_kernel(qa, sa, qw, sw, drop_block=3))                                  # dropped k-block
    # scales swapped between rows and columns: c[r][n] = (sum_k a[r][k] w[n][k]) * sw[r] * sa[n], r, n < 8
    sa2 = torch.rand(8, generator=g) + 0.5
    sw2 = torch.rand(64, generator=g) + 0.5
    ref2, b2 = F.linear64(qa, sa2, qw, sw2), F.bound(qa, sa2, qw, sw2)
    raw = F.linear64(qa, torch.ones(8), qw, torch.ones(64))[:, :8]
    swapped = (raw * sw2[:8].double()[:, None] * sa2.double()[None, :]).to(torch.bfloat16)
    assert bool(((swapped.double() - ref2[:, :8]).abs() > b2[:, :8]).any())
    # quantising the fp32 norm output instead of the bf16-rounded one (what lade_rmsnorm_quant_fp8 must quantise):
    # the emulated kernel's output on the wrongly quantised activations differs from the one on the right ones
    h = torch.randn(8, 1024, generator=g) * 3
    nw = torch.rand(1024, generator=g) + 0.5
    n32 = nw * (h * torch.rsqrt(h.pow(2).mean(-1, keepdim=True) + 1e-5))
    nT = (nw.to(torch.bfloat16).float() * (h * torch.rsqrt(h.pow(2).mean(-1, keepdim=True) + 1e-5)).to(torch.bfloat16).float()).to(torch.bfloat16)
    qa_ok, sa_ok = F.quant_rows(nT)
    qa_bad, sa_bad = F.quant_rows(n32)
    assert not torch.equal(qa_ok, qa_bad)
    assert not F.bits_equal(F.emulate_kernel(qa_ok, sa_ok, qw, sw), F.emulate_kernel(qa_bad, sa_bad, qw, sw))
    # missing promotion: the exact probe
    qa, sa, qw, sw = _probe_operands()
    exact = F.linear64(qa, sa, qw, sw)
    assert torch.equal(exact, torch.ones(2, 4, dtype=torch.float64))
    assert torch.equal(F.emulate_kernel(qa, sa, qw, sw).double(), exact)
    assert not torch.equal(F.emulate_kernel(qa, sa, qw, sw, promote=False).double(), exact)
