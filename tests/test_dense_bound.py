"""The references of the projection GEMM and the glue kernels (oracle.llama_ref.linear_fp64, rms_norm_fp64,
swiglu_fp64), checked without a GPU.

GEMM: lade_gemm_bf16's numerics are emulated in fp32 -- one addition to the accumulator per k16 step, k-blocks of 64 in
order, split-K partials added in split order, one rounding to bf16.  The accumulation error must stay <= 0.6 of the
gamma term of the bound (the derived part; the half-ulp term is exact, a correctly rounded output may use all of it),
the rounded output inside the whole bound, and each planted error must break the bound or one of the exact probes the
GPU tests run (integer operands, one-hot rows).
RMSNorm / SwiGLU: fp32 emulations with the sum of squares taken in several orders must leave no element that is
neither the reference value nor its stated rounding alternative, and each planted error must leave some.

The data builders are shared with tests/test_gpu_gemm_edges.py and tests/test_gpu_layer_ops_edges.py."""
import pytest
import torch

from oracle import llama_ref as LR

DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}
HONEST_ACC = 0.6
BF16 = torch.bfloat16


# ---- data -------------------------------------------------------------------------------------------------------
def gemm_data(kind, m, n, k, gen, device="cpu"):
    """bf16 operands a [m, k], w [n, k]."""
    def rn(*s):
        return torch.randn(*s, generator=gen, device=device)
    if kind == "randn":
        a, w = rn(m, k), rn(n, k) * 0.05
    elif kind == "positive":                       # no cancellation: |ref| = sum |a w|, the accumulation term at its largest
        a, w = rn(m, k).abs() + 0.1, rn(n, k).abs() * 0.05 + 0.01
    elif kind == "huge":                           # one element per row 2^12 times the rest
        a, w = rn(m, k), rn(n, k) * 0.05
        a[torch.arange(m), torch.arange(m) * 37 % k] *= 4096.0
    elif kind == "cancel":                         # columns 2j and 2j+1 cancel up to a 2^-6 remainder
        a = rn(m, k)
        a[:, 1::2] = a[:, 0::2]
        w = rn(n, k) * 0.05
        w[:, 1::2] = -w[:, 0::2] * (1 + 2.0 ** -6)
    elif kind == "wide":                           # magnitudes spread over 2^-12 .. 2^12
        a = rn(m, k) * torch.exp2(torch.randint(-12, 13, (m, k), generator=gen, device=device).float())
        w = rn(n, k) * 0.05 * torch.exp2(torch.randint(-12, 13, (n, k), generator=gen, device=device).float())
    else:
        raise ValueError(kind)
    return a.to(BF16), w.to(BF16)


def integer_data(m, n, k, gen, device="cpu"):
    """a in {-2..2}, w in {-2..2} with about half the entries zero: every partial sum is an integer below 2^16, so
    fp32 accumulation is exact in any order and the bf16 output is T(ref) bit for bit."""
    a = torch.randint(-2, 3, (m, k), generator=gen, device=device).to(BF16)
    w = torch.randint(-2, 3, (n, k), generator=gen, device=device)
    w = (w * torch.randint(0, 2, (n, k), generator=gen, device=device)).to(BF16)
    return a, w


def random_bf16_bits(shape, gen, device="cpu"):
    """Random finite bf16 bit patterns, both signs, every normal exponent, no subnormals (and no NaN / inf)."""
    mant = torch.randint(0, 128, shape, generator=gen, device=device)
    expo = torch.randint(1, 255, shape, generator=gen, device=device)
    sign = torch.randint(0, 2, shape, generator=gen, device=device)
    bits = (sign << 15) | (expo << 7) | mant
    return (bits - ((bits >> 15) << 16)).to(torch.int16).view(BF16)


def one_hot_columns(m, k, split):
    """k_r for r < m: the first / last column of a 64-block, in the first / last block of every split, then the rest of
    K walked with a stride co-prime to 64."""
    kb = k // 64
    per = kb // split
    cols = []
    for s in range(split):
        for b in sorted({s * per, (s + 1) * per - 1}):
            cols += [b * 64, b * 64 + 63, b * 64 + 15, b * 64 + 16]
    r = 0
    while len(cols) < m:
        cols.append((r * 67 + 5) % k)
        r += 1
    return torch.tensor(cols[:m], dtype=torch.long)


def norm_data(rows, hidden, dtype, gen, device="cpu"):
    """x, delta, w.  Row 0: zeros (rstd = rsqrt(eps)); row 1: one huge element; row 2: every element +-60000 (fp16's
    sum of squares must be formed in fp32) with a zero delta; row 3: 1e-4 (eps dominates); the rest randn."""
    x = torch.randn(rows, hidden, generator=gen, device=device)
    d = torch.randn(rows, hidden, generator=gen, device=device) * 0.5
    if rows > 4:
        x[0], d[0] = 0.0, 0.0
        x[1], d[1] = 0.0, 0.0
        x[1, hidden // 3] = 60000.0 if dtype == torch.float16 else 2.0 ** 50
        x[2] = torch.where(x[2] > 0, 60000.0, -60000.0)
        d[2] = 0.0
        x[3], d[3] = 1e-4, 2e-4
    w = 1 + 0.1 * torch.randn(hidden, generator=gen, device=device)
    return x.to(dtype), d.to(dtype), w.to(dtype)


SPECIAL_GATES = [120.0, -120.0, 88.5, -88.5, 89.0, -89.0, 0.0, -0.0, 30.0, -30.0, 1e-40, -1e-40, 2.0 ** -20, 11.0]


def swiglu_data(rows, inter, dtype, gen, device="cpu"):
    """[rows, 2 * inter]: gates uniform in [-120, 120] in the first row(s), randn * 2 in the rest, the special values
    (+-120, +-88.5, +-0, subnormals) sprinkled over the head of row 0; the up half is randn, and in fp16 a stretch of
    row 0 carries gate 11 x up 60000, a product that overflows."""
    g = torch.randn(rows, inter, generator=gen, device=device) * 2
    u = torch.randn(rows, inter, generator=gen, device=device)
    g[0] = torch.rand(inter, generator=gen, device=device) * 240 - 120
    sp = torch.tensor(SPECIAL_GATES, device=device)
    n = min(inter, sp.numel())
    g[0, :n] = sp[:n]
    u[0, :n] = torch.tensor([1.0, -1.5, 0.5, 3.0], device=device).repeat(4)[:n]
    if dtype == torch.float16 and inter >= 16:
        g[0, 13] = 11.0
        u[0, 13] = 60000.0
    return torch.cat([g, u], dim=-1).to(dtype)


# ---- GEMM emulation -----------------------------------------------------------------------------------------------
def emulate_gemm(a, w, split, plant=None):
    """fp32 result [M, N] before the output rounding, as the kernel forms it; `plant` names one planted error."""
    af, wf = a.float(), w.float()
    m, k = af.shape
    kb = k // 64
    per = kb // split
    parts = []
    for s in range(split):
        acc = torch.zeros(m, wf.shape[0])
        for b in range(s * per, (s + 1) * per):
            src = b - 1 if (plant == "k-block read twice" and b == kb - 1 and kb > 1) else b
            for j in range(4):
                if plant == "k16 slice dropped" and b == kb // 2 and j == 2:
                    continue
                sl = slice(src * 64 + j * 16, src * 64 + j * 16 + 16)
                acc = acc + af[:, sl] @ wf[:, sl].t()
        if plant == "partials rounded to bf16":
            acc = acc.to(BF16).float()
        parts.append(acc)
    if plant == "split partial dropped":
        parts = parts[:-1]
    out = parts[0]
    for p in parts[1:]:
        out = out + p
    if plant == "last 8 columns shifted by one group":
        out = torch.cat([out[:, :-8], out[:, -16:-8]], dim=1)
    if plant == "rows 64.. take rows 0..":
        out = torch.cat([out[:64], out[:m - 64]], dim=0)
    return out


PLANTS = ["k16 slice dropped", "k-block read twice", "split partial dropped", "partials rounded to bf16",
          "last 8 columns shifted by one group", "rows 64.. take rows 0.."]


@pytest.mark.parametrize("kind", ["randn", "positive", "huge", "cancel", "wide"])
@pytest.mark.parametrize("k", [64, 4096, 11008])
def test_emulated_gemm_sits_inside_the_bound(k, kind):
    gen = torch.Generator().manual_seed(k + len(kind))
    a, w = gemm_data(kind, 24, 136, k, gen)
    ref, bound = LR.linear_fp64(a, w, BF16)
    acc_term = LR.linear_gamma(k) * (a.double().abs() @ w.double().abs().t())
    for split in (1, 2, 4, 8):
        if (k // 64) % split:
            continue
        pre = emulate_gemm(a, w, split)
        acc_ratio = ((pre.double() - ref).abs() / acc_term).max().item()
        ok, mx, mean = LR.within_bound(pre.to(BF16), ref, bound, LR.LINEAR_MEAN_RATIO)
        print(f"k {k} {kind} split {split}: accumulation {acc_ratio:.4f} of its term, output max {mx:.3f} mean {mean:.3f}")
        assert acc_ratio <= HONEST_ACC, (split, acc_ratio)
        assert ok, (split, mx, mean)


def test_integer_and_one_hot_probes_are_exact_in_the_emulation():
    gen = torch.Generator().manual_seed(1)
    m, n, k = 128, 136, 2048
    a, w = integer_data(m, n, k, gen)
    ref, _ = LR.linear_fp64(a, w, BF16)
    assert ref.abs().max() < 2 ** 16 and torch.equal(ref, ref.round())
    for split in (1, 4):
        assert torch.equal(emulate_gemm(a, w, split).to(BF16), ref.to(BF16))
    cols = one_hot_columns(m, k, 4)
    a1 = torch.zeros(m, k, dtype=BF16)
    a1[torch.arange(m), cols] = 1.0
    w1 = random_bf16_bits((n, k), gen)
    assert torch.equal(emulate_gemm(a1, w1, 4).to(BF16), w1[:, cols].t())
    assert torch.equal(LR.linear_fp64(a1, w1, BF16)[0].to(BF16), w1[:, cols].t())


@pytest.mark.parametrize("plant", PLANTS)
def test_planted_gemm_errors_are_caught(plant):
    """Each planted error must fail the bound on randn data or an exact probe; the honest emulation passes all three."""
    gen = torch.Generator().manual_seed(7)
    m, n, k, split = 128, 136, 4096, 4
    cols = one_hot_columns(m, k, split)
    a1 = torch.zeros(m, k, dtype=BF16)
    a1[torch.arange(m), cols] = 1.0
    cases = {"bound": gemm_data("randn", m, n, k, gen), "integer": integer_data(m, n, k, gen),
             "one-hot": (a1, random_bf16_bits((n, k), gen))}
    for p in (None, plant):
        caught = []
        for name, (a, w) in cases.items():
            ref, bound = LR.linear_fp64(a, w, BF16)
            got = emulate_gemm(a, w, split, p).to(BF16)
            if name == "bound":
                ok, mx, mean = LR.within_bound(got, ref, bound, LR.LINEAR_MEAN_RATIO)
                print(f"{p}: bound max {mx:.2f} mean {mean:.3f}")
            else:
                ok = torch.equal(got, ref.to(BF16))
            if not ok:
                caught.append(name)
        print(f"{p}: caught by {caught}")
        assert bool(caught) == (p is not None), (p, caught)


# ---- RMSNorm / SwiGLU emulation -----------------------------------------------------------------------------------
def _sum_sq(h32, order):
    sq = h32 * h32
    hidden = sq.shape[-1]
    if order == "torch":
        return sq.sum(-1, keepdim=True)
    if order == "sequential":
        return sq.cumsum(-1)[..., -1:]
    if order == "reversed":
        return sq.flip(-1).cumsum(-1)[..., -1:]
    if order == "kernel":                           # 8 per thread in sequence, then a butterfly over the threads
        t = sq.reshape(*sq.shape[:-1], hidden // 8, 8).cumsum(-1)[..., -1]
        while t.shape[-1] > 1:
            if t.shape[-1] % 2:
                t = torch.cat([t, torch.zeros_like(t[..., :1])], dim=-1)
            t = t[..., 0::2] + t[..., 1::2]
        return t
    raise ValueError(order)


def emulate_norm(x, delta, w, eps, dtype, order="torch", plant=None):
    h = x if delta is None else x + delta
    h32 = h.float()
    if plant == "sum of squares in the model dtype":
        tot = (h * h).cumsum(-1)[..., -1:].float()
    else:
        tot = _sum_sq(h32, order)
    eps32 = torch.tensor(eps, dtype=torch.float32)
    if plant == "eps after the rsqrt":
        rstd = torch.rsqrt(tot / h.shape[-1]) + eps32
    else:
        rstd = torch.rsqrt(tot / h.shape[-1] + eps32)
    n = (h32 * rstd).to(dtype)
    return h, (w.float() * n.float()).to(dtype)


def emulate_swiglu(gate_up, dtype, plant=None):
    inter = gate_up.shape[-1] // 2
    g, u = gate_up[..., :inter].float(), gate_up[..., inter:].float()
    silu = g / (1.0 + torch.exp(-g))
    if plant == "rounded after the multiply":
        return (silu * u).to(dtype)
    return (silu.to(dtype).float() * u).to(dtype)


@pytest.mark.parametrize("dtn", list(DTYPES))
@pytest.mark.parametrize("hidden", [8, 264, 4096, 12288])
def test_emulated_rmsnorm_has_no_unexplained_element(hidden, dtn):
    dtype = DTYPES[dtn]
    gen = torch.Generator().manual_seed(hidden)
    x, d, w = norm_data(12, hidden, dtype, gen)
    for delta in (None, d):
        h_ref, out, alt = LR.rms_norm_fp64(x, delta, w, 1e-5, dtype)
        assert torch.isfinite(out.float()).all()
        assert torch.all(out[0] == 0)               # the zero row
        for order in ("torch", "sequential", "reversed", "kernel"):
            h, got = emulate_norm(x, delta, w, 1e-5, dtype, order)
            bad, used = LR.unexplained(got, out, alt)
            print(f"hidden {hidden} {dtn} delta {delta is not None} {order}: {used} of {got.numel()} took the alternative")
            assert torch.equal(h, h_ref) and bad == 0, (order, bad)
            assert used <= 0.02 * got.numel()


@pytest.mark.parametrize("dtn", list(DTYPES))
@pytest.mark.parametrize("plant", ["sum of squares in the model dtype", "eps after the rsqrt"])
def test_planted_rmsnorm_errors_are_flagged(plant, dtn):
    dtype = DTYPES[dtn]
    gen = torch.Generator().manual_seed(11)
    x, d, w = norm_data(12, 4096, dtype, gen)
    _, out, alt = LR.rms_norm_fp64(x, d, w, 1e-5, dtype)
    _, got = emulate_norm(x, d, w, 1e-5, dtype, plant=plant)
    bad, _ = LR.unexplained(got, out, alt)
    print(f"{plant} {dtn}: {bad} unexplained")
    assert bad > 0


@pytest.mark.parametrize("dtn", list(DTYPES))
def test_emulated_swiglu_has_no_unexplained_element(dtn):
    dtype = DTYPES[dtn]
    gen = torch.Generator().manual_seed(5)
    gu = swiglu_data(40, 2048, dtype, gen)
    out, alt = LR.swiglu_fp64(gu, dtype)
    got = emulate_swiglu(gu, dtype)
    bad, used = LR.unexplained(got, out, alt)
    print(f"swiglu {dtn}: {used} of {got.numel()} took the alternative")
    assert bad == 0 and used <= 1e-3 * got.numel()
    assert not torch.isnan(out.float()).any() and not torch.isnan(got.float()).any()
    assert torch.all(out[0, [1, 5]] == 0)           # gates -120 and -89: exp(-g) overflows fp32, silu is -0
    if dtype == torch.float16:
        assert torch.isinf(out[0, 13]) and torch.isinf(got[0, 13])
    bad, _ = LR.unexplained(emulate_swiglu(gu, dtype, plant="rounded after the multiply"), out, alt)
    assert bad > 0
