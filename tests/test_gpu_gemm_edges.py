"""lade_gemm_bf16 at its edges, against oracle.llama_ref.linear_fp64.

* exact probes, bit for bit: integer operands (fp32 accumulation is exact in any order) and one-hot rows of `a` against
  random bf16 bit patterns in `w` (c[r, :] must be column k_r of w) and the transpose, at every row count where the
  kernel changes shape (1 .. 63 | 64 | 65 .. 128: one or two consumer warpgroups), with and without split-K, K from
  one k-block to 11008, N from 8 to 128256, every forced tile x split, grids of several waves, pipeline depth caps;
* the float64 bound on randn, all-positive and wide-dynamic-range data at the 7B, 13B and 70B projection shapes;
* isolation: NaN canaries right of a ragged last tile (ldc > n) and below row m for both epilogues, NaN / inf in the
  rows [m, a_rows) of `a`, one weight or activation address reused under another tile width or shape (the tensor-map
  cache), and every documented argument error, which must launch nothing.
In every exact probe the rows [m, 128) of the `a` buffer hold NaN.

The forced-configuration rule, from include/lade_sm100.h: tile a multiple of 32 in [32, 256]; split_k 1, 2, 4 or 8
dividing the k / 64 k-blocks; with split_k > 1, 128 * (tile + 4) * 4 <= stages * (16384 + 128 * tile) where
stages = min(floor(231232 / (16384 + 128 * tile)), 11, k / 64 / split_k, depth cap if given); LADE_EINVAL otherwise."""
import pytest
import torch

from oracle import llama_ref as LR
from test_dense_bound import BF16, gemm_data, integer_data, one_hot_columns, random_bf16_bits

pytestmark = pytest.mark.gpu
NAN = float("nan")


def _lib():
    from lookaheaddecoding_b200 import _cabi
    return _cabi.load(), _cabi


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _knobs(tile, depth=0, no_prefill=False):
    return tile | (depth << 16) | (int(no_prefill) << 20)


def _launch(a, w, c, m, n, k, ldc, tile_n=0, split=0, a_rows=None):
    lib, _ = _lib()
    return lib.lade_gemm_bf16(torch.cuda.current_stream().cuda_stream, a.data_ptr(), w.data_ptr(), c.data_ptr(), m,
                              a.shape[0] if a_rows is None else a_rows, n, k, ldc, tile_n, split)


def _run(a, w, m, tile_n=0, split=0, ldc=None, c_rows=None, a_rows=None):
    """Launch into a NaN-filled c [c_rows or m + 3, ldc or n]; returns (rc, c) after a synchronise."""
    n, k = w.shape
    ldc = ldc or n
    c = torch.full((c_rows or m + 3, ldc), NAN, dtype=BF16, device="cuda")
    rc = _launch(a, w, c, m, n, k, ldc, tile_n, split, a_rows)
    torch.cuda.synchronize()
    return rc, c


def _pad_a(a, rows=128):
    """`a` [m, k] in a buffer of `rows` rows whose tail is NaN."""
    buf = torch.full((rows, a.shape[1]), NAN, dtype=BF16, device="cuda")
    buf[:a.shape[0]] = a
    return buf


def forced_config_code(k, tile, split, depth=0):
    """The documented return code of a forced (tile, split_k, depth cap)."""
    _, cabi = _lib()
    if tile % 32 or not 32 <= tile <= 256 or split not in (1, 2, 4, 8) or (k // 64) % split:
        return cabi.LADE_EINVAL
    stage = 16384 + 128 * tile
    stages = min(231232 // stage, 11, k // 64 // split, depth or 11)
    if split > 1 and 128 * (tile + 4) * 4 > stages * stage:
        return cabi.LADE_EINVAL
    return cabi.LADE_OK


def _assert_exact(c, want, m, n, what, names_k=None):
    """c[:m, :n] == want bit for bit; canary rows >= m untouched.  A failure names the first wrong (row, column)."""
    got = c[:m, :n]
    bad = ~(got == want)                      # NaN counts as wrong
    if bad.any():
        r, col = bad.nonzero()[0].tolist()
        k_of = f", k = {int(names_k[r])}" if names_k is not None else ""
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements wrong, first at row {r}, column {col}"
                             f"{k_of}: got {got[r, col].item()}, want {want[r, col].item()}; wrong rows "
                             f"{bad.any(1).nonzero().flatten().tolist()[:16]}")
    assert torch.isnan(c[m:]).all(), f"{what}: rows >= m were written"
    assert torch.isnan(c[:m, n:]).all(), f"{what}: columns >= n were written"


def _exact_probes(m, n, k, tile_n, split, seed, **kw):
    """The integer probe and the two one-hot probes for one launch shape; `split` only steers the one-hot columns."""
    _, cabi = _lib()
    gen = _gen(seed)
    tag = f"m {m} n {n} k {k} tile_n {tile_n:#x} split {split}"
    a, w = integer_data(m, n, k, gen, "cuda")
    rc, c = _run(_pad_a(a), w, m, tile_n, split, **kw)
    cabi.check(rc, tag)
    _assert_exact(c, LR.linear_fp64(a, w, BF16)[0].to(BF16), m, n, tag + " integer")
    # one-hot rows of a: c[r, :] = w[:, k_r]
    cols = one_hot_columns(m, k, max(split, 1)).cuda()
    a1 = torch.zeros(m, k, dtype=BF16, device="cuda")
    a1[torch.arange(m, device="cuda"), cols] = 1.0
    w1 = random_bf16_bits((n, k), gen, "cuda")
    rc, c = _run(_pad_a(a1), w1, m, tile_n, split, **kw)
    cabi.check(rc, tag)
    _assert_exact(c, w1[:, cols].t(), m, n, tag + " one-hot a", names_k=cols)
    # one-hot rows of w: c[:, j] = a[:, k_j]
    colw = one_hot_columns(min(n, 4096), k, max(split, 1)).cuda()
    colw = colw.repeat(-(-n // colw.numel()))[:n].roll(n // 3)
    w2 = torch.zeros(n, k, dtype=BF16, device="cuda")
    w2[torch.arange(n, device="cuda"), colw] = 1.0
    a2 = random_bf16_bits((m, k), gen, "cuda")
    rc, c = _run(_pad_a(a2), w2, m, tile_n, split, **kw)
    cabi.check(rc, tag)
    _assert_exact(c, a2[:, colw], m, n, tag + " one-hot w")


@pytest.mark.parametrize("tile,split", [(96, 1), (64, 4)])
@pytest.mark.parametrize("m", [1, 8, 16, 63, 64, 65, 127, 128])
def test_exact_at_every_row_count(m, tile, split):
    _exact_probes(m, 1000, 2048, tile, split, seed=m)


@pytest.mark.parametrize("m,n,k,tile,split", [
    (120, 256, 64, 0, 0),          # one k-block: the ring has one stage, the prefill issues the whole problem
    (64, 256, 128, 32, 2),         # one k-block per split
    (65, 512, 512, 32, 8),         # one k-block per split, eight splits
    (128, 96, 704, 32, 1),         # 11 k-blocks: the deepest ring, filled exactly once
    (127, 96, 1408, 32, 2),        # 11 k-blocks per split
    (33, 4096, 11008, 0, 0),       # down_proj: 172 k-blocks
    (16, 512, 11008, 128, 4),
    (128, 8, 512, 0, 0),           # n below every tile width
    (40, 24, 512, 32, 2),
    (128, 40, 1024, 64, 4),        # n < tile, n % 32 != 0, split-K
    (76, 32000, 1024, 0, 0),
])
def test_exact_at_k_and_n_edges(m, n, k, tile, split):
    _exact_probes(m, n, k, tile, split, seed=n + k)


@pytest.mark.parametrize("m,n,k,tile,split", [
    (128, 32000, 512, 32, 1),      # 1000 CTAs, no cluster
    (100, 32000, 1024, 64, 2),     # 500 clusters of 2
    (128, 128256, 1024, 0, 0),     # nothing fits one wave: tile 256, split 1, 501 CTAs
])
def test_exact_on_grids_of_several_waves(m, n, k, tile, split):
    _exact_probes(m, n, k, tile, split, seed=n)


@pytest.mark.parametrize("tile,split,depth,no_prefill", [(32, 4, 1, False), (64, 4, 2, False), (64, 4, 0, True),
                                                         (64, 1, 1, False), (256, 2, 3, True)])
def test_exact_under_depth_caps_and_without_prefill(tile, split, depth, no_prefill):
    _, cabi = _lib()
    assert forced_config_code(2048, tile, split, depth) == cabi.LADE_OK
    _exact_probes(120, 1000, 2048, _knobs(tile, depth, no_prefill), split, seed=tile + depth)


def test_every_forced_configuration_is_exact_or_rejected_as_documented():
    """tile 32 .. 256 x split 1 .. 8 at m 128, n 1000, k 2048, then the shapes where the staging rule bites."""
    _, cabi = _lib()
    gen = _gen(11)
    m, n = 128, 1000
    seen = {cabi.LADE_OK: 0, cabi.LADE_EINVAL: 0}
    for k, tiles, splits, depth in [(2048, range(32, 257, 32), (1, 2, 4, 8), 0), (512, range(32, 257, 32), (8,), 0),
                                    (2048, (32, 64, 128, 256), (2, 8), 1), (2048, (16, 48, 288, 0), (1, 2), 0),
                                    (2048, (64,), (3, 5, 16), 0), (1088, (64,), (2, 4, 8), 0)]:
        a, w = integer_data(m, n, k, gen, "cuda")
        want = LR.linear_fp64(a, w, BF16)[0].to(BF16)
        for tile in tiles:
            for split in splits:
                code = forced_config_code(k, tile, split, depth) if tile else cabi.LADE_OK   # tile 0: library's choice
                rc, c = _run(a, w, m, _knobs(tile, depth), split)
                assert rc == code, f"k {k} tile {tile} split {split} depth cap {depth}: rc {rc}, documented {code}"
                seen[code] += 1
                if code == cabi.LADE_OK:
                    _assert_exact(c, want, m, n, f"k {k} tile {tile} split {split} depth cap {depth}")
                else:
                    assert torch.isnan(c).all(), "a rejected configuration wrote to c"
    print(f"forced configurations: {seen[cabi.LADE_OK]} exact, {seen[cabi.LADE_EINVAL]} rejected")
    assert seen[cabi.LADE_OK] >= 32 and seen[cabi.LADE_EINVAL] >= 16


FAMILIES = {
    "7B": [(4096, 4096), (12288, 4096), (11008, 4096), (22016, 4096), (4096, 11008), (32000, 4096)],
    "13B": [(5120, 5120), (15360, 5120), (27648, 5120), (5120, 13824)],
    "70B gate/up": [(28672, 8192)],
}


@pytest.mark.parametrize("kind", ["randn", "positive", "wide"])
@pytest.mark.parametrize("family", list(FAMILIES))
def test_projection_shapes_within_the_float64_bound(family, kind):
    _, cabi = _lib()
    worst = (0.0, 0.0)
    for n, k in FAMILIES[family]:
        a, w = gemm_data(kind, 120, n, k, _gen(n + k), "cuda")
        rc, c = _run(_pad_a(a), w, 120)
        cabi.check(rc)
        ref, bound = LR.linear_fp64(a, w, BF16)
        ok, mx, mean = LR.within_bound(c[:120], ref, bound, LR.LINEAR_MEAN_RATIO)
        acc = ((c[:120].double() - ref).abs() - 0.5 * LR.ulp(ref, BF16)).clamp_min(0) / (bound - 0.5 * LR.ulp(ref, BF16))
        print(f"{family} n {n} k {k} {kind}: err/bound max {mx:.3f} mean {mean:.3f}; beyond the half ulp: "
              f"{acc.max().item():.4f} of the accumulation term")
        assert ok, (n, k, kind, mx, mean)
        assert torch.isnan(c[120:]).all()
        worst = max(worst, (mx, mean))
        del ref, bound, acc
    print(f"{family} {kind}: worst err/bound {worst[0]:.3f} (mean {worst[1]:.3f})")


@pytest.mark.parametrize("tile,split", [(96, 1), (64, 2), (256, 4), (0, 0)])
@pytest.mark.parametrize("m", [60, 120])
def test_ragged_last_tile_next_to_live_memory(m, tile, split):
    """n = 1000 inside ldc = 1024: the last tile hangs over columns [1000, 1024), which belong to someone else."""
    _, cabi = _lib()
    a, w = integer_data(m, 1000, 1024, _gen(m + tile), "cuda")
    rc, c = _run(_pad_a(a), w, m, tile, split, ldc=1024, c_rows=136)
    cabi.check(rc)
    _assert_exact(c, LR.linear_fp64(a, w, BF16)[0].to(BF16), m, 1000, f"m {m} tile {tile} split {split}")


@pytest.mark.parametrize("tile,split", [(128, 1), (64, 4), (32, 8)])
@pytest.mark.parametrize("a_rows", ["m", 128, 200])
@pytest.mark.parametrize("m", [45, 64, 65])
def test_poison_below_row_m_stays_out(m, a_rows, tile, split):
    _, cabi = _lib()
    a_rows = m if a_rows == "m" else a_rows
    a, w = integer_data(m, 512, 2048, _gen(m), "cuda")
    buf = _pad_a(a, a_rows)
    buf[m::2] = float("inf")                       # NaN and inf alternate in [m, a_rows)
    rc, c = _run(buf, w, m, tile, split)
    cabi.check(rc)
    _assert_exact(c, LR.linear_fp64(a, w, BF16)[0].to(BF16), m, 512, f"m {m} a_rows {a_rows} tile {tile} split {split}")


def test_one_address_under_two_descriptors():
    """The tensor maps are cached by (address, rows, columns, box rows): the same weight storage at two tile widths
    and as two shapes, and the same activation address with 45 and then 128 addressable rows, alternately."""
    _, cabi = _lib()
    gen = _gen(21)
    n, k = 1024, 1024
    a, w = integer_data(128, n, k, gen, "cuda")
    a_wide, _ = integer_data(128, 8, 2 * k, gen, "cuda")
    w_wide = w.view(n // 2, 2 * k)                 # the same storage as [n / 2, 2 k]
    want = LR.linear_fp64(a, w, BF16)[0].to(BF16)
    want_wide = LR.linear_fp64(a_wide, w_wide, BF16)[0].to(BF16)
    for _ in range(2):
        for tile in (64, 128):
            rc, c = _run(a, w, 128, tile, 2)
            cabi.check(rc)
            _assert_exact(c, want, 128, n, f"w at tile {tile}")
            rc, c = _run(a_wide, w_wide, 128, tile, 2)
            cabi.check(rc)
            _assert_exact(c, want_wide, 128, n // 2, f"w storage as [n/2, 2k] at tile {tile}")
        rc, c = _run(a, w, 45, 64, 2, a_rows=45)
        cabi.check(rc)
        _assert_exact(c, want[:45], 45, n, "a with 45 addressable rows")
        rc, c = _run(a, w, 128, 64, 2, a_rows=128)
        cabi.check(rc)
        _assert_exact(c, want, 128, n, "the same a with 128 addressable rows")


def test_argument_errors_launch_nothing():
    _, cabi = _lib()
    a = torch.ones(136, 1024, dtype=BF16, device="cuda")
    w = torch.ones(264, 1024, dtype=BF16, device="cuda")
    c = torch.full((136, 272), NAN, dtype=BF16, device="cuda")
    U, E = cabi.LADE_EUNSUPPORTED, cabi.LADE_EINVAL
    off = lambda t: t.view(-1)[1:]                 # 2 bytes past a 16-byte boundary
    cases = [
        ("m = 0", dict(m=0), U), ("m = 129", dict(m=129), U), ("a_rows < m", dict(a_rows=63), U),
        ("n % 8", dict(n=260), U), ("n = 0", dict(n=0), U), ("k % 64", dict(k=1000), U), ("k = 0", dict(k=0), U),
        ("ldc < n", dict(ldc=256), U), ("ldc % 8", dict(ldc=268), U),
        ("a unaligned", dict(a=off(a)), E), ("w unaligned", dict(w=off(w)), E), ("c unaligned", dict(c=off(c)), E),
        ("tile 48", dict(tile_n=48), E), ("split 3", dict(split=3), E),
    ]
    for what, kw, code in cases:
        args = dict(a=a, w=w, c=c, m=64, n=264, k=1024, ldc=272, tile_n=0, split=0, a_rows=136)
        args.update(kw)
        rc = _launch(**args)
        assert rc == code, f"{what}: rc {rc}, documented {code}"
    torch.cuda.synchronize()
    assert torch.isnan(c).all()
    cabi.check(_launch(a, w, c, 64, 264, 1024, 272, a_rows=136))
    torch.cuda.synchronize()
    assert (c[:64, :264] == 1024).all() and torch.isnan(c[64:]).all() and torch.isnan(c[:, 264:]).all()
