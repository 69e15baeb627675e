"""The error bound of oracle.llama_ref.attention_fp64, checked without a GPU.

Each attention kernel's numerics are emulated in float64 with the model-dtype rounding points where the kernel has them:
  impl 2 (wgmma, default): online softmax over 128-column tiles, probabilities exp(s - running max) rounded to the model
         dtype before they are summed and multiplied, balanced KV splits merged with weights exp(m_s - m);
  impl 3 (reference order): probabilities normalised by the whole row, then rounded;
  impl 1 (mma.sync): 64-column tiles, rounded probabilities in P.V but the row sum adds the unrounded ones.
Every emulation must sit well inside the bound (worst element <= 0.6 of it), and the planted errors that an absolute
tolerance lets through at long contexts must break it."""
import math

import pytest
import torch

from oracle import llama_ref as LR
from oracle import lookahead as LA

DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}
KVS = [0, 1, 64, 127, 517, 1278, 3001]
HONEST_MAX = 0.6


def _kernel_scores(q, k, vis, dtype):
    """s = T(T(raw) * fp32(1/sqrt(D))) with raw summed in fp32, as the kernels form it; masked scores are -inf."""
    D = q.shape[-1]
    inv = torch.tensor(1.0, dtype=torch.float32) / torch.sqrt(torch.tensor(float(D), dtype=torch.float32))
    raw = q.float() @ k.float().transpose(1, 2)
    s = (raw.to(dtype).float() * inv).to(dtype).double()
    return s.masked_fill(~vis, -math.inf)


def _tiles(n_tiles, n_splits, balanced):
    """[(first tile, tile count)] of every active split: impl 2/3 balance the tiles, impl 1 gives ceil(n/splits) each."""
    if balanced:
        base, rem = divmod(n_tiles, n_splits)
        return [(s * base + min(s, rem), base + (s < rem)) for s in range(min(n_tiles, n_splits))]
    tps = -(-n_tiles // n_splits)
    return [(s * tps, min(tps, n_tiles - s * tps)) for s in range(-(-n_tiles // tps))]


def _online(s, v, dtype, n_splits, bn, round_sum, split_weight=None):
    """Split-KV online softmax over bn-column tiles; returns the merged fp64 output before the final rounding."""
    n_tiles = -(-s.shape[-1] // bn)
    parts = []
    for lo, cnt in _tiles(n_tiles, n_splits, balanced=(bn == 128)):
        m = torch.full(s.shape[:-1] + (1,), -math.inf, dtype=torch.float64)
        l = torch.zeros_like(m)
        o = torch.zeros(s.shape[:-1] + (v.shape[-1],), dtype=torch.float64)
        for j in range(lo, lo + cnt):
            st, vt = s[..., j * bn:(j + 1) * bn], v[:, j * bn:(j + 1) * bn]
            mt = st.amax(-1, keepdim=True)
            grow = mt > m
            scale = torch.where(grow & torch.isfinite(m), torch.exp(m - mt), 1.0)
            m = torch.where(grow, mt, m)
            e = torch.exp(st - torch.where(torch.isfinite(m), m, 0.0))
            pr = e.to(dtype).double()
            l = l * scale + (pr if round_sum else e).sum(-1, keepdim=True)
            o = o * scale + pr @ vt
        parts.append((m, l, o))
    mmax = torch.stack([m for m, _, _ in parts]).amax(0)
    acc, lsum = 0.0, 0.0
    for i, (m, l, o) in enumerate(parts):
        w = torch.where(torch.isfinite(m), torch.exp(m - torch.where(torch.isfinite(mmax), mmax, 0.0)), 0.0)
        if split_weight is not None and i == split_weight[0]:
            w = w * split_weight[1]
        acc, lsum = acc + w * o, lsum + w * l
    return torch.where(lsum > 0, acc / torch.where(lsum > 0, lsum, 1.0), 0.0)


def emulate(impl, q, k, v, vis, dtype, n_splits, scale_out=1.0, split_weight=None):
    """Output [Hq, R, D] (model dtype values, as float64) of the emulated kernel `impl`."""
    n_rep = q.shape[0] // k.shape[0]
    k, v = k.repeat_interleave(n_rep, 0), v.repeat_interleave(n_rep, 0).double()
    s = _kernel_scores(q, k, vis, dtype)
    if impl == 3:
        m = s.amax(-1, keepdim=True)
        e = torch.exp(s - torch.where(torch.isfinite(m), m, 0.0))
        l = e.sum(-1, keepdim=True)
        o = torch.where(l > 0, e / torch.where(l > 0, l, 1.0), 0.0).to(dtype).double() @ v
    else:
        o = _online(s, v, dtype, n_splits, 128 if impl == 2 else 64, round_sum=(impl == 2), split_weight=split_weight)
    return (o * scale_out).to(dtype).double()


def _case(kv_len, dtype, seed, peaked=False, Hq=2, Hkv=1):
    """The steady lookahead step of W=15, N=5, G=15 (120 rows) over kv_len cache rows, randn inputs; `peaked` scales
    Q so that the scaled scores span about +-25 instead of +-4."""
    g = torch.Generator().manual_seed(seed)
    lay = LA.layout_from_shape([14, 15, 15, 15], 1, 60, 4)
    T = kv_len + lay.q_len
    q = torch.randn(Hq, lay.q_len, 128, generator=g)
    if peaked:
        q = q * 6.0
    k = torch.randn(Hkv, T, 128, generator=g)
    v = torch.randn(Hkv, T, 128, generator=g)
    vis = LR.visibility(torch.from_numpy(LA.step_mask(lay)), kv_len)
    return q.to(dtype), k.to(dtype), v.to(dtype), vis, lay


def _ratios(got, o_ref, bound):
    r = LR.bound_ratio(got, o_ref, bound)
    return r.max().item(), r.mean().item()


@pytest.mark.parametrize("dtn", list(DTYPES))
@pytest.mark.parametrize("impl", [2, 3, 1])
def test_emulated_kernels_sit_inside_the_bound(impl, dtn):
    dtype = DTYPES[dtn]
    worst = 0.0
    for kv_len in KVS:
        if impl == 3 and kv_len + 120 > 384 * 8:
            continue                                   # impl 3 holds at most 8 splits of 3 tiles
        for peaked in (False, True):
            q, k, v, vis, _ = _case(kv_len, dtype, seed=kv_len + 7 * impl, peaked=peaked)
            o_ref, bound = LR.attention_fp64(q, k, v, vis, dtype)
            got = emulate(impl, q, k, v, vis, dtype, n_splits=4)
            mx, mean = _ratios(got, o_ref, bound)
            print(f"impl {impl} {dtn} kv {kv_len} peaked {peaked}: max {mx:.3f} mean {mean:.3f}")
            assert mx <= HONEST_MAX, (kv_len, peaked, mx)
            assert mean <= LR.MEAN_RATIO / 2, (kv_len, peaked, mean)
            worst = max(worst, mx)
    print(f"impl {impl} {dtn}: worst err/bound {worst:.3f}")


def test_rows_that_see_nothing_are_exactly_zero():
    q, k, v, vis, _ = _case(0, torch.bfloat16, seed=1)
    vis = vis.clone()
    vis[5] = False
    o_ref, bound = LR.attention_fp64(q, k, v, vis, torch.bfloat16)
    assert torch.all(o_ref[:, 5] == 0) and torch.all(bound[:, 5] < 1e-29)
    for impl in (1, 2, 3):
        assert torch.all(emulate(impl, q, k, v, vis, torch.bfloat16, 2)[:, 5] == 0)


@pytest.mark.parametrize("dtn", list(DTYPES))
@pytest.mark.parametrize("kv_len", [64, 517, 1278, 3001])
def test_planted_errors_break_the_bound(kv_len, dtn):
    """The errors an absolute 2e-2 / 2e-3 tolerance lets through from kv 517 on: one extra visible step column in one
    row, every output scaled by 1.01, one of four KV splits weighted by e^0.05 in the merge."""
    dtype = DTYPES[dtn]
    q, k, v, vis, lay = _case(kv_len, dtype, seed=kv_len)
    o_ref, bound = LR.attention_fp64(q, k, v, vis, dtype)
    honest = _ratios(emulate(2, q, k, v, vis, dtype, 4), o_ref, bound)
    assert honest[0] <= HONEST_MAX
    # a window row (it does not see most of the step block) gains the hidden step column it scores highest
    r = 10
    hidden = (~vis[r]).nonzero().flatten()
    s_row = _kernel_scores(q, k.repeat_interleave(2, 0), torch.ones_like(vis), dtype)[0, r]
    vis_bad = vis.clone()
    vis_bad[r, hidden[s_row[hidden].argmax()]] = True
    last_split = len(_tiles(-(-(kv_len + lay.q_len) // 128), 4, balanced=True)) - 1
    planted = {
        "extra column": emulate(2, q, k, v, vis_bad, dtype, 4),
        "scale 1.01": emulate(2, q, k, v, vis, dtype, 4, scale_out=1.01),
        "split weight e^0.05": emulate(2, q, k, v, vis, dtype, 4, split_weight=(last_split, math.exp(0.05))),
    }
    passed = []
    for name, got in planted.items():
        ok, mx, mean = LR.within_bound(got, o_ref, bound)
        print(f"kv {kv_len} {dtn} {name}: max {mx:.2f} mean {mean:.3f} (honest {honest[0]:.2f} / {honest[1]:.3f})")
        if ok:
            passed.append(name)
    assert not passed, f"planted errors inside the bound: {passed}"
