"""The error bound of the sampling accept chain (``csrc/sampling.cu``), checked without a GPU.

After the candidates Z were rejected at one position, the reference accepts candidate c with probability
p64 = e_c / sum over K \\ Z of e_t (K the warped kept set, e_t = exp(s_t - max), float64).  The kernel computes it
from fp32 e_t = __expf(x_t), x_t = s_t - max in fp32.  The bound the GPU tests hold every accept decision to is

    b = p64 (exp_rel(x_c) + eps_R + 3u) + u,     eps_R = sum over K \\ Z of e_t exp_rel(x_t) / sum of e_t
                                                          + (ceil(V / 1024) + 10) u

(u = 2^-24; exp_rel from ``test_gpu_sampling_kernel``): what a fresh block-wide sum of the remaining positive terms
achieves -- the per-term exp errors, ceil(V / 1024) strided adds per thread and 10 reduction levels -- plus the
division, the rounding of p to fp32 and the comparison with an fp32 uniform.  It does not depend on the depth of the
chain.

The emulations below run the chain's arithmetic in numpy fp32 (exp correctly rounded: the real __expf only adds error
the bound already carries):
* ``old``: the normaliser the kernel had, p = (e_c / S) / (1 - sum of rejected e_j / S) in fp32.  Its error grows like
  1 / (remaining mass): it breaks the bound at remaining mass 1e-3 and below, and on a light chain of 1000 rejections;
* ``new``: the normaliser the kernel has, the float64 kept mass not yet rejected (fresh block sum at the first
  rejection, then minus each rejected e_j, summed afresh below 2^-12 of the last fresh sum).  It stays within 0.6 b.

And the accept rule: u from curand_uniform lies in (0, 1]; accepting iff u <= p accepts with probability p (within
the fp32 grid of the uniforms), like the reference's random.random() < p on [0, 1), counted exactly over all 2^32
Philox words.  The strict u < p would reject a probability-1 token once in 2^25 draws."""
import math

import numpy as np
import pytest
import torch

from oracle import philox as PX
from test_gpu_sampling_kernel import U, exp_rel

HONEST_MAX = 0.6
THREADS = 1024
f32 = np.float32


# ---------------------------------------------------------------------------------------------- bound
def chain_bound(x, kept, z_mask, c, vocab):
    """(p64, b) of candidate c after rejecting the tokens of z_mask.  x: float64 of the fp32 differences s - max."""
    live = kept & ~z_mask
    e = np.where(live, np.exp(x), 0.0)
    tot = e.sum()
    p64 = e[c] / tot
    eps_r = float((e * exp_rel(x)).sum() / tot) + (math.ceil(vocab / THREADS) + 10) * U
    return p64, p64 * (float(exp_rel(x[c])) + eps_r + 3 * U) + U


def chain_bounds(x, kept, order, vocab):
    """(p64, b) of every decision of a chain that tests order[0], order[1], ... rejecting each in turn (distinct
    tokens): one pass of suffix sums instead of one V-long sum per rejection."""
    e = np.where(kept, np.exp(x), 0.0)
    er = e * exp_rel(x)
    ec, erc = e[order], er[order]
    # remaining before decision j: everything kept minus order[:j]
    rem = e.sum() - np.concatenate([[0.0], np.cumsum(ec)[:-1]])
    rem_tail = (e.sum() - ec.sum()) + np.cumsum(ec[::-1])[::-1]         # no cancellation: suffix sum + the rest
    rem_r = (er.sum() - erc.sum()) + np.cumsum(erc[::-1])[::-1]
    assert np.allclose(rem, rem_tail, rtol=1e-6)
    p64 = ec / rem_tail
    eps_r = rem_r / rem_tail + (math.ceil(vocab / THREADS) + 10) * U
    return p64, p64 * (exp_rel(x[order]) + eps_r + 3 * U) + U


# ---------------------------------------------------------------------------------------------- emulation
def fp32_block_sum(e):
    """The kernel's fp32 sum: thread t adds e[t], e[t + 1024], ... in order, then a tree over the 1024 partials."""
    n = -(-len(e) // THREADS) * THREADS
    cols = np.zeros(n, dtype=f32)
    cols[:len(e)] = e
    cols = cols.reshape(-1, THREADS)
    acc = np.zeros(THREADS, dtype=f32)
    for r in cols:
        acc = (acc + r).astype(f32)
    while len(acc) > 1:
        acc = (acc[0::2] + acc[1::2]).astype(f32)
    return acc[0]


def kernel_e(row, T=1.0):
    """fp32 e_t and the float64 x_t of a row of the model dtype (exp correctly rounded)."""
    s = (row.astype(f32) / f32(T)).astype(f32)
    xf = (s - s.max()).astype(f32)
    return np.exp(xf.astype(np.float64)).astype(f32), xf.astype(np.float64)


def p_old(e, S, order):
    """Accept probability of every decision under the subtract-based normaliser (the kernel before the fix)."""
    out, z = [], f32(0)
    for t in order:
        p_raw = f32(e[t] / S)
        d = f32(f32(1) - z)
        out.append(float(f32(p_raw / d)) if d > 0 else 1.0)
        z = f32(z + p_raw)
    return np.array(out)


def p_new(e, S, order, kept):
    """... under the float64 kept mass not yet rejected (fresh sums below 2^-12 of the last one)."""
    e64 = np.where(kept, e.astype(np.float64), 0.0)
    out, rem, ref, fresh = [], -1.0, 0.0, 0
    zmask = np.zeros(len(e), dtype=bool)
    for j, t in enumerate(order):
        if j == 0:
            out.append(float(f32(e[t] / S)))
        else:
            if not rem >= 2.0 ** -12 * ref:
                rem = ref = float(e64[~zmask].sum())
                fresh += 1
            out.append(min(1.0, float(f32(e64[t] / rem))))
        zmask[t] = True
        rem -= e64[t]
    return np.array(out), fresh


def chain_row(rng, vocab, k, remaining, dtype, cand_share=0.3, equal=False):
    """A row whose first k candidates carry 1 - remaining of the mass, candidate k cand_share of what remains and the
    rest of the vocabulary the others (equal: the k candidates share alike).  Returns (row rounded to dtype, order of
    the k + 1 candidates)."""
    p = np.zeros(vocab)
    order = rng.choice(vocab, k + 1, replace=False)
    p[order[:k]] = (np.full(k, 1.0 / k) if equal else rng.dirichlet(np.full(k, 4.0))) * (1 - remaining)
    p[order[k]] = cand_share * remaining
    bg = np.ones(vocab, dtype=bool)
    bg[order] = False
    w = rng.random(bg.sum()) + 0.5
    p[bg] = w / w.sum() * (1 - cand_share) * remaining
    row = torch.tensor(np.log(p), dtype=torch.float32).to(dtype).double().numpy()
    return row, order


def emulate(rng, vocab, k, remaining, dtype, equal=False):
    row, order = chain_row(rng, vocab, k, remaining, dtype, equal=equal)
    e, x = kernel_e(row)
    kept = np.ones(vocab, dtype=bool)
    S = fp32_block_sum(e)
    p64, b = chain_bounds(x, kept, order, vocab)
    old = p_old(e, S, order)
    new, fresh = p_new(e, S, order, kept)
    rem_true = 1.0 - np.where(kept, np.exp(x), 0)[order[:k]].sum() / np.exp(x).sum()
    return p64, b, old, new, fresh, rem_true


DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}
VOCABS = [32000, 128256, 152064]
REMAINING = [1e-1, 1e-2, 1e-3, 1e-4, 1e-5, 1e-6]


def test_bound_pieces_match_a_direct_evaluation():
    rng = np.random.default_rng(0)
    row, order = chain_row(rng, 4096, 5, 1e-2, torch.bfloat16)
    _, x = kernel_e(row)
    kept = np.ones(4096, dtype=bool)
    p64, b = chain_bounds(x, kept, order, 4096)
    for j in range(len(order)):
        z = np.zeros(4096, dtype=bool)
        z[order[:j]] = True
        q, bq = chain_bound(x, kept, z, order[j], 4096)
        assert abs(q - p64[j]) <= 1e-12 * q and abs(bq - b[j]) <= 1e-9 * bq


@pytest.mark.parametrize("remaining", [1e-3, 1e-4, 1e-6])
def test_old_normaliser_breaks_the_bound_at_small_remaining_mass(remaining):
    rng = np.random.default_rng(int(-math.log10(remaining)))
    worst = 0.0
    for k in (8, 60):
        p64, b, old, _, _, _ = emulate(rng, 152064, k, remaining, torch.bfloat16)
        worst = max(worst, float((np.abs(old - p64) / b).max()))
    print(f"remaining {remaining:g}: old normaliser err / b = {worst:.1f}")
    assert worst > 1.0


def test_old_normaliser_breaks_the_bound_on_a_light_chain():
    """1000 rejections of equal probability that together hold half of the mass: no cancellation to speak of, yet
    the 1000 fp32 adds of equal terms round the same way and drift past b (at V 32000, where b is tightest)."""
    rng = np.random.default_rng(1)
    p64, b, old, new, _, rem = emulate(rng, 32000, 1000, 0.5, torch.bfloat16, equal=True)
    assert 0.4 < rem < 0.6
    worst = float((np.abs(old - p64) / b).max())
    print(f"light chain: old normaliser err / b = {worst:.2f}, new {float((np.abs(new - p64) / b).max()):.3f}")
    assert worst > 1.0
    assert float((np.abs(new - p64) / b).max()) <= HONEST_MAX


@pytest.mark.parametrize("dtype", list(DTYPES), ids=list(DTYPES))
@pytest.mark.parametrize("vocab", VOCABS)
def test_new_normaliser_stays_within_the_bound(dtype, vocab):
    rng = np.random.default_rng(vocab)
    worst, fresh_max = 0.0, 0
    for remaining in REMAINING:
        for k in (8, 60, 1023):
            p64, b, _, new, fresh, rem = emulate(rng, vocab, k, remaining, DTYPES[dtype])
            assert 0.3 * remaining < rem < 3 * remaining
            r = np.abs(new - p64) / b
            worst = max(worst, float(r.max()))
            fresh_max = max(fresh_max, fresh)
            assert r.max() <= HONEST_MAX, f"remaining {remaining:g} k {k}: decision {int(r.argmax())} err / b {r.max():.2f}"
    print(f"{dtype} V {vocab}: new normaliser worst err / b = {worst:.3f}, at most {fresh_max} fresh sums per chain")


def test_new_normaliser_gives_a_sole_survivor_probability_one():
    """Every kept token but the last is rejected: the last one's p must be exactly 1 (no residual draw from an empty
    set), however small its mass."""
    for dtype in DTYPES.values():
        for tiny in (0.5, 1e-3, 1e-9, 1e-30):
            V = 64
            p = np.zeros(V)
            p[:V - 1] = (1 - tiny) / (V - 1)
            p[V - 1] = tiny
            row = torch.tensor(np.log(p), dtype=torch.float32).to(dtype).double().numpy()
            e, _ = kernel_e(row)
            if e[V - 1] == 0:
                continue                      # underflowed: not a kept token with mass
            new, _ = p_new(e, fp32_block_sum(e), list(range(V)), np.ones(V, dtype=bool))
            assert new[-1] == 1.0, (dtype, tiny, new[-1])


# ---------------------------------------------------------------------------------------------- accept rule
def _count_uniforms_le(p):
    """How many of the 2^32 Philox words give curand_uniform(word) <= p (the uniform is monotone in the word)."""
    lo, hi = 0, 1 << 32
    while lo < hi:
        m = (lo + hi) // 2
        if PX.to_uniform(np.uint32(m)) <= f32(p):
            lo = m + 1
        else:
            hi = m
    return lo


def _count_uniforms_lt(p):
    lo, hi = 0, 1 << 32
    while lo < hi:
        m = (lo + hi) // 2
        if PX.to_uniform(np.uint32(m)) < f32(p):
            lo = m + 1
        else:
            hi = m
    return lo


@pytest.mark.parametrize("p", [0.0, 2.0 ** -32, 1e-9, 0.5, 1 - 2.0 ** -24, 1.0])
def test_accept_rule_accepts_with_probability_p(p):
    """P(u <= p) over the (0, 1] stream.  curand_uniform rounds word * 2^-32 + 2^-33 to fp32, so its values near p
    are spaced one fp32 ulp apart: P equals p within half that spacing plus 2^-32 (exactly p at p = 0, 2^-32, 1)."""
    pf = float(f32(p))
    prob = _count_uniforms_le(pf) / 2.0 ** 32
    ulp = float(np.spacing(f32(pf))) if pf < 1 else 2.0 ** -24
    assert abs(prob - pf) <= ulp / 2 + 2.0 ** -32, (p, prob - pf)
    if pf in (0.0, 2.0 ** -32, 1.0):
        assert prob == pf
    if pf == 1.0:
        assert _count_uniforms_lt(1.0) / 2.0 ** 32 == 1 - 2.0 ** -25      # the strict rule rejects p = 1 sometimes
