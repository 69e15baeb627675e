"""TEST INFRASTRUCTURE ONLY -- restatement of the sampling verification of ``jacobi_sample_multilevel``
(``/root/reference/lade/decoding.py:445-546``) as a pure function of the uniforms it consumes.

The reference draws ``random.random()`` per accept test (``:507``) and ``torch.multinomial`` for the residual / plain
draw (``:462,:472,:533,:545``).  The device kernel (``lade_sample_verify``) runs the same procedure on one Philox
stream and can export the uniforms it used; ``verify_given_uniforms`` replays the reference's control flow with those
numbers, so the kernel's decision can be checked exactly (up to a uniform landing within float rounding of a
threshold, which the caller may skip).  Multinomial = inverse CDF over the surviving tokens in index order.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np


def softmax_T(row: np.ndarray, temperature: float, top_k: int = 0, top_p: float = 1.0) -> np.ndarray:
    """softmax of the warped scores in float64: TemperatureLogitsWarper (row / T, fp32), TopKLogitsWarper (keep every
    score >= the k-th largest), TopPLogitsWarper (ascending cumulative probability of the filtered softmax: drop while
    cum <= 1 - top_p, keep at least one) -- the warpers the reference admits (:375-377,:445,:485-489).  Scores of equal
    value are kept or dropped together (torch.sort leaves their order, hence HF's cut inside such a group, undefined);
    `tests/test_oracle_sampling_device.py` pins this function to the HF warpers on tie-free rows."""
    s = (row.astype(np.float32) / np.float32(temperature)).astype(np.float64)
    keep = np.ones(s.shape, dtype=bool)
    if top_k and top_k < s.size:
        kth = np.sort(s)[-top_k]
        keep &= s >= kth
    e = np.where(keep, np.exp(s - s.max()), 0.0)
    if top_p < 1.0:
        lim = (1.0 - top_p) * e.sum()
        vals = np.unique(s[keep])                        # ascending
        cum = 0.0
        thr = vals[-1]
        for v in vals:
            m = e[s == v].sum()
            if not (cum + m <= lim):
                thr = v
                break
            cum += m
        keep &= s >= min(thr, vals[-1])
        e = np.where(keep, e, 0.0)
    return e / e.sum()


def verify_given_uniforms(out_row: np.ndarray, guess_rows: Optional[np.ndarray], guess_tokens: Optional[Sequence[int]], gs: int,
                          temperature: float, uniforms: Sequence[float], top_k: int = 0, top_p: float = 1.0):
    """Returns dict(hits, max_hit_idx, used, checks) where `checks` lists every comparison made:
    ("accept", u, p) or ("draw", u, probs) so that the caller can judge near-threshold cases."""
    it = iter(uniforms)
    checks = []
    hits: List[int] = []
    max_hit_idx = 0
    used = 0
    if not guess_tokens:                                                                   # :458-480,:543-546
        u = next(it); used += 1
        probs = softmax_T(out_row, temperature, top_k, top_p)
        checks.append(("draw", u, probs))
        return dict(hits=None, max_hit_idx=0, used=used, checks=checks, n_hits=1)
    probs_next = softmax_T(out_row, temperature, top_k, top_p)
    n_ng = len(guess_tokens) // gs
    alive = list(range(n_ng))
    n_hits = 0
    for i in range(gs):                                                                    # :491
        accepted = False
        for e in list(alive):                                                              # :495
            draft = guess_tokens[e * gs + i]
            p = min(1.0, float(probs_next[draft]))                                         # :505
            u = next(it); used += 1
            checks.append(("accept", u, p, draft))
            if u <= p:                                    # :508 r < p for r in [0, 1) == u <= p for u in (0, 1]
                hits.append(draft)
                max_hit_idx = e
                alive = [g for g in alive if guess_tokens[g * gs + i] == draft]            # :513-516
                accepted = True
                row = guess_rows[e * gs + i]
                break
            probs_next = probs_next.copy()
            probs_next[draft] = 0.0                                                        # :518-520
            tot = probs_next.sum()
            if tot > 0:
                probs_next = probs_next / tot
        if accepted:
            probs_next = softmax_T(row, temperature, top_k, top_p)                         # :530
            n_hits = i + 1
            continue
        u = next(it); used += 1                                                            # :533
        checks.append(("draw", u, probs_next))
        n_hits = i + 1
        hits.append(None)                       # to be filled by the caller's draw check
        break
    return dict(hits=hits, max_hit_idx=max_hit_idx, used=used, checks=checks, n_hits=n_hits)


def draw_is_consistent(u: float, probs: np.ndarray, token: int, rel_eps: float = 2e-5) -> bool:
    """`token` is the inverse-CDF pick for u (uniform in (0,1]) within a float-rounding margin."""
    c = np.cumsum(probs)
    lo = c[token - 1] if token > 0 else 0.0
    hi = c[token]
    target = u * c[-1]
    return probs[token] > 0 and (lo - rel_eps * c[-1]) <= target <= (hi + rel_eps * c[-1])
