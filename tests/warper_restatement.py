"""TEST INFRASTRUCTURE ONLY -- float64 restatement of the sampling verification under HF's MinP / Epsilon / Eta
warpers, on top of ``oracle/sampling_device.py`` (temperature, top-k, top-p).

``softmax_T`` applies, each on the softmax of what is still kept and in HF's list order after top-p:
MinPLogitsWarper (drop p < min_p * max p), EpsilonLogitsWarper (drop p < epsilon unless the score is the maximum) and
EtaLogitsWarper (drop p < min(eta, sqrt(eta) exp(-entropy)) unless the score is the maximum; eta held in fp32 as HF's
tensor is); 0 switches each off, and with all three off the result is ``oracle.sampling_device.softmax_T``'s.  Tied
scores carry equal mass, so every cut keeps or drops them together.  ``tests/test_oracle_warpers.py`` pins it to HF's
own warper chain.  ``verify_given_uniforms`` is the reference's control flow (``sampling_device.verify_given_uniforms``)
with every row warped this way."""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np

from oracle import sampling_device as SD


def softmax_T(row: np.ndarray, temperature: float, top_k: int = 0, top_p: float = 1.0, min_p: float = 0.0,
              epsilon: float = 0.0, eta: float = 0.0) -> np.ndarray:
    base = SD.softmax_T(row, temperature, top_k, top_p)
    if not (min_p > 0.0 or epsilon > 0.0 or eta > 0.0):
        return base
    s = (row.astype(np.float32) / np.float32(temperature)).astype(np.float64)
    x = s - s.max()
    keep = base > 0
    e = np.where(keep, np.exp(x), 0.0)
    top = s == s.max()
    if min_p > 0.0:                                      # the top token's e is 1: p < min_p * max p  <=>  e < min_p
        keep &= e >= min_p
        e = np.where(keep, e, 0.0)
    if epsilon > 0.0:
        keep &= (e / e.sum() >= epsilon) | top
        e = np.where(keep, e, 0.0)
    if eta > 0.0:
        S = e.sum()
        ent = np.log(S) - float((e[keep] * x[keep]).sum()) / S
        ep = float(np.float32(eta))
        keep &= (e / S >= min(ep, np.sqrt(ep) * np.exp(-ent))) | top
        e = np.where(keep, e, 0.0)
    return e / e.sum()


def verify_given_uniforms(out_row: np.ndarray, guess_rows: Optional[np.ndarray], guess_tokens: Optional[Sequence[int]],
                          gs: int, temperature: float, uniforms: Sequence[float], top_k: int = 0, top_p: float = 1.0,
                          min_p: float = 0.0, epsilon: float = 0.0, eta: float = 0.0):
    """dict(hits, max_hit_idx, used, checks, n_hits) as ``sampling_device.verify_given_uniforms``."""
    warp = lambda r: softmax_T(r, temperature, top_k, top_p, min_p, epsilon, eta)      # noqa: E731
    it = iter(uniforms)
    checks = []
    hits: List[Optional[int]] = []
    max_hit_idx = 0
    used = 0
    if not guess_tokens:
        u = next(it); used += 1
        checks.append(("draw", u, warp(out_row)))
        return dict(hits=None, max_hit_idx=0, used=used, checks=checks, n_hits=1)
    probs_next = warp(out_row)
    n_ng = len(guess_tokens) // gs
    alive = list(range(n_ng))
    n_hits = 0
    for i in range(gs):
        accepted = False
        for e in list(alive):
            draft = guess_tokens[e * gs + i]
            p = min(1.0, float(probs_next[draft]))
            u = next(it); used += 1
            checks.append(("accept", u, p, draft))
            if u <= p:                                   # the kernel's rule on (0, 1]: sampling_device.py
                hits.append(draft)
                max_hit_idx = e
                alive = [g for g in alive if guess_tokens[g * gs + i] == draft]
                accepted = True
                row = guess_rows[e * gs + i]
                break
            probs_next = probs_next.copy()
            probs_next[draft] = 0.0
            tot = probs_next.sum()
            if tot > 0:
                probs_next = probs_next / tot
        if accepted:
            probs_next = warp(row)
            n_hits = i + 1
            continue
        u = next(it); used += 1
        checks.append(("draw", u, probs_next))
        n_hits = i + 1
        hits.append(None)
        break
    return dict(hits=hits, max_hit_idx=max_hit_idx, used=used, checks=checks, n_hits=n_hits)
