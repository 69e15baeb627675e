"""``lade_sample_verify_warped`` / ``_f16``: the sampling verification under MinP / Epsilon / Eta, against float64.

Launched directly on crafted logits through the harness of ``test_gpu_sampling_kernel.py`` (a tiny engine's ctx,
guess tokens written into the device state, every uniform known from the host Philox), plus the engine and the
``generate()`` surface end to end:

* cuts off: records, exported uniforms and the offset advance equal ``lade_sample_verify``'s bit for bit;
* kept set: rows with tokens one key step either side of each cut; the kernel's threshold key equals the float64 one
  (only where the float64 margin of both neighbours exceeds the fp32 error bound), S' matches, and 4096 plain draws
  per row are each the float64 inverse-CDF token;
* accept probes 1.25 to 4 error bounds either side of the float64 accept probability with each cut on;
* the chain after an accept at n-gram e > 0, and a G-test of the emitted (hits, max_hit_idx) against the exact
  enumeration with min_p and with eta on;
* engine: graph == eager, pipelined == synchronous, T -> 0 == greedy, first-token frequencies, and the plugin routes
  ``generate(do_sample=True, min_p=...)`` to the device (host loop under SAMPLING_ON_HOST)."""
import math
import random

import numpy as np
import pytest
import torch

from oracle import philox as PX
from oracle import sampling_device as SD
import warper_restatement as WR
from test_gpu_sampling_kernel import (DTYPES, GS, R, REC, U, WCAP, Harness, _g_test, _offset_where, bits_of,
                                      exp_rel, find_probes, host_rows, logits_tensor, probe_row, step_rows)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", params=DTYPES, ids=["bf16", "fp16"])
def H(request):
    h = Harness(request.param)
    h.cuts = torch.zeros(1 + 2 * GS, dtype=torch.float32, device="cuda")
    h.fn_w = h.eng.k_sample_verify_warped
    yield h
    h.eng.close()


def launch_w(h, logits, vocab, meta, T, top_k=0, top_p=1.0, min_p=0.0, epsilon=0.0, eta=0.0, rec=None, dbg=True):
    rec = torch.full((REC,), -7, dtype=torch.int32, device="cuda") if rec is None else rec
    w = h.C.LadeWarpers(float(T), int(top_k), float(top_p), float(min_p), float(epsilon), float(eta))
    stream = torch.cuda.current_stream().cuda_stream
    import ctypes as C
    h.C.check(h.fn_w(h.eng._ctx, stream, logits.data_ptr(), logits.shape[1], vocab, h.am.data_ptr(), meta.data_ptr(),
                     C.byref(w), h.rng.data_ptr(), rec.data_ptr(), h.dbg.data_ptr() if dbg else 0,
                     h.cuts.data_ptr() if dbg else 0), "lade_sample_verify_warped")
    return rec


def cuts_of(h):
    c = h.cuts.cpu().numpy()
    n = int(c[0])
    return [(int(c[1 + 2 * i]), float(c[2 + 2 * i])) for i in range(n)]


def keys_of(h, t, vocab):
    """The kernel's 16-bit order key of every logit (key_of in csrc/sampling.cu)."""
    b = t[0, :vocab].view(torch.int16).cpu().numpy().astype(np.int64) & 0xFFFF
    b = np.where(b == 0x8000, 0, b)
    return np.where(b & 0x8000, ~b & 0xFFFF, b | 0x8000)


# ---------------------------------------------------------------------------------------------- cuts off
def test_cuts_off_is_bit_identical_to_lade_sample_verify(H):
    rng = np.random.default_rng(1)
    vocab = 4096
    row0 = rng.normal(0, 1.0, vocab)
    toks = [11, 12, 13, 21, 22, 23, 31, 32, 33]
    row0[[11, 21, 31]] += 7.5
    guess = {}
    for j in range(len(toks)):
        guess[j] = rng.normal(0, 1.0, vocab)
        if (j + 1) % GS:
            guess[j][toks[j + 1]] += 7.5
    lg = step_rows(H, row0, guess)
    n = 0
    for meta, params in [(H.set_guess(toks), (1.0, 0, 1.0)), (H.set_guess(toks), (0.7, 50, 0.9)),
                         (H.plain_meta(), (1.3, 0, 0.95))]:
        for seed in (3, 2 ** 62 + 5):
            for it in range(200 // 6 + 1):
                off = 4 * it + 1
                H.seed(seed, off)
                a = H.launch(lg, vocab, meta, *params).cpu()
                ua, sa = H.exported().copy(), H.rng.cpu()
                H.seed(seed, off)
                b = launch_w(H, lg, vocab, meta, *params).cpu()
                ub, sb = H.exported().copy(), H.rng.cpu()
                assert torch.equal(a, b) and torch.equal(sa, sb), f"seed {seed} launch {it}"
                assert np.array_equal(bits_of(ua), bits_of(ub))
                n += 1
    assert n >= 200


# ---------------------------------------------------------------------------------------------- error bounds
def kept_bounds(row, T, top_k, top_p, vocab):
    """Bounds on the fp32 quantities of the cuts at the float64 distribution before them: the relative error of S
    (summed e_t) and the absolute error of the entropy H = ln S - sum e x / S."""
    p = WR.softmax_T(row, T, top_k, top_p)
    s = (row.astype(np.float32) / np.float32(T)).astype(np.float64)
    x = s - s.max()
    kept = p > 0
    s_err = float((p[kept] * exp_rel(x[kept])).sum()) + (math.ceil(vocab / 1024) + 10) * U + \
        (vocab * 2.0 ** -41 if top_p < 1.0 else 0.0)
    ax = np.abs(x[kept])
    mx = float((p[kept] * ax).sum())
    # sum e x: each term e(1 + exp_rel)(x)(1 + u) plus the fp32 adds (ceil(V/1024) + 10 levels, u of the running sum
    # of |e x| each); divided by S (s_err + u); ln S: s_err + 2 ulp of ln S
    h_err = float((p[kept] * ax * (exp_rel(x[kept]) + U)).sum()) + (math.ceil(vocab / 1024) + 10) * U * mx + \
        mx * (s_err + U) + s_err + 4 * U * abs(math.log(max(float(np.exp(x[kept]).sum()), 1e-300)))
    return s_err, h_err


def cut_margin_ok(row, T, top_k, top_p, cut, vocab):
    """True when every token's keep decision has a float64 margin over the fp32 bound: at 1.5 bounds the kernel and
    float64 agree on the kept set."""
    s = (row.astype(np.float32) / np.float32(T)).astype(np.float64)
    x = s - s.max()
    e = np.exp(x)
    p_prev = WR.softmax_T(row, T, top_k, top_p)
    kept = p_prev > 0
    s_err, h_err = kept_bounds(row, T, top_k, top_p, vocab)
    top = s == s.max()
    if cut.get("min_p"):
        mp = cut["min_p"]
        m = kept & (x != 0)                              # __expf(0) is exactly 1: min_p = 1 keeps the top tie group
        rel = np.abs(e[m] - mp) / mp
        if (rel <= 1.5 * (exp_rel(x[m]) + U)).any():
            return False
        p_prev = WR.softmax_T(row, T, top_k, top_p, min_p=mp)
        kept = p_prev > 0
    if cut.get("epsilon"):
        eps = cut["epsilon"]
        m = kept & ~top
        rel = np.abs(p_prev[m] - eps) / eps
        if (rel <= 1.5 * (exp_rel(x[m]) + 2 * s_err + 2 * U)).any():
            return False
        p_prev = WR.softmax_T(row, T, top_k, top_p, cut.get("min_p", 0.0), eps)
        kept = p_prev > 0
    if cut.get("eta"):
        ep = float(np.float32(cut["eta"]))
        S = e[kept].sum()
        ent = math.log(S) - float((e[kept] * x[kept]).sum()) / S
        eta = min(ep, math.sqrt(ep) * math.exp(-ent))
        m = kept & ~top
        eta_err = (2 * h_err + 6 * U) if eta < ep else 2 * U
        rel = np.abs(p_prev[m] - eta) / eta
        if (rel <= 1.5 * (exp_rel(x[m]) + 2 * s_err + eta_err + 2 * U)).any():
            return False
    return True


# ---------------------------------------------------------------------------------------------- kept set
def _step(h, v, k):
    """v moved k representable steps of the harness dtype (k < 0: downwards)."""
    t = torch.tensor([v], dtype=torch.float32).to(h.dtype)
    for _ in range(abs(k)):
        b = t.view(torch.int16).item()
        up = k > 0
        if t.item() == 0:
            b = 1 if up else -32767
        elif (t.item() > 0) == up:
            b += 1
        else:
            b -= 1
        t = torch.tensor([b], dtype=torch.int16).view(h.dtype)
    return t.float().item()


def _ladder(h, r, lo_tok, centre, n=24):
    """Tokens lo_tok.. at 2n consecutive values of the dtype around `centre` (one key step apart)."""
    c = torch.tensor([centre], dtype=torch.float32).to(h.dtype).float().item()
    for j in range(-n, n):
        r[lo_tok + j + n] = _step(h, c, j)


def warper_cases(h):
    """(name, row, vocab, T, top_k, top_p, cut, pad)."""
    rng = np.random.default_rng(17)
    cases = []
    V = 32000
    for T in (0.05, 1.0, 4.0):
        for top_k, top_p in ((0, 1.0), (300, 1.0), (0, 0.97)):
            # min_p: the cut in logit space sits at T * ln(min_p) below the maximum
            r = rng.normal(0, 1.0, V) * T; r[7] = 4.0 * T
            mp = 0.05
            _ladder(h, r, 1000, 4.0 * T + T * math.log(mp))
            cases.append((f"min_p T={T} k={top_k} p={top_p}", r, V, T, top_k, top_p, dict(min_p=mp), None))
            # epsilon / eta: the cut is a probability; place the ladder at the score of that probability
            for kind, val in (("epsilon", 3e-4), ("eta", 2e-3)):
                r = rng.normal(0, 1.0, V) * T; r[7] = 4.0 * T
                lt = logits_tensor(h, r)
                p = WR.softmax_T(host_rows(lt, V)[0], T, top_k, top_p)
                s = host_rows(lt, V)[0] / T
                S = np.exp(s - s.max())[p > 0].sum()
                level = val
                if kind == "eta":
                    q = p[p > 0]
                    ent = float(-(q * np.log(q)).sum())
                    level = min(val, math.sqrt(val) * math.exp(-ent))
                _ladder(h, r, 1000, T * (s.max() + math.log(level * S)))
                cases.append((f"{kind} T={T} k={top_k} p={top_p}", r, V, T, top_k, top_p, {kind: val}, None))
    r = rng.normal(0, 1.0, V); r[[3, 9, 40]] = 5.0
    for cut in (dict(min_p=1.0), dict(epsilon=0.9), dict(eta=0.9)):
        cases.append((f"tie at the maximum {cut}", r, V, 1.0, 0, 1.0, cut, float("nan")))
    r = rng.uniform(-30, -20, 4096); r[[1, 2]] = 0.0; r[3] = -0.0; r[[4, 5]] = -0.01; r[6] = 0.5
    cases.append(("+0 and -0 at the min_p cut", r, 4096, 1.0, 0, 1.0, dict(min_p=math.exp(-0.505)), None))
    r = rng.normal(0, 1.0, 4096); r[:8] += 3.0
    cases.append(("all three", r, 4096, 1.0, 0, 1.0, dict(min_p=0.01, epsilon=1e-4, eta=1e-3), float("nan")))
    return cases


def _draws_w(h, logits, vocab, T, top_k, top_p, cut, seed, offset, n):
    meta = h.plain_meta()
    recs = torch.zeros(n, REC, dtype=torch.int32, device="cuda")
    h.seed(seed, offset)
    for j in range(n):
        launch_w(h, logits, vocab, meta, T, top_k, top_p, rec=recs[j], dbg=False, **cut)
    assert h.rng.cpu().tolist() == [seed, offset + 4 * n]
    u = PX.uniforms(seed, offset + 4 * np.arange(n, dtype=np.uint64), 1)[:, 0]
    return recs[:, 3].cpu().numpy(), u


def test_kept_set_threshold_and_inverse_cdf(H):
    from test_gpu_sampling_kernel import _check_draws
    checked = 0
    for i, (name, row, vocab, T, top_k, top_p, cut, pad) in enumerate(warper_cases(H)):
        logits = logits_tensor(H, row, ld=vocab + 13, pad=pad)
        hrow = host_rows(logits, vocab)[0]
        if not cut_margin_ok(hrow, T, top_k, top_p, cut, vocab):
            continue
        probs = WR.softmax_T(hrow, T, top_k, top_p, **cut)
        before = WR.softmax_T(hrow, T, top_k, top_p)
        keys = keys_of(H, logits, vocab)
        H.seed(1, 0)
        launch_w(H, logits, vocab, H.plain_meta(), T, top_k, top_p, **cut)
        (thr, S1), = cuts_of(H)
        kept64 = probs > 0
        assert (keys >= thr).tolist() == kept64.tolist(), f"{name}: kernel kept {(keys >= thr).sum()}, " \
            f"float64 {kept64.sum()}"
        if kept64.sum() < (before > 0).sum():
            assert thr == keys[kept64].min(), name
            s = hrow / T
            S64 = np.exp(s - s.max())[kept64].sum()
            assert abs(S1 - S64) <= 1e-5 * S64, f"{name}: S' {S1} vs {S64}"
        toks, u = _draws_w(H, logits, vocab, T, top_k, top_p, cut, 11 + i, 8 * i, 4096)
        _check_draws(probs, toks, u, name)
        checked += 1
    print(f"{checked} kept-set cases checked")
    assert checked >= 12


# ---------------------------------------------------------------------------------------------- accept probes
def accept_bound_w(row, T, top_k, top_p, cut, vocab, cands, k):
    """accept_bound of test_gpu_sampling_kernel for the distribution after the cuts: S' is an fp32 sum over the final
    kept set once a cut moved the threshold (and the top-p integer mass otherwise, covered by the same bound)."""
    p_row = WR.softmax_T(row, T, top_k, top_p, **cut)
    s = (row.astype(np.float32) / np.float32(T)).astype(np.float64)
    x = s - s.max()
    kept = p_row > 0
    s_err = float((p_row[kept] * exp_rel(x[kept])).sum()) + (math.ceil(vocab / 1024) + 10) * U + \
        (vocab * 2.0 ** -41 if top_p < 1.0 else 0.0)
    raw = lambda t: p_row[t]                                                  # noqa: E731
    z = sum(raw(c) for c in cands[:k])
    z_abs = sum(raw(c) * (exp_rel(x[c]) + s_err + 2 * U) for c in cands[:k])
    p = raw(cands[k]) / (1.0 - z)
    rel = exp_rel(x[cands[k]]) + s_err + 2 * U + z_abs / (1.0 - z)
    return p, min(1.0, p) * rel + U, [raw(c) / (1.0 - sum(raw(c2) for c2 in cands[:j])) for j, c in enumerate(cands[:k])]


PROBE_TARGETS = [(0.05, 1), (0.3, 3), (0.5, 4), (0.9, 2), (0.6, 0)]
PROBE_CUTS = [dict(min_p=0.02), dict(epsilon=2e-3), dict(eta=1e-2), dict(min_p=0.01, epsilon=1e-3, eta=5e-3)]


@pytest.mark.parametrize("cut", PROBE_CUTS, ids=lambda c: ",".join(c))
@pytest.mark.parametrize("T,top_k,top_p", [(1.0, 0, 1.0), (0.05, 0, 1.0), (4.0, 40, 1.0), (1.0, 0, 0.995)])
def test_accept_probability_with_cuts_matches_float64(H, cut, T, top_k, top_p):
    rng = np.random.default_rng(int(T * 100) + len(cut))
    vocab, seed = 32000, 99
    checked = 0
    for p_t, k in PROBE_TARGETS:
        lg, cands = probe_row(rng, vocab, T, p_t, k)
        logits = step_rows(H, lg, ld=vocab + 8)
        row = host_rows(logits, vocab)[0]
        if not cut_margin_ok(row, T, top_k, top_p, cut, vocab):
            continue
        p64, b, rejects = accept_bound_w(row, T, top_k, top_p, cut, vocab, cands, k)
        if not 0 < p64 or any(r >= 0.999 for r in rejects):
            continue
        if (WR.softmax_T(row, T, top_k, top_p, **cut) > 0).sum() == (WR.softmax_T(row, T, top_k, top_p) > 0).sum():
            continue                                   # top-k alone already keeps less than the cut would
        meta = H.set_guess([t for c in cands for t in (c, 5, 6)])
        sides = [("accept", p64 - 4 * b, p64 - 1.25 * b)]
        if p64 + 1.25 * b < 1.0:
            sides.append(("reject", p64 + 1.25 * b, min(1.0, p64 + 4 * b)))
        for kind, lo, hi in sides:
            for o in find_probes(seed, k, rejects, lo, hi, 2):
                H.seed(seed, int(o))
                rec = launch_w(H, logits, vocab, meta, T, top_k, top_p, **cut).cpu().tolist()
                u = H.exported()
                accepted = rec[3] == cands[k]
                assert accepted == (kind == "accept"), \
                    f"T={T} {cut} k={k}: p64={p64:.9g} b={b:.3g} u={float(u[k]):.9g} ({(u[k] - p64) / b:+.2f} b)"
                assert len(cuts_of(H)) == (2 if accepted else 1)
                checked += 1
    assert checked >= 6 or (top_k and checked >= 2)


# ---------------------------------------------------------------------------------------------- chain, distribution
def test_chain_after_an_accept_at_a_later_ngram_warps_that_row(H):
    """n-gram 1 wins position 0; its row 1 + WCAP + GS is the next distribution, and min_p cuts it: the tokens the cut
    removes there are never emitted, and every visited row reports its own cut."""
    rng = np.random.default_rng(23)
    vocab = 4096
    guess = [50, 51, 52, 60, 61, 62]
    row0 = rng.normal(0, 1.0, vocab); row0[[50, 60]] = [9.0, 9.0]
    gr = {GS: rng.normal(0, 1.0, vocab)}
    gr[GS][[61, 70, 71]] = [8.0, 8.0, 5.0]            # min_p 0.1 keeps 61 and 70 (e = 1), drops 71 (e ~ 0.05)
    logits = step_rows(H, row0, gr)
    rows = host_rows(logits, vocab)
    cut = dict(min_p=0.1)
    meta = H.set_guess(guess)
    seen = set()
    for trial in range(40):
        off = _offset_where(31 + trial, lambda u: u[0] > 0.6 and u[1] < 0.9)
        H.seed(31 + trial, off)
        rec = launch_w(H, logits, vocab, meta, 1.0, **cut).cpu().tolist()
        us = PX.uniforms(31 + trial, off, 16).astype(np.float64)
        want = WR.verify_given_uniforms(rows[0], rows[1 + WCAP:], guess, GS, 1.0, us.tolist(), **cut)
        assert rec[3] == 60 and rec[R] == 1 and want["hits"][0] == 60
        n_hits = rec[1] + 1
        assert n_hits == want["n_hits"]
        if n_hits > 1:
            if want["hits"][1] is None:
                _, u, probs = [c for c in want["checks"] if c[0] == "draw"][-1][:3]
                assert SD.draw_is_consistent(u, probs, rec[4])
            else:
                assert rec[4] == want["hits"][1]
            seen.add(rec[4])
            assert rec[4] != 71 and rec[4] in (61, 70)
            c = cuts_of(H)
            assert len(c) >= 2 and c[1][0] == int(keys_of(H, logits[1 + WCAP + GS:], vocab)[70])
    assert seen == {61, 70}


def enumerate_outcomes_w(rows, guess, T, cut):
    out = {}
    n_ng = len(guess) // GS

    def add(key, w):
        out[key] = out.get(key, 0.0) + w

    def pos(i, alive, probs, hits, mhi, w):
        probs = probs.copy()
        for e in alive:
            d = guess[e * GS + i]
            p = min(1.0, float(probs[d]))
            if p > 0:
                h2 = hits + (d,)
                if i + 1 == GS:
                    add((h2, e), w * p)
                else:
                    pos(i + 1, [g for g in alive if guess[g * GS + i] == d],
                        WR.softmax_T(rows[1 + WCAP + e * GS + i], T, **cut), h2, e, w * p)
            w *= 1.0 - p
            if w <= 0:
                return
            probs[d] = 0.0
            probs = probs / probs.sum()
        for t in np.nonzero(probs)[0]:
            add((hits + (int(t),), mhi if hits else 0), w * float(probs[t]))

    pos(0, list(range(n_ng)), WR.softmax_T(rows[0], T, **cut), (), 0, 1.0)
    return out


@pytest.mark.parametrize("cut", [dict(min_p=0.02), dict(eta=2e-2)], ids=["min_p", "eta"])
def test_emitted_distribution_with_cuts_matches_exact_enumeration(H, cut):
    rng = np.random.default_rng(9)
    vocab = 2048
    guess = [10, 11, 12, 10, 14, 15, 20, 21, 22]
    row0 = rng.normal(0, 1.0, vocab); row0[[10, 20, 30]] = [7.5, 7.0, 6.5]
    gr = {}
    for j in range(3 * GS):
        r = rng.normal(0, 1.0, vocab)
        r[guess[j + 1] if (j + 1) % GS else 5] += 7.0
        r[14] += 6.5 if j == 0 else 0.0
        gr[j] = r
    logits = step_rows(H, row0, gr)
    rows = host_rows(logits, vocab)
    for r in [rows[0]] + [rows[1 + WCAP + j] for j in range(3 * GS)]:
        assert cut_margin_ok(r, 1.0, 0, 1.0, cut, vocab)
        assert (WR.softmax_T(r, 1.0, **cut) > 0).sum() < (WR.softmax_T(r, 1.0) > 0).sum()
    exact = enumerate_outcomes_w(rows, guess, 1.0, cut)
    assert abs(sum(exact.values()) - 1.0) < 1e-9
    n = 1 << 16
    meta = H.set_guess(guess)
    recs = torch.zeros(n, REC, dtype=torch.int32, device="cuda")
    H.seed(4243, 0)
    for j in range(n):
        launch_w(H, logits, vocab, meta, 1.0, rec=recs[j], dbg=False, **cut)
    obs = {}
    for r in recs.cpu().numpy():
        nh = int(r[1]) + 1
        key = (tuple(int(x) for x in r[3:3 + nh]), int(r[R]) if nh > 1 else 0)
        obs[key] = obs.get(key, 0) + 1
    assert set(obs) <= set(exact), f"outcomes the procedure cannot emit: {sorted(set(obs) - set(exact))[:3]}"
    g, df, p = _g_test(obs, exact, n)
    print(f"{cut}: G = {g:.1f} on {df} dof, p = {p:.3g}")
    assert p > 1e-6 and df >= 10


# ---------------------------------------------------------------------------------------------- engine end to end
CUT_SETS = [dict(min_p=0.05), dict(min_p=0.05, epsilon=3e-4, eta=2e-3)]


def test_engine_graph_equals_eager_and_pipelined_equals_synchronous():
    from lookaheaddecoding_b200 import LookaheadEngine
    from test_gpu_sampling_device import _in_cycle_prompt, peaked_periodic_model
    model = peaked_periodic_model(scale=8.0)
    prompt = _in_cycle_prompt(model, 32)
    outs = {}
    for graph, pipe in ((False, False), (True, False), (True, True)):
        eng = LookaheadEngine(model, 7, 4, 7, pool_from_prompt=True, max_total_len=32 + 64, use_cuda_graph=graph,
                              pipeline_host=pipe)
        res = []
        for cut in CUT_SETS:
            res.append(eng.generate(prompt, 64, rng=random.Random(1),
                                    sampling=dict(temperature=1.0, top_k=0, seed=11, **cut)))
        res.append(eng.generate(prompt, 64, rng=random.Random(1), sampling=dict(temperature=1.0, seed=11)))
        eng.close()
        outs[(graph, pipe)] = res
    assert outs[(False, False)] == outs[(True, False)] == outs[(True, True)]
    assert len({tuple(r) for r in outs[(True, True)]}) >= 2, "the cuts never changed a draw"


def test_low_temperature_with_min_p_reproduces_greedy():
    from lookaheaddecoding_b200 import LookaheadEngine
    from test_gpu_sampling_device import _assert_equal_up_to_a_tie, _in_cycle_prompt, peaked_periodic_model
    model = peaked_periodic_model(scale=30.0)
    prompt = _in_cycle_prompt(model, 32)
    eng = LookaheadEngine(model, 7, 4, 7, pool_from_prompt=True, max_total_len=32 + 64)
    greedy = eng.generate(prompt, 64, rng=random.Random(1))
    cold = eng.generate(prompt, 64, rng=random.Random(1),
                        sampling={"temperature": 0.02, "min_p": 0.1, "epsilon": 1e-4, "seed": 7})
    assert eng.last_steps < 64
    _assert_equal_up_to_a_tie(model, cold, greedy, "T=0.02 min_p=0.1")
    eng.close()


@pytest.mark.parametrize("cut", [dict(min_p=0.1), dict(eta=0.02)], ids=["min_p", "eta"])
def test_first_token_follows_the_warped_softmax(cut):
    from lookaheaddecoding_b200 import LookaheadEngine
    from test_gpu_sampling_device import _prompt, peaked_periodic_model
    from scipy.stats import chi2 as chi2_dist
    model = peaked_periodic_model(scale=4.0)
    prompt = _prompt(16, seed=5)
    eng = LookaheadEngine(model, 5, 3, 3, max_total_len=16 + 8, use_cuda_graph=False)
    T, n = 0.9, 1200
    counts = {}
    for s in range(n):
        out = eng.generate(prompt, 1, rng=random.Random(0), sampling=dict(temperature=T, seed=s, **cut))
        counts[out[-1]] = counts.get(out[-1], 0) + 1
    row = eng.logits[0].float().cpu().numpy().astype(np.float64)
    probs = WR.softmax_T(row, T, **cut)
    assert 1 < (probs > 0).sum() < (WR.softmax_T(row, T) > 0).sum(), "the cut must matter on this row"
    assert set(counts) <= set(np.nonzero(probs)[0].tolist()), "a token the cut removes was drawn"
    cells = [int(t) for t in np.argsort(-probs)[:12] if n * probs[t] >= 5]
    obs = [counts.get(t, 0) for t in cells]
    exp = [n * probs[t] for t in cells]
    rest_e = n - sum(exp)
    if rest_e >= 5:
        obs.append(n - sum(obs)); exp.append(rest_e)
    chi2 = sum((o - e) ** 2 / e for o, e in zip(obs, exp))
    p = chi2_dist.sf(chi2, len(obs) - 1)
    print(f"{cut}: chi2 = {chi2:.2f} on {len(obs) - 1} dof, p = {p:.3g}")
    assert len(obs) >= 3 and p > 1e-4
    eng.close()


def _plugin_generate(monkeypatch, on_host, **kw):
    import lade
    from lookaheaddecoding_b200 import engine as E
    from lookaheaddecoding_b200 import sampling as S
    from lookaheaddecoding_b200.decoding import CONFIG_MAP
    from test_gpu_sampling_device import _prompt, peaked_periodic_model
    model = peaked_periodic_model(scale=12.0)
    model.generation_config.pad_token_id = 0
    model.generation_config.eos_token_id = None
    ids = torch.tensor([_prompt(24, seed=4)], device="cuda")
    calls = {"device": [], "host": 0}
    orig_gen, orig_host = E.LookaheadEngine.generate, S.sample_lookahead

    def spy(self, *a, **k):
        calls["device"].append(k.get("sampling"))
        return orig_gen(self, *a, **k)

    def host(*a, **k):
        if not on_host:
            raise AssertionError("the host-RNG loop was entered")
        calls["host"] += 1
        return orig_host(*a, **k)
    monkeypatch.setattr(E.LookaheadEngine, "generate", spy)
    monkeypatch.setattr(S, "sample_lookahead", host)
    monkeypatch.setenv("USE_LADE", "1")
    lade.augment_all()
    try:
        lade.config_lade(LEVEL=4, WINDOW_SIZE=7, GUESS_SET_SIZE=7, DEBUG=0, POOL_FROM_PROMPT=True)
        CONFIG_MAP["SAMPLING_ON_HOST"] = 1 if on_host else 0
        outs = []
        for seed in (1, 1, 2):
            torch.manual_seed(seed)
            random.seed(seed)
            outs.append(model.generate(ids, attention_mask=torch.ones_like(ids), max_new_tokens=24, do_sample=True,
                                       **kw))
        return outs, calls
    finally:
        CONFIG_MAP.pop("SAMPLING_ON_HOST", None)
        lade.restore_generate()


def test_generate_min_p_runs_on_device(monkeypatch):
    outs, calls = _plugin_generate(monkeypatch, False, top_k=0, min_p=0.1)
    a, b, c = outs
    assert torch.equal(a, b) and a.shape == (1, 24 + 24)
    assert calls["host"] == 0 and len(calls["device"]) == 3
    assert all(abs(s["min_p"] - 0.1) < 1e-7 and s["top_k"] == 0 for s in calls["device"])


def test_generate_min_p_on_host_uses_hf_warpers(monkeypatch):
    outs, calls = _plugin_generate(monkeypatch, True, top_k=0, min_p=0.1, eta_cutoff=2e-3)
    a, b, _ = outs
    assert torch.equal(a, b) and a.shape == (1, 24 + 24)
    assert calls["host"] == 3
