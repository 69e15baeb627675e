"""The sampling accept chain (``lade_sample_verify`` / ``_warped``, bf16 and fp16) against float64 at production shapes,
through deep rejection chains, and on probability-1 / probability-0 candidates.

Launches go through the bare contexts of ``tests/sampling_ctx.py``; the test writes the guess tokens through a view
of the device state and crafts ``meta``.  The float64 side is ``tests/warper_restatement.py`` (which is
``oracle/sampling_device.py`` with the threshold warpers), fed the uniforms of the host Philox; the error bound b is
the one of ``test_sampling_chain_bound.py``.

* shapes (W, N, G) = (15, 5, 15) (the benchmark's), (60, 8, 60), (20, 33, 1024) (GS 32, G at the kernel's limit),
  (1024, 33, 1024) (a record longer than one 1024-thread pass), and G 1025, which both kernels refuse, writing nothing;
* probability 1 / 0: Philox offsets whose uniform is exactly 1.0 (seed 99 offsets 24912034, 24912035, 27778407) on
  top_k = 1, T = 0.05, min_p = 1 rows and after a rejected p = 0.5 candidate: the kernel must accept p = 1 and never
  emit a token of probability 0;
* deep chains: rows whose first k candidates (k = 8, 60, 1023, with duplicates) hold all but eps of the mass
  (eps = 1e-2 ... 1e-6), at vocabularies 32000 to 152064 with padded rows, T 0.7 / 1 and top-k, top-p, min_p, eta.
  The offsets are those whose uniforms reject the k candidates with a margin of 4 b and put the deciding uniform in a
  window around p64 (probability eps x width, found by a scan of the host stream); every decision with |u - p64| > b
  must equal float64;
* structure at G 1024, GS 32: an accept by n-gram 1023 at position 31 on rows that each give probability 1 to their own
  n-gram's next token only; the alive set pruned at the last n-gram; the EOS filter at W 60; the debug uniform count
  equal to the draws, up to 1 + G + W of them (about G + GS + W is the most a launch can draw: a rejected
  n-gram is pruned at the next accept); every record field against the restatement;
* with the cuts off, the warped kernel's record, uniforms and offset equal the plain kernel's bit for bit;
* the min_p / epsilon / eta threshold key and S' at V 128256 and 152064 (eta's entropy summed over the whole row);
* end to end: a V 151936 Qwen3 model sampled at (15, 5, 15) and (60, 8, 60), every step replayed through the
  restatement from the captured rows and the exported uniforms, and graph == eager.

The re-sum of the kept mass below 2^-12 of the last block sum is not reached here: a chain gets there only by
rejecting all but that share of the mass left at a block sum, which itself happens only where fp32 S cannot settle a
decision, and the chance of both is below 1e-8 per launch.  ``test_sampling_chain_bound.py`` exercises it."""
import ctypes as C
import math
import random

import numpy as np
import pytest
import torch

import warper_restatement as WR
from oracle import philox as PX
from oracle import sampling_device as SD
from sampling_ctx import EOS, Bare, device_logits
from test_gpu_sampling_kernel import U, bits_of
from test_sampling_chain_bound import chain_bounds, fp32_block_sum, p_old

pytestmark = pytest.mark.gpu

S_N_OLD = 4
DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}
P1_SEED, P1_OFFSETS = 99, (24912034, 24912035, 27778407)      # uniforms (0.566, 1.0), (1.0, ...), (1.0, ...)


# ---------------------------------------------------------------------------------------------- harness
_CTX = {}


def bare(W, N, G):
    if (W, N, G) not in _CTX:
        _CTX[(W, N, G)] = Bare(W, N, G)
    return _CTX[(W, N, G)]


@pytest.fixture(scope="module", autouse=True)
def _close_contexts():
    yield
    for h in _CTX.values():
        h.close()
    _CTX.clear()


class LazyRows:
    """Host float64 rows of a device logits tensor, copied on first use (the restatement reads a handful)."""

    def __init__(self, logits, vocab, base=0):
        self.t, self.vocab, self.base, self.cache = logits, vocab, base, {}

    def __getitem__(self, j):
        j = int(j) + self.base
        if j not in self.cache:
            self.cache[j] = self.t[j, :self.vocab].float().cpu().numpy().astype(np.float64)
        return self.cache[j]


def check_record(h, dtype, rec, logits, vocab, guess, T, top_k=0, top_p=1.0, cuts=None, seed=0, offset=0,
                 eos_tail=0):
    """The whole record, the exported uniforms and the offset against the restatement fed the host stream."""
    rows = LazyRows(logits, vocab)
    n_u = len(guess) + h.GS + h.W + 8
    us = PX.uniforms(seed, offset, n_u).astype(np.float64)
    mp, ep, et = cuts or (0.0, 0.0, 0.0)
    want = WR.verify_given_uniforms(rows[0], LazyRows(logits, vocab, 1 + h.WCAP) if guess else None, guess, h.GS, T,
                                    us.tolist(), top_k, top_p, mp, ep, et)
    exp = h.exported()
    assert np.array_equal(bits_of(exp), bits_of(us[:len(exp)].astype(np.float32))), "not the host stream"
    assert len(exp) == want["used"] + eos_tail, f"kernel drew {len(exp)}, restatement {want['used']} + {eos_tail}"
    assert h.rng.cpu().tolist() == [seed, offset + PX.advance(len(exp))]
    for c in want["checks"]:
        if c[0] == "accept" and c[2] not in (0.0, 1.0):
            assert abs(c[1] - c[2]) > 1e-4, "uniform too close to its threshold: pick another offset"
    n_hits = rec[1] + 1
    assert want["n_hits"] == n_hits, f"n_hits {n_hits}, restatement {want['n_hits']}"
    hits = rec[3:3 + n_hits]
    for k, t in enumerate(want["hits"] if guess else [None]):
        if t is None:
            _, u, probs = [c for c in want["checks"] if c[0] == "draw"][-1][:3]
            assert probs[hits[k]] > 0, f"residual draw emitted token {hits[k]} of probability 0"
            assert SD.draw_is_consistent(u, probs, hits[k]), "residual draw"
        else:
            assert hits[k] == t, f"position {k}: kernel {hits[k]}, restatement {t}"
    assert rec[3 + n_hits:3 + h.GS] == [0] * (h.GS - n_hits)
    assert rec[0] == hits[0] and rec[2] == h.W
    assert rec[h.R] == (want["max_hit_idx"] if n_hits > 1 else 0)
    am = h.am.cpu().tolist()
    assert rec[3 + h.GS:3 + h.GS + h.WCAP] == [am[1 + j] if j < h.W else 0 for j in range(h.WCAP)]
    assert rec[h.R + 1] == 3 and rec[h.R + 3] == 0                 # sampling, filtered row present (n_eos = 1)
    return want


def warped_equals_plain(h, dtype, logits, vocab, meta, T, top_k, top_p, seed, offset):
    a = h.launch(dtype, logits, vocab, meta, T, top_k, top_p, seed=seed, offset=offset)
    ua, ra = bits_of(h.exported()), h.rng.cpu().tolist()
    b = h.launch(dtype, logits, vocab, meta, T, top_k, top_p, cuts=(0.0, 0.0, 0.0), seed=seed, offset=offset)
    assert a == b and np.array_equal(ua, bits_of(h.exported())) and ra == h.rng.cpu().tolist(), "warped != plain"
    return a


# ---------------------------------------------------------------------------------------------- G beyond the limit
@pytest.mark.parametrize("dtype", list(DTYPES), ids=list(DTYPES))
def test_guess_set_beyond_the_kernel_limit_is_refused_and_writes_nothing(dtype):
    h = bare(20, 3, 1025)
    logits = device_logits(DTYPES[dtype], np.zeros((1, 64)), 64, 0.0)
    meta = h.set_guess([5, 6] * 1025)
    for cuts in (None, (0.0, 0.0, 0.0)):
        rec = torch.full((h.REC,), -7, dtype=torch.int32, device="cuda")
        h.rng.copy_(torch.tensor([3, 17], dtype=torch.int64))
        h.dbg.fill_(-5.0)
        sfx = "" if dtype == "bf16" else "_f16"
        if cuts is None:
            rc = getattr(h.lib, "lade_sample_verify" + sfx)(h.ctx, h.stream, logits.data_ptr(), 64, 64, h.am.data_ptr(),
                                                            meta.data_ptr(), 1.0, 0, 1.0, h.rng.data_ptr(),
                                                            rec.data_ptr(), h.dbg.data_ptr())
        else:
            w = h.C.LadeWarpers(1.0, 0, 1.0, 0.0, 0.0, 0.0)
            rc = getattr(h.lib, "lade_sample_verify_warped" + sfx)(h.ctx, h.stream, logits.data_ptr(), 64, 64,
                                                                   h.am.data_ptr(), meta.data_ptr(), C.byref(w),
                                                                   h.rng.data_ptr(), rec.data_ptr(), h.dbg.data_ptr(), 0)
        torch.cuda.synchronize()
        assert rc == h.C.LADE_EUNSUPPORTED
        assert (rec == -7).all() and h.rng.cpu().tolist() == [3, 17] and (h.dbg == -5.0).all()


# ---------------------------------------------------------------------------------------------- probability 1 / 0
def test_probe_offsets_hold_uniforms_of_exactly_one():
    assert PX.uniforms(P1_SEED, P1_OFFSETS[1], 1)[0] == 1.0
    assert PX.uniforms(P1_SEED, P1_OFFSETS[2], 1)[0] == 1.0
    u = PX.uniforms(P1_SEED, P1_OFFSETS[0], 2)
    assert 0.5 < u[0] < 0.6 and u[1] == 1.0


def _p1_cases(vocab):
    """(name, row0, guess rows {slot: row}, guess tokens (GS 4), T, top_k, cuts, offset, expected first hits)."""
    rng = np.random.default_rng(vocab)
    bg = lambda: rng.normal(0, 1.0, vocab)                       # noqa: E731
    A, B, X = vocab - 300, 1234, vocab - 7
    out = []
    r = bg(); r[A] = 6.0
    out.append(("top_k=1, one n-gram: p = 1 at u = 1", r, {}, [A, 1, 2, 3], 1.0, 1, None, P1_OFFSETS[1], [A]))
    out.append(("top_k=1, second u = 1", r, {}, [A, 1, 2, 3], 1.0, 1, None, P1_OFFSETS[2], [A]))
    r = bg() - 20.0; r[A] = r[B] = 4.0; r[X] = 3.0
    out.append(("two of 0.5, then a top-k-removed candidate", r, {}, [A, 1, 2, 3, B, 1, 2, 3, X, 1, 2, 3], 1.0, 2,
                None, P1_OFFSETS[0], [B]))
    r = bg(); r[A] = 9.0
    out.append(("T = 0.05, the other scores underflow", r, {}, [A, 1, 2, 3, X, 1, 2, 3], 0.05, 0, None,
                P1_OFFSETS[1], [A]))
    r = bg(); r[A] = 8.0
    out.append(("min_p = 1", r, {}, [A, 1, 2, 3, X, 1, 2, 3], 1.0, 0, (1.0, 0.0, 0.0), P1_OFFSETS[1], [A]))
    r = bg(); r[A] = 30.0
    g = bg(); g[B] = 9.0
    out.append(("position 1 after an accept", r, {0: g}, [A, B, 2, 3, A, X, 2, 3], 0.05, 0, None, P1_OFFSETS[0],
                [A, B]))
    return out


@pytest.mark.parametrize("dtype", list(DTYPES), ids=list(DTYPES))
@pytest.mark.parametrize("vocab", [32000, 152064])
def test_probability_one_is_accepted_and_probability_zero_never_emitted(dtype, vocab):
    h = bare(15, 5, 15)
    dt = DTYPES[dtype]
    for name, row0, grows, guess, T, top_k, cuts, off, first in _p1_cases(vocab):
        rows = np.tile(row0, (1 + h.WCAP + len(guess), 1))
        for j, r in grows.items():
            rows[1 + h.WCAP + j] = r
        logits = device_logits(dt, rows, vocab + 8, float("nan"))
        meta = h.set_guess(guess)
        rec = h.launch(dt, logits, vocab, meta, T, top_k, cuts=cuts, seed=P1_SEED, offset=off)
        assert rec[3:3 + len(first)] == first, f"{name}: emitted {rec[3:3 + len(first)]}, want {first}"
        check_record(h, dt, rec, logits, vocab, guess, T, top_k, cuts=cuts, seed=P1_SEED, offset=off)


# ---------------------------------------------------------------------------------------------- deep chains
SCAN_SEED, SCAN_WORDS = 7, 1 << 24
_STREAM = {}


def scan_stream():
    if "u" not in _STREAM:
        _STREAM["u"] = PX.uniforms(SCAN_SEED, 0, SCAN_WORDS + 1100).astype(np.float64)
    return _STREAM["u"]


def deep_row(rng, vocab, k, eps, T, n_dup):
    """k distinct candidates that hold 1 - eps of the mass, rejected in turn with conditional probabilities no higher
    than about 0.8 (so that every rejection has room for its 4 b margin): the first min(k, 8) bring what is left down
    to 10 eps (all the way to eps when k = 8), the others share the rest alike.  n_dup duplicates of the first are
    spread through the chain, the deciding candidate c holds 0.3 eps and the rest of the vocabulary 0.7 eps.
    Returns (logits = T log p, candidate order ending in c)."""
    toks = rng.choice(vocab, k + 1, replace=False)
    p = np.zeros(vocab)
    head = min(k, 8)
    q = [1 - (eps if k == head else 10 * eps) ** (1 / head)] * head + [1 - 0.1 ** (1 / max(k - head, 1))] * (k - head)
    rem = 1.0
    for j in range(k):
        p[toks[j]] = q[j] * rem
        rem -= p[toks[j]]
    p[toks[k]] = 0.3 * rem
    bg = np.ones(vocab, dtype=bool)
    bg[toks] = False
    w = rng.uniform(0.5, 1.5, bg.sum())
    p[bg] = w / w.sum() * 0.7 * rem
    order = list(toks[:k])
    for j in range(n_dup):
        order.insert(1 + (j * (k - 1)) // n_dup, toks[0])
    return T * np.log(p), order + [toks[k]]


# (vocab, k distinct rejected, eps, T, top_k, top_p, cuts, duplicates); at most 1024 n-grams in all
DEEP = [
    (32000, 8, 1e-2, 1.0, 0, 1.0, None, 0), (32000, 60, 1e-4, 0.7, 0, 1.0, None, 3),
    (32000, 1023, 1e-6, 1.0, 0, 1.0, None, 0), (128256, 8, 1e-3, 1.0, 4000, 1.0, None, 0),
    (128256, 60, 1e-5, 1.0, 0, 1.0, (1e-9, 0.0, 0.0), 0), (151936, 8, 1e-6, 0.7, 0, 1.0, None, 2),
    (151936, 60, 1e-2, 1.0, 0, 1.0, (0.0, 0.0, 1e-4), 0), (152064, 1015, 1e-4, 1.0, 0, 1.0, None, 8),
    (152064, 60, 1e-6, 1.0, 0, 1.0, None, 0), (152064, 8, 1e-5, 0.7, 0, 1.0 - 2e-6, None, 0),
]


@pytest.mark.parametrize("dtype", list(DTYPES), ids=list(DTYPES))
@pytest.mark.parametrize("case", DEEP, ids=[f"v{c[0]}-k{c[1]}-eps{c[2]:g}" for c in DEEP])
def test_deep_rejection_chain_decisions_match_float64(dtype, case):
    vocab, k, eps, T, top_k, top_p, cuts, n_dup = case
    dt = DTYPES[dtype]
    h = bare(20, 3, 1024)
    rng = np.random.default_rng(vocab + k)
    row, order = deep_row(rng, vocab, k, eps, T, n_dup)
    pad = float("nan") if k != 60 else float(torch.finfo(dt).max)
    logits = device_logits(dt, row, vocab + 8, pad)
    n_rows = 1 + h.WCAP + len(order) * h.GS
    logits = logits.expand(n_rows, -1).contiguous()                 # every guess row = row 0 (only row 0 decides)
    hrow = logits[0, :vocab].float().cpu().numpy().astype(np.float64)
    mp, ep, et = cuts or (0.0, 0.0, 0.0)
    p_row = WR.softmax_T(hrow, T, top_k, top_p, mp, ep, et)
    kept = p_row > 0
    s = (hrow.astype(np.float32) / np.float32(T)).astype(np.float64)
    x = s - s.max()
    distinct = list(dict.fromkeys(order))
    p64d, bd = chain_bounds(x, kept, np.asarray(distinct), vocab)
    first = {}
    p64, b = [], []
    for t in order:                                                  # a repeated token has probability 0
        if t in first:
            p64.append(0.0); b.append(U)
        else:
            first[t] = len(first)
            p64.append(p64d[first[t]]); b.append(bd[first[t]])
    p64, b = np.array(p64), np.array(b)
    c = order[-1]
    pc, bc = float(p64[-1]), float(b[-1])
    assert kept[c] and 0 < pc <= 1
    # the rejected candidates must clear their thresholds by 4 b; the deciding uniform lands in a window around pc
    n = len(order) - 1
    width = 1.0 if pc == 1.0 else min(0.5, 24.0 / (SCAN_WORDS * eps))    # a sole survivor: every uniform accepts
    lo, hi = max(0.0, pc - width / 2), min(1.0, pc + width / 2)
    u = scan_stream()
    idx = np.arange(SCAN_WORDS)
    for j in range(n):
        idx = idx[u[idx + j] >= p64[j] + 4 * b[j]]
    idx = idx[(u[idx + n] >= lo) & (u[idx + n] <= hi)][:24]
    assert len(idx) >= 3, f"only {len(idx)} offsets found"
    # the arithmetic the kernel had: (e_c / S) / (1 - rejected mass) in fp32
    e32 = np.where(kept, np.exp((s.astype(np.float32) - np.float32(s.max())).astype(np.float64)), 0).astype(np.float32)
    old = p_old(e32, fp32_block_sum(e32), distinct)[-1]
    guess = [t for tok in order for t in (tok, 11)]
    meta = h.set_guess(guess)
    decided = old_wrong = 0
    for o in idx.tolist():
        uc = float(u[o + n])
        rec = h.launch(dt, logits, vocab, meta, T, top_k, top_p, cuts=cuts, seed=SCAN_SEED, offset=o)
        ex = h.exported()
        assert np.array_equal(bits_of(ex[:n + 1]), bits_of(u[o:o + n + 1].astype(np.float32)))
        accepted = rec[3] == c
        if not accepted:
            assert kept[rec[3]] and rec[3] not in order, f"residual emitted {rec[3]} (kept {kept[rec[3]]})"
        if abs(uc - pc) > bc:
            assert accepted == (uc <= pc), \
                f"u={uc:.9g} p64={pc:.9g} b={bc:.3g} ({(uc - pc) / bc:+.1f} b): kernel {'accepted' if accepted else 'rejected'}"
            decided += 1
            old_wrong += (uc < old) != (uc <= pc)
    print(f"{dtype} V {vocab} k {k} eps {eps:g}: {decided} decisions, p64 {pc:.6g}, old arithmetic {old:.6g} "
          f"(rel {abs(old - pc) / pc:.1e}) would decide {old_wrong} of them wrongly")
    assert decided >= 3


# ---------------------------------------------------------------------------------------------- structure
def _peaked_rows(n_rows, vocab, peak_of, decoy, seed):
    """Device logits: every row random normal, peaked (+20) at peak_of.get(row, decoy)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    t = torch.randn(n_rows, vocab, generator=g, device="cuda")
    peaks = torch.full((n_rows,), decoy, dtype=torch.long, device="cuda")
    for r, tok in peak_of.items():
        peaks[r] = tok
    t.scatter_(1, peaks[:, None], 20.0)
    return t


def path_case(h):
    """n-gram e proposes the path token P_i at position i iff e >= thr_i (thr_0 = 0 ... thr_31 = 1023), else a token
    no row favours.  Under top_k = 1 every row gives probability 1 to one token: row 0 to P_0, the row after the
    accept of (thr_i, i) to P_(i+1), every other row to a decoy.  So position i rejects n-grams thr_(i-1) .. thr_i - 1
    and accepts thr_i, the chain ends with n-gram 1023 at position 31, and a wrong row index emits the decoy."""
    GS, G = h.GS, h.G
    thr = [round((G - 1) * i / (GS - 1)) for i in range(GS)]
    P = [100 + i for i in range(GS)]
    guess = [P[i] if e >= thr[i] else 200 + e for e in range(G) for i in range(GS)]
    peaks = {0: P[0]}
    for i in range(GS - 1):
        peaks[1 + h.WCAP + thr[i] * GS + i] = P[i + 1]
    return guess, peaks, P


def prune_case(h):
    """n-grams 0 .. G-2 agree on X at position 0 and propose tokens of probability 0 at position 1; n-gram G-1 proposes
    Y at 0 (pruned by the accept of X) and Z, the only token of the row after (0, 0), at position 1.  The chain must
    reject the G-1 live candidates and draw Z from the residual; a kernel that kept n-gram G-1 alive accepts it."""
    GS, G = h.GS, h.G
    guess = []
    for e in range(G - 1):
        guess += [100] + [300 + (e % 3000)] * (GS - 1)
    guess += [150, 120] + [121] * (GS - 2)
    return guess, {0: 100, 1 + h.WCAP: 120}


@pytest.mark.parametrize("dtype", list(DTYPES), ids=list(DTYPES))
@pytest.mark.parametrize("shape", [(20, 33, 1024), (1024, 33, 1024)])
def test_accept_by_the_last_ngram_at_the_last_position_reads_the_right_rows(dtype, shape):
    h = bare(*shape)
    dt = DTYPES[dtype]
    vocab = 4096
    guess, peaks, P = path_case(h)
    logits = _peaked_rows(h.n_rows, vocab, peaks, 7, 1).to(dt)
    meta = h.set_guess(guess)
    for seed, off in [(1, 0), (P1_SEED, P1_OFFSETS[1])]:
        rec = warped_equals_plain(h, dt, logits, vocab, meta, 1.0, 1, 1.0, seed, off)
        assert rec[1] == h.GS - 1 and rec[3:3 + h.GS] == P and rec[h.R] == h.G - 1, rec[:3 + h.GS]
        assert len(h.exported()) == (h.G - 1) + h.GS
        check_record(h, dt, rec, logits, vocab, guess, 1.0, 1, seed=seed, offset=off)


@pytest.mark.parametrize("dtype", list(DTYPES), ids=list(DTYPES))
def test_alive_set_drops_the_last_ngram(dtype):
    h = bare(20, 33, 1024)
    dt = DTYPES[dtype]
    vocab = 4096
    guess, peaks = prune_case(h)
    logits = _peaked_rows(h.n_rows, vocab, peaks, 7, 2).to(dt)
    meta = h.set_guess(guess)
    rec = warped_equals_plain(h, dt, logits, vocab, meta, 1.0, 1, 1.0, 5, 0)
    assert rec[1] == 1 and rec[3:5] == [100, 120] and rec[h.R] == 0
    assert len(h.exported()) == 1 + (h.G - 1) + 1
    check_record(h, dt, rec, logits, vocab, guess, 1.0, 1, seed=5, offset=0)


def _with_old_tokens(h, old, win):
    d = h.d
    saved = (h.st[d.off_old:d.off_old + len(old)].clone(), h.st[S_N_OLD].clone(), h.am.clone())
    h.st[d.off_old:d.off_old + len(old)] = torch.tensor(old, dtype=torch.int32)
    h.st[S_N_OLD] = len(old)
    h.am[1:1 + len(win)] = torch.tensor(win, dtype=torch.int32)
    return saved


def _restore(h, old_len, saved):
    d = h.d
    h.st[d.off_old:d.off_old + old_len], h.st[S_N_OLD] = saved[0], saved[1]
    h.am.copy_(saved[2])


def _expected_filter(win, old, tail):
    out, k = [], 0
    for v in win:
        if v == EOS:
            j = min(int(np.float32(tail[k]) * np.float32(len(old))), len(old) - 1)
            out.append(old[j]); k += 1
        else:
            out.append(v)
    return out


@pytest.mark.parametrize("dtype", list(DTYPES), ids=list(DTYPES))
def test_eos_filter_at_w60(dtype):
    h = bare(60, 8, 60)
    dt = DTYPES[dtype]
    rng = np.random.default_rng(60)
    vocab = 32000
    row = rng.normal(0, 1.0, vocab); row[77] = 3.0
    logits = device_logits(dt, np.tile(row, (h.n_rows, 1)), vocab, 0.0)
    old = list(range(500, 800))
    win = [EOS if j % 3 != 1 else 40 + j for j in range(h.W)]
    saved = _with_old_tokens(h, old, win)
    try:
        guess = [t for e in range(h.G) for t in [77 + e] + [5] * (h.GS - 1)]
        meta = h.set_guess(guess)
        for seed in (1, 2):
            rec = warped_equals_plain(h, dt, logits, vocab, meta, 1.0, 0, 1.0, seed, 9)
            us = h.exported()
            n_eos = win.count(EOS)
            assert rec[h.R + 4:h.R + 4 + h.W] == _expected_filter(win, old, us[len(us) - n_eos:])
            check_record(h, dt, rec, logits, vocab, guess, 1.0, seed=seed, offset=9, eos_tail=n_eos)
    finally:
        _restore(h, len(old), saved)


@pytest.mark.parametrize("dtype", list(DTYPES), ids=list(DTYPES))
def test_most_draws_of_one_launch_are_exported(dtype):
    """(1024, 33, 1024): all 1024 n-grams rejected at position 0 (each proposes a token of probability 0 but the
    first), the residual draw, and 1024 EOS columns: 2049 uniforms, in a buffer of 2 + G GS + W."""
    h = bare(1024, 33, 1024)
    dt = DTYPES[dtype]
    vocab = 4096
    old = list(range(900, 1400))
    win = [EOS] * h.W
    saved = _with_old_tokens(h, old, win)
    try:
        logits = _peaked_rows(h.n_rows, vocab, {0: 9}, 7, 3).to(dt)
        guess = [t for e in range(h.G) for t in [2000 + e] + [5] * (h.GS - 1)]
        meta = h.set_guess(guess)
        rec = warped_equals_plain(h, dt, logits, vocab, meta, 1.0, 1, 1.0, 11, 0)
        us = h.exported()
        assert len(us) == h.G + 1 + h.W and rec[3] == 9
        assert rec[h.R + 4:h.R + 4 + h.W] == _expected_filter(win, old, us[len(us) - h.W:])
        check_record(h, dt, rec, logits, vocab, guess, 1.0, 1, seed=11, offset=0, eos_tail=h.W)
    finally:
        _restore(h, len(old), saved)


@pytest.mark.parametrize("dtype", list(DTYPES), ids=list(DTYPES))
@pytest.mark.parametrize("shape", [(15, 5, 15), (60, 8, 60)])
def test_chains_at_benchmark_shapes_match_the_restatement(dtype, shape):
    """Random peaked rows with shared-prefix n-grams at T 0.7: 40 offsets, each record against the restatement."""
    h = bare(*shape)
    dt = DTYPES[dtype]
    vocab = 32000
    rng = np.random.default_rng(shape[0])
    base = [int(t) for t in rng.choice(vocab, 6, replace=False)]
    guess = []
    for e in range(h.G):
        g = [base[e % 3]] + [base[3 + (e + i) % 3] if (e + i) % 4 else int(rng.integers(vocab)) for i in range(h.GS - 1)]
        guess += g
    rows = rng.normal(0, 1.0, (h.n_rows, vocab))
    rows[0, base[:3]] += [11.5, 11.2, 10.9]
    rows[1 + h.WCAP:, base[3]] += 11.5
    rows[1 + h.WCAP:, base[4]] += 11.0
    logits = device_logits(dt, rows, vocab + 8, float("nan"))
    meta = h.set_guess(guess)
    lens, checked = set(), 0
    for off in range(0, 4 * 40, 4):
        rec = warped_equals_plain(h, dt, logits, vocab, meta, 0.7, 0, 1.0, 3, off)
        try:
            check_record(h, dt, rec, logits, vocab, guess, 0.7, seed=3, offset=off)
        except AssertionError as e:
            if "too close" in str(e):
                continue
            raise
        lens.add(rec[1])
        checked += 1
    print(f"{shape} {dtype}: {checked} records checked, max_hit in {sorted(lens)}")
    assert checked >= 20


# ---------------------------------------------------------------------------------------------- warpers, large V
def _warper_rows(vocab, T, seed):
    """Rows of a real vocabulary's size: randn * 1.5 logits, a few peaked tokens past id 2^17."""
    rng = np.random.default_rng(seed)
    r = rng.normal(0, 1.5, vocab) * T
    r[[vocab - 11, vocab // 2, 3]] = np.array([6.0, 5.5, 5.0]) * T
    return r


WARPER_CUTS = [dict(min_p=0.05), dict(min_p=0.002), dict(epsilon=3e-6), dict(epsilon=1e-5), dict(eta=1e-4),
               dict(eta=3e-3), dict(min_p=0.001, epsilon=2e-6, eta=5e-4)]
WARPER_SETTINGS = [(1.0, 0, 1.0), (0.7, 2000, 1.0), (1.0, 0, 0.9), (1.3, 0, 1.0), (0.8, 0, 1.0)]


@pytest.mark.parametrize("dtype", list(DTYPES), ids=list(DTYPES))
@pytest.mark.parametrize("vocab", [128256, 152064])
def test_warper_cuts_at_large_vocabularies(dtype, vocab):
    """The threshold key and S' of every cut on rows of 128256 / 152064 tokens, where eta's entropy is an fp32 sum
    over the whole vocabulary: the kept set equals float64's wherever every token's keep decision clears the fp32
    bound by 1.5 times (cut_margin_ok), S' is within 1.5 of its bound, and the plain draw is the float64 one."""
    from test_gpu_sampling_warpers import cut_margin_ok, keys_of
    from test_gpu_sampling_kernel import exp_rel
    dt = DTYPES[dtype]
    h = bare(15, 5, 15)
    wdbg = torch.zeros(1 + 2 * h.GS, dtype=torch.float32, device="cuda")
    meta = h.meta(0)
    checked = etas = 0
    for i, cut in enumerate(WARPER_CUTS):
        for T, top_k, top_p in WARPER_SETTINGS:
            logits = device_logits(dt, _warper_rows(vocab, T, 100 * i + int(T * 10) + top_k), vocab + 8, float("nan"))
            hrow = logits[0, :vocab].float().cpu().numpy().astype(np.float64)
            if not cut_margin_ok(hrow, T, top_k, top_p, cut, vocab):
                continue
            probs = WR.softmax_T(hrow, T, top_k, top_p, **cut)
            before = WR.softmax_T(hrow, T, top_k, top_p)
            kept64 = probs > 0
            if kept64.sum() == (before > 0).sum():
                continue                                 # top-k / top-p already keep less than the cut would
            args = (cut.get("min_p", 0.0), cut.get("epsilon", 0.0), cut.get("eta", 0.0))
            rec = h.launch(dt, logits, vocab, meta, T, top_k, top_p, cuts=args, seed=5, offset=4 * i, dbg_cuts=wdbg)
            c = wdbg.cpu().numpy()
            assert int(c[0]) == 1
            thr, S1 = int(c[1]), float(c[2])
            keys = keys_of(None, logits, vocab)
            assert (keys >= thr).tolist() == kept64.tolist(), \
                f"{cut} T={T} k={top_k} p={top_p}: kernel kept {(keys >= thr).sum()}, float64 {kept64.sum()}"
            assert thr == keys[kept64].min()
            s = (hrow.astype(np.float32) / np.float32(T)).astype(np.float64)
            x = s - s.max()
            S64 = np.exp(x)[kept64].sum()
            s_err = float((probs[kept64] * exp_rel(x[kept64])).sum()) + (math.ceil(vocab / 1024) + 10) * U
            assert abs(S1 - S64) <= 1.5 * s_err * S64 + U * S64, f"{cut} T={T}: S' {S1} vs {S64} (bound {s_err:.2g})"
            u = float(PX.uniforms(5, 4 * i, 1)[0])
            assert SD.draw_is_consistent(u, probs, rec[3]), f"{cut} T={T}: draw {rec[3]}"
            checked += 1
            etas += "eta" in cut
    print(f"{dtype} V {vocab}: {checked} warped rows checked, {etas} with eta")
    assert checked >= 10 and etas >= 2


# ---------------------------------------------------------------------------------------------- end to end
@pytest.mark.parametrize("shape", [(15, 5, 15), (60, 8, 60)])
def test_qwen3_vocabulary_sampling_steps_replay_and_graph_equals_eager(shape):
    """A V 151936 Qwen3 model sampled by the engine (T 0.1 with top-k 50 / top-p 0.9: a random model then repeats
    itself enough for the pool to propose candidates), one eager step at a time with the logits captured: every
    step's hits replay through the float64 restatement from the captured rows and the exported uniforms.  Then
    generate() with the CUDA graph and eagerly emit the same tokens."""
    from test_gpu_capture_logits import _engine, lockstep
    from test_gpu_qwen3 import _prompt, build_qwen3
    W, N, G = shape
    model = build_qwen3()
    prompt, new = _prompt(32), 40
    s = dict(temperature=0.1, top_k=50) if W == 15 else dict(temperature=0.1, top_p=0.9)
    T, top_k, top_p = s["temperature"], s.get("top_k", 0), s.get("top_p", 1.0)
    eng = _engine(model, len(prompt) + new, W=W, N=N, G=G, use_cuda_graph=False)
    steps = lockstep(eng, prompt, new, sampling=s)
    GS, WCAP, V = eng.GS, eng.WCAP, eng.V
    assert V == 151936
    nan_row = np.full(V, np.nan)
    checked = tested = 0
    for k, st in enumerate(steps):
        rows = st["rows"].float().cpu().numpy().astype(np.float64)
        guess = st["guess"] if st["phase"] == 2 and st["guess"] else None
        captured = {slot - 1 - WCAP: rows[j] for j, slot in enumerate(st["slots"][1:], start=1)}
        guess_rows = type("Rows", (), {"__getitem__": lambda self, j: captured.get(int(j), nan_row)})()
        with np.errstate(invalid="ignore"):
            want = SD.verify_given_uniforms(rows[0], guess_rows if guess else None, guess, GS, T, st["uniforms"],
                                            top_k, top_p)
        if any(c[0] == "accept" and 0 < c[2] < 1 and abs(c[1] - c[2]) < 1e-6 for c in want["checks"]):
            continue
        assert want["used"] == len(st["uniforms"]) and want["n_hits"] == len(st["hits"]), f"step {k}"
        draws = [c for c in want["checks"] if c[0] == "draw"]
        for j, hit in enumerate(want["hits"] or [None]):
            if hit is None:
                _, u, probs = draws[-1][:3]
                assert SD.draw_is_consistent(u, probs, st["hits"][j]), f"step {k} draw"
            else:
                assert st["hits"][j] == hit, f"step {k} token {j}"
        checked += 1
        tested += sum(c[0] == "accept" for c in want["checks"])
    eng.close()
    print(f"{shape}: {checked} of {len(steps)} steps replayed, {tested} candidates tested")
    assert checked >= len(steps) - 2 and tested >= 5
    outs = []
    for graph in (True, False):
        eng = _engine(model, len(prompt) + new, W=W, N=N, G=G, use_cuda_graph=graph)
        outs.append(eng.generate(prompt, new, rng=random.Random(0), sampling=dict(s, seed=7)))
        eng.close()
    assert outs[0] == outs[1] and len(outs[0]) == len(prompt) + new
