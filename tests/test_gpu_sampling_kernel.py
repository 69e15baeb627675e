"""``lade_sample_verify`` / ``lade_sample_verify_f16`` launched directly, on crafted logits, against float64.

The engine only ever hands the kernel a tiny model's own logits.  Here a tiny-model engine is brought to a phase-2
step once (the loop of ``test_gpu_sampling_device.py``); its ctx then serves any number of direct launches on rows
the test controls.  The kernel reads from the ctx state only the guess tokens (``off_guess``), ``S_DONE``,
``S_N_OLD`` and the old tokens (``off_old``); the test writes those through a view of the device state.  Every
uniform the kernel draws is known before the launch from the host Philox (``oracle/philox.py``).  The float64 side
is ``oracle/sampling_device.py``.

* stream: exported uniforms == host Philox bit for bit, the offset advance, no word used twice over 200 launches,
  and the engine's steps continue one stream;
* accept-threshold probes: uniforms 1.25 to 4 error bounds b below (must accept) or above (must reject) the float64
  accept probability, after 0 to 4 rejections, for T in {0.05, 1, 4} with and without top-k / top-p;
* kept set and inverse CDF of plain draws on rows built around the top-k / top-p cut-offs;
* the accept chain against the restatement; the distribution of the emitted (hits, max_hit_idx) against an exact
  enumeration (G-test); the EOS filter, a finished state, and run-to-run determinism.

Every test runs for bf16 and fp16."""
import ctypes as C
import math
import random

import numpy as np
import pytest
import torch

from oracle import philox as PX
from oracle import sampling_device as SD

pytestmark = pytest.mark.gpu

W, N, G = 7, 4, 7
GS, WCAP = N - 1, W + N - 3
R = 3 + GS + WCAP                       # lp_rec_ints: [first, max_hit, n_new, hits[GS], new_tok[WCAP]]
REC = R + 4 + W                         # + [max_hit_idx, flags, extra_finished, 0, filtered[W]]
EOS = 4097                              # outside the tiny model's vocabulary: never generated, only crafted
S_N_OLD, S_DONE = 4, 5
U = 2.0 ** -24
DTYPES = [torch.bfloat16, torch.float16]


# ---------------------------------------------------------------------------------------------- harness
class _Dims(C.Structure):                  # lade::Dims (csrc/state.cuh)
    _fields_ = [(n, C.c_int32) for n in "W N G GS WCAP V cap pool_from_prompt n_eos D rank".split()] + \
               [("eos", C.c_int32 * 4), ("lm_cap", C.c_int32)] + \
               [(n, C.c_int32) for n in "off_win off_win_len off_guess off_out off_old off_cnt".split()] + \
               [("off_tup", C.c_int64), ("total_ints", C.c_int64)]


class _DevInts:
    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = dict(shape=(n,), typestr="<i4", data=(ptr, False), version=3)


class Harness:
    def __init__(self, dtype):
        from lookaheaddecoding_b200 import LookaheadEngine, _cabi
        from test_gpu_sampling_device import _prompt, peaked_periodic_model
        self.C = _cabi
        self.dtype = dtype
        model = peaked_periodic_model()
        if dtype != torch.bfloat16:
            model = model.to(dtype)
        prompt = _prompt(24)
        eng = LookaheadEngine(model, W, N, G, pool_from_prompt=True, max_total_len=24 + 96, use_cuda_graph=False)
        eng.sample_temperature, eng.sample_top_k, eng.sample_top_p = 0.8, 0, 1.0
        eng.begin(prompt, 24 + 96, (EOS,), eng.draw_window(prompt, random.Random(3)))
        eng.rng_state.copy_(torch.tensor([1234, 0], dtype=torch.int64))
        for step in range(96):                  # to the first verification step (the kernel reads phase, tiny and
            eng.run_forward_step(step, 24, commit="sample")     # the guess count from meta: set_guess edits them)
            torch.cuda.synchronize()
            meta = eng.meta.cpu()
            assert not eng.res[_cabi.R_DONE]
            if meta[_cabi.M_PHASE] == 2:
                break
        self.eng, self.meta2 = eng, meta
        fields = [("cfg", _cabi.LadeConfig), ("d", _Dims), ("state", C.c_void_p)]
        ctx = type("_Ctx", (C.Structure,), {"_fields_": fields}).from_address(eng._ctx.value)
        d = ctx.d
        assert (d.W, d.N, d.G, d.GS, d.WCAP, d.n_eos, d.eos[0]) == (W, N, G, GS, WCAP, 1, EOS), "ctx layout"
        self.d = d
        self.st = torch.as_tensor(_DevInts(ctx.state, int(d.total_ints)), device="cuda")
        self.fn = eng.k_sample_verify
        self.rng = torch.zeros(2, dtype=torch.int64, device="cuda")
        self.dbg = torch.zeros(64, dtype=torch.float32, device="cuda")
        self.am = torch.zeros(eng.lm_cap, dtype=torch.int32, device="cuda")

    def set_guess(self, tokens):
        """n-gram e proposes tokens[e*GS:(e+1)*GS]; returns the meta of a phase-2 step with those n-grams."""
        self.st[self.d.off_guess:self.d.off_guess + len(tokens)] = torch.tensor(tokens, dtype=torch.int32)
        m = self.meta2.clone()
        m[self.C.M_PHASE] = 2
        m[self.C.M_N_GUESS_TOK] = len(tokens)
        return m.cuda()

    def plain_meta(self):
        m = self.meta2.clone()
        m[self.C.M_PHASE] = 1
        m[self.C.M_N_GUESS_TOK] = 0
        return m.cuda()

    def launch(self, logits, vocab, meta, T, top_k=0, top_p=1.0, rec=None, dbg=True):
        rec = torch.full((REC,), -7, dtype=torch.int32, device="cuda") if rec is None else rec
        stream = torch.cuda.current_stream().cuda_stream
        self.C.check(self.fn(self.eng._ctx, stream, logits.data_ptr(), logits.shape[1], vocab, self.am.data_ptr(),
                             meta.data_ptr(), float(T), int(top_k), float(top_p), self.rng.data_ptr(), rec.data_ptr(),
                             self.dbg.data_ptr() if dbg else 0), "lade_sample_verify")
        return rec

    def seed(self, seed, offset):
        self.rng.copy_(torch.tensor([seed, offset], dtype=torch.int64))

    def exported(self):
        d = self.dbg.cpu().numpy()
        return d[1:1 + int(d[0])]


@pytest.fixture(scope="module", params=DTYPES, ids=["bf16", "fp16"])
def H(request):
    h = Harness(request.param)
    yield h
    h.eng.close()


def logits_tensor(h, rows, ld=None, pad=None):
    """(n_rows, ld) device logits of the harness dtype from float rows of length vocab; the padding columns hold
    `pad` (default: the dtype's largest finite value), which the kernel must never read."""
    rows = np.atleast_2d(np.asarray(rows, dtype=np.float64))
    vocab = rows.shape[1]
    ld = ld or vocab
    full = np.full((rows.shape[0], ld), torch.finfo(h.dtype).max if pad is None else pad, dtype=np.float64)
    full[:, :vocab] = rows
    return torch.tensor(full, dtype=torch.float32).to(h.dtype).cuda()


def host_rows(t, vocab):
    return t[:, :vocab].float().cpu().numpy().astype(np.float64)


def step_rows(h, row0, guess_rows=None, ld=None, pad=None):
    """Logits of a phase-2 step: slot 0 = row0, slots 1+WCAP+e*GS+i = guess_rows[e*GS+i] (default: row0)."""
    n = 1 + WCAP + G * GS
    rows = np.tile(np.asarray(row0, dtype=np.float64), (n, 1))
    if guess_rows is not None:
        for j, r in guess_rows.items():
            rows[1 + WCAP + j] = r
    return logits_tensor(h, rows, ld, pad)


def bits_of(x):
    return np.asarray(x, dtype=np.float32).view(np.uint32)


# ---------------------------------------------------------------------------------------------- stream
@pytest.mark.parametrize("seed", [0, 77, 2 ** 63 - 1])
@pytest.mark.parametrize("offset", [0, 6, 2 ** 40 + 3])
def test_stream_is_the_host_philox_and_never_reused(H, seed, offset):
    rng = np.random.default_rng(seed % 1000)
    vocab = 4096
    row0 = rng.normal(0, 1.0, vocab)
    toks = [11, 12, 13, 21, 22, 23, 31, 32, 33]
    row0[[11, 21, 31]] += 7.5                         # intermediate accept probabilities: the draw count varies
    guess = {}
    for j in range(len(toks)):
        guess[j] = rng.normal(0, 1.0, vocab)
        if (j + 1) % GS:
            guess[j][toks[j + 1]] += 7.5
    lg = step_rows(H, row0, guess)
    meta = H.set_guess(toks)
    H.seed(seed, offset)
    used, off, counts = [], offset, set()
    for it in range(200):
        H.launch(lg, vocab, meta, 1.0)
        u = H.exported()
        n = len(u)
        counts.add(n)
        assert n >= 1
        assert np.array_equal(bits_of(u), bits_of(PX.uniforms(seed, off, n))), f"launch {it}: not the host stream"
        off += PX.advance(n)
        got = H.rng.cpu().tolist()
        assert got[0] == seed and got[1] == off, f"launch {it}: rng_state {got}, want offset {off}"
        used.append((off - PX.advance(n), off - PX.advance(n) + n))
    words = [w for a, b in used for w in range(a, b)]
    assert len(words) == len(set(words))
    assert len(counts) >= 2, "the draw count never varied"


def test_engine_steps_continue_one_stream(H):
    eng = H.eng
    saved = H.st.clone()
    eng.debug_uniforms = torch.zeros(4 + G * GS + W, dtype=torch.float32, device="cuda")
    from test_gpu_sampling_device import _prompt
    prompt = _prompt(24)
    eng.begin(prompt, 24 + 64, (EOS,), eng.draw_window(prompt, random.Random(3)))
    seed = 2 ** 63 - 1
    eng.rng_state.copy_(torch.tensor([seed, 5], dtype=torch.int64))
    off, n_steps = 5, 0
    for step in range(40):
        eng.run_forward_step(step, 24, commit="sample")
        torch.cuda.synchronize()
        if eng.res[H.C.R_DONE]:
            break
        dbg = eng.debug_uniforms.cpu().numpy()
        u = dbg[1:1 + int(dbg[0])]
        if len(u):
            assert np.array_equal(bits_of(u), bits_of(PX.uniforms(seed, off, len(u)))), f"step {step}"
            n_steps += 1
        off += PX.advance(len(u))
        assert eng.rng_state.cpu().tolist() == [seed, off]
    eng.debug_uniforms = None
    H.st.copy_(saved)
    assert n_steps >= 10


# ---------------------------------------------------------------------------------------------- error bound
def exp_rel(x):
    """Relative error of the kernel's __expf(s - mx) at x = s - mx (float64 of the fp32 difference).  The CUDA C++
    Programming Guide documents __expf's error as 2 + floor(|c x|) ulp with c just under 1.2; one ulp of a result in
    (0, 1] is at most 2u of it (u = 2^-24).  The fp32 subtraction s - mx rounds once more: |x| u."""
    x = np.abs(np.asarray(x, dtype=np.float64))
    return (2.0 + np.floor(1.2 * x)) * 2 * U + x * U


def accept_bound(row, T, top_k, top_p, vocab, cands, k):
    """(p64, b): the float64 probability that the kernel accepts cands[k] after rejecting cands[:k] at position 0, and
    a bound b on |p_kernel - p64|.

    p_kernel = e_c / S / (1 - zmass) in fp32 where
    * e_c = __expf(x_c): relative error exp_rel(x_c);
    * S sums every kept e_t: each term carries exp_rel(x_t) (so the mass-weighted mean of it), the fp32 sum adds
      ceil(vocab / 1024) sequential adds per thread and 10 shuffle levels, each at most u of the running sum; the
      top-p kept mass is instead an exact integer sum of e_t rounded to 2^-40, vocab 2^-41 / S at most;
    * two divisions, u each;
    * zmass accumulates the rejected p_raw_j, each with the error above plus one add: the error of 1 - zmass is that
      absolute error, relative to 1 - zmass (>= 0.1 in every probe: at most 9x amplification);
    plus u absolute for the comparison with an fp32 uniform."""
    p_row = SD.softmax_T(row, T, top_k, top_p)
    s = (row.astype(np.float32) / np.float32(T)).astype(np.float64)
    x = s - s.max()
    kept = p_row > 0
    e_err = float((p_row[kept] * exp_rel(x[kept])).sum())
    s_err = e_err + (math.ceil(vocab / 1024) + 10) * U + (vocab * 2.0 ** -41 if top_p < 1.0 else 0.0)
    raw = lambda t: p_row[t]
    z = sum(raw(c) for c in cands[:k])
    z_abs = sum(raw(c) * (exp_rel(x[c]) + s_err + 2 * U) for c in cands[:k])
    p = raw(cands[k]) / (1.0 - z)
    rel = exp_rel(x[cands[k]]) + s_err + 2 * U + z_abs / (1.0 - z)
    return p, min(1.0, p) * rel + U, [raw(c) / (1.0 - sum(raw(c2) for c2 in cands[:j])) for j, c in enumerate(cands[:k])]


def find_probes(seed, k, rejects, lo, hi, n_want, start=0, max_words=1 << 27):
    """Offsets o (multiples of 1) such that the uniforms u_0..u_{k-1} at o reject (u_j >= p_j with a margin) and
    u_k at o lies in [lo, hi]."""
    found, chunk, o = [], 1 << 22, start
    while len(found) < n_want and o - start < max_words:
        u = PX.uniforms(seed, o, chunk + k)
        ok = (u[k:k + chunk] >= lo) & (u[k:k + chunk] <= hi)
        for j, pj in enumerate(rejects):
            ok &= u[j:j + chunk] >= pj * (1 + 1e-4) + 1e-6
        found += (o + np.nonzero(ok)[0]).tolist()[: n_want - len(found)]
        o += chunk
    return found


def probe_row(rng, vocab, T, p, k, spread=64):
    """A row where position-0 candidates 0..k-1 carry 0.15 each and candidate k carries p of what remains."""
    target = np.zeros(vocab)
    cands = list(range(100, 100 + 10 * (k + 1), 10))
    q = 0.15
    rest = 1.0 - q * k
    target[cands[:k]] = q
    target[cands[k]] = p * rest
    bg = np.setdiff1d(np.arange(200, 200 + 4 * spread, 4), cands)[:spread]
    w = np.exp(-np.linspace(0, 6, spread))
    target[bg] = max(rest * (1 - p), 1e-300) * w / w.sum()
    with np.errstate(divide="ignore"):
        lg = T * np.log(target)
    lg = np.where(np.isfinite(lg), lg, -40.0 * max(T, 1.0))       # exp(-40) and below: no mass
    lg -= lg.max() - 2.0
    return lg, cands


PROBE_TARGETS = [(1e-3, 0), (0.05, 1), (0.3, 3), (0.5, 4), (0.9, 2), (1 - 1e-6, 0)]


@pytest.mark.parametrize("T,warp", [(0.05, "none"), (1.0, "none"), (4.0, "none"), (1.0, "top_k"), (0.05, "top_k"),
                                    (4.0, "top_p")])
def test_accept_probability_matches_float64(H, T, warp):
    rng = np.random.default_rng(int(T * 100))
    vocab, seed = 32000, 99
    checked = 0
    for p_t, k in PROBE_TARGETS:
        lg, cands = probe_row(rng, vocab, T, p_t, k)
        top_k = top_p = None
        logits = step_rows(H, lg, ld=vocab + 8)
        row = host_rows(logits, vocab)[0]
        p_row = SD.softmax_T(row, T)
        top_k, top_p = 0, 1.0
        if warp == "top_k":
            top_k = int((p_row >= 0.5 * min(p_row[c] for c in cands)).sum()) + 3
        elif warp == "top_p":
            if p_t > 0.99 or p_t < 0.01:
                continue
            top_p = 1.0 - 0.3 * float(np.sort(p_row)[:-(2 + k + 8)].sum())      # cuts into the background
        p64, b, rejects = accept_bound(row, T, top_k, top_p, vocab, cands, k)
        if not 0 < p64:
            pytest.fail(f"probe row lost its candidate (T={T} {warp} p={p_t})")
        meta = H.set_guess([t for c in cands for t in (c, 5, 6)])
        sides = [("accept", p64 - 4 * b, p64 - 1.25 * b)]
        if p64 + 1.25 * b < 1.0:
            sides.append(("reject", p64 + 1.25 * b, min(1.0, p64 + 4 * b)))
        for kind, lo, hi in sides:
            offs = find_probes(seed, k, rejects, lo, hi, 3)
            assert offs, f"no probe found for p64={p64} ({kind})"
            for o in offs:
                H.seed(seed, int(o))
                rec = H.launch(logits, vocab, meta, T, top_k, top_p).cpu().tolist()
                u = H.exported()
                assert abs(float(u[k]) - (lo + hi) / 2) <= (hi - lo) / 2 + 1e-12
                accepted = rec[3] == cands[k]
                assert accepted == (kind == "accept"), \
                    f"T={T} {warp} k={k}: p64={p64:.9g} b={b:.3g} u={float(u[k]):.9g} ({(u[k] - p64) / b:+.2f} b) -> " \
                    f"{'accepted' if accepted else 'rejected'}"
                checked += 1
    assert checked >= 16


def test_accept_bound_is_tight_enough():
    """b stays far below the top-p kept-mass cancellation error it must expose (1e-5 relative and more)."""
    rng = np.random.default_rng(1)
    lg, cands = probe_row(rng, 32000, 1.0, 0.5, 2)
    p64, b, _ = accept_bound(lg.astype(np.float32).astype(np.float64), 1.0, 0, 1.0, 32000, cands, 2)
    assert b < 1e-5 * p64


@pytest.mark.parametrize("sigma,top_p", [(0.5, 0.1), (0.1, 0.05), (0.02, 0.01)])
def test_top_p_accept_probability_at_llama_vocab(H, sigma, top_p):
    """The table rows of randn * sigma logits at vocab 32000: candidates hold about half of the kept mass."""
    rng = np.random.default_rng(int(sigma * 1000))
    vocab, seed, T = 32000, 5, 1.0
    bg = rng.normal(0, sigma, vocab)
    tot = np.exp(bg).sum()
    checked = 0
    for p_t, k in [(0.4, 0), (0.5, 1), (0.6, 2)]:
        row = bg.copy()
        cands = [1000 + 7 * j for j in range(k + 1)]
        kept = top_p * tot
        for c in cands[:k]:
            row[c] = math.log(0.1 * kept)
        row[cands[k]] = math.log(p_t * (1 - 0.1 * k) * kept)
        logits = step_rows(H, row, ld=vocab + 3)
        row = host_rows(logits, vocab)[0]
        p64, b, rejects = accept_bound(row, T, 0, top_p, vocab, cands, k)
        assert 0.05 < p64 < 0.99
        meta = H.set_guess([t for c in cands for t in (c, 5, 6)])
        for kind, lo, hi in [("accept", p64 - 4 * b, p64 - 1.25 * b), ("reject", p64 + 1.25 * b, p64 + 4 * b)]:
            for o in find_probes(seed, k, rejects, lo, hi, 3):
                H.seed(seed, int(o))
                rec = H.launch(logits, vocab, meta, T, 0, top_p).cpu().tolist()
                accepted = rec[3] == cands[k]
                u = float(H.exported()[k])
                assert accepted == (kind == "accept"), \
                    f"sigma={sigma} top_p={top_p} k={k}: p64={p64:.9g} b={b:.3g} u={u:.9g} ({(u - p64) / b:+.2f} b)"
                checked += 1
    assert checked >= 12


# ---------------------------------------------------------------------------------------------- kept set and CDF
def _bf(h, v):
    return torch.tensor([v], dtype=torch.float32).to(h.dtype).float().item()


def _next_below(h, v):
    t = torch.tensor([v], dtype=torch.float32).to(h.dtype)
    b = t.view(torch.int16).item()
    b = -32767 if v == 0 else (b - 1 if v > 0 else b + 1)        # below +-0: the smallest negative subnormal
    return torch.tensor([b], dtype=torch.int16).view(h.dtype).float().item()


def kept_set_cases(h):
    """(name, row, vocab, T, top_k, top_p)."""
    rng = np.random.default_rng(7)
    V = 32000
    low = lambda n: rng.uniform(-30, -20, n)               # no mass to speak of, never in a kept set
    cases = []
    r = low(V); r[10:15] = 2.0; r[[20, 40, 60, 80, 100, 120]] = 1.5; r[200:260] = 1.0
    cases.append(("tie group straddles the k-th", r, V, 1.0, 8, 1.0))
    for name, bits in [("k-th at low byte 0x00", 0x3F00), ("k-th at low byte 0xff", 0x3FFF if h.dtype == torch.bfloat16 else 0x3BFF)]:
        kth = torch.tensor([bits], dtype=torch.int16).view(h.dtype).float().item()
        r = low(V); r[[3, 9, 17]] = kth + 0.25 * abs(kth); r[[5, 33]] = kth; r[[7, 8, 900]] = _next_below(h, kth)
        cases.append((name, r, V, 1.0, 5, 1.0))
    r = low(V); r[[1, 2]] = -0.5; r[[50, 51]] = -1.0; r[[60, 61, 62]] = _next_below(h, -1.0)
    cases.append(("negative k-th", r, V, 1.0, 4, 1.0))
    r = low(V); r[[1, 2, 3]] = 0.5; r[40] = 0.0; r[41] = -0.0; r[[42, 43]] = _next_below(h, 0.0)
    cases.append(("+0 and -0 at the top-k cut", r, V, 1.0, 4, 1.0))
    r = low(V); r[[1, 2, 3]] = 3.0; r[40] = 0.0; r[41] = -0.0; r[[42, 43]] = _next_below(h, 0.0)
    p = np.exp(np.array([3.0] * 3 + [0.0] * 2 + [r[42]] * 2))
    cases.append(("+0 and -0 at the top-p cut", r, V, 1.0, 0, float(1 - 3.5 / p.sum())))
    cases.append(("all values equal", np.full(4096, 0.75), 4096, 1.0, 5, 0.3))
    base = rng.normal(0, 1.0, 4096); base[:8] += 4.0
    for k in (1, 2, 4095, 4096, 4101):
        cases.append((f"top_k={k}", base, 4096, 1.0, k, 1.0))
    peaked = rng.normal(0, 0.5, 32000); peaked[[3, 500, 20000]] = [6.0, 5.5, 5.0]
    cases.append(("top_p=1e-6", peaked, 32000, 1.0, 0, 1e-6))
    cases.append(("top_p=1-2^-20", rng.normal(0, 2.0, 32000), 32000, 1.0, 0, 1 - 2.0 ** -20))
    r = rng.normal(0, 1.0, 4096); r[:4] += 3.0; r[100:4096:2] = -100.0
    cases.append(("exp underflows", r, 4096, 1.0, 0, 1.0))
    r = rng.normal(0, 1.0, 4096); r[:4] += 3.0; r[100:4096:2] = -100.0
    cases.append(("exp underflows, top-k 60", r, 4096, 0.5, 60, 1.0))
    return cases


def _draw_many(h, logits, vocab, T, top_k, top_p, seed, offset, n):
    """n chained plain draws (rng_state advances by 4 each); returns the drawn tokens and their uniforms."""
    meta = h.plain_meta()
    recs = torch.zeros(n, REC, dtype=torch.int32, device="cuda")
    h.seed(seed, offset)
    for j in range(n):
        h.launch(logits, vocab, meta, T, top_k, top_p, rec=recs[j], dbg=False)
    assert h.rng.cpu().tolist() == [seed, offset + 4 * n]
    u = PX.uniforms(seed, offset + 4 * np.arange(n, dtype=np.uint64), 1)[:, 0]
    return recs[:, 3].cpu().numpy(), u


def _check_draws(probs, toks, u, what, rel_eps=2e-5):
    c = np.cumsum(probs)
    lo = np.where(toks > 0, c[np.maximum(toks - 1, 0)], 0.0)
    hi = c[toks]
    tgt = u.astype(np.float64) * c[-1]
    ok = (probs[toks] > 0) & (lo - rel_eps * c[-1] <= tgt) & (tgt <= hi + rel_eps * c[-1])
    bad = np.nonzero(~ok)[0]
    assert not len(bad), f"{what}: draw {bad[0]} u={u[bad[0]]:.9g} -> token {toks[bad[0]]} (p={probs[toks[bad[0]]]:.3g})"


def test_kept_set_and_inverse_cdf_of_plain_draws(H):
    for i, (name, row, vocab, T, top_k, top_p) in enumerate(kept_set_cases(H)):
        pad = float("nan") if i == 0 else None
        logits = logits_tensor(H, row, ld=vocab + 37, pad=pad)
        hrow = host_rows(logits, vocab)[0]
        probs = SD.softmax_T(hrow, T, top_k, top_p)
        toks, u = _draw_many(H, logits, vocab, T, top_k, top_p, 11 + i, 3 + 8 * i, 4096)
        _check_draws(probs, toks, u, name)
        big = np.nonzero(probs >= 0.02)[0]
        missing = set(big.tolist()) - set(toks.tolist())
        assert not missing, f"{name}: tokens {sorted(missing)[:5]} of the kept set never drawn"


@pytest.mark.parametrize("low", [0.5, 0.25])
def test_top_p_cut_exactly_at_a_bucket_boundary(H, low):
    """T = 1e38 makes both scores subnormal: in fp32 and in float64 both tokens then carry mass exactly 1, so with
    top_p = 0.5 the ascending cumulative mass of the lower one equals 1 - top_p exactly and TopPLogitsWarper's
    `cum <= 1 - top_p` drops it.  The lower token sits first in index order, where a kept one would be drawn for u <= 1/2."""
    row = np.array([low, 1.0])
    logits = logits_tensor(H, row, ld=9)
    probs = SD.softmax_T(host_rows(logits, 2)[0], 1e38, 0, 0.5)
    assert probs.tolist() == [0.0, 1.0]
    toks, _ = _draw_many(H, logits, 2, 1e38, 0, 0.5, 3, 0, 64)
    assert (toks == 1).all()


# ---------------------------------------------------------------------------------------------- accept chain
def run_chain(h, logits, vocab, guess, T, top_k=0, top_p=1.0, seed=21, offset=0):
    """One launch against verify_given_uniforms fed the host Philox's uniforms."""
    meta = h.set_guess(guess)
    h.seed(seed, offset)
    rec = h.launch(logits, vocab, meta, T, top_k, top_p).cpu().tolist()
    rows = host_rows(logits, vocab)
    n_u = 4 * len(guess) + 8
    us = PX.uniforms(seed, offset, n_u).astype(np.float64)
    want = SD.verify_given_uniforms(rows[0], rows[1 + WCAP:], guess, GS, T, us.tolist(), top_k, top_p)
    exp = h.exported()
    assert np.array_equal(bits_of(exp), bits_of(us[:len(exp)].astype(np.float32)))
    for c in want["checks"]:
        if c[0] == "accept":
            assert abs(c[1] - c[2]) > 1e-4, "uniform too close to its threshold: pick another offset"
    assert want["used"] == len(exp), f"kernel drew {len(exp)}, restatement {want['used']}"
    n_hits = rec[1] + 1
    assert want["n_hits"] == n_hits
    hits = rec[3:3 + n_hits]
    for k, t in enumerate(want["hits"]):
        if t is None:
            _, u, probs = [c for c in want["checks"] if c[0] == "draw"][-1][:3]
            assert SD.draw_is_consistent(u, probs, hits[k]), "residual draw"
        else:
            assert hits[k] == t, f"accepted token {k}"
    if n_hits > 1:
        assert rec[R] == want["max_hit_idx"]
    return rec, want


def _peak(vocab, tok, rng, h=8.0):
    r = rng.normal(0, 1.0, vocab)
    r[tok] = h
    return r


def _offset_where(seed, pred, n=8, limit=1 << 16):
    u = PX.uniforms(seed, 0, limit + n).astype(np.float64)
    for o in range(limit):
        if pred(u[o:o + n]):
            return o
    pytest.fail("no offset found")


def test_chain_candidate_outside_top_k_draws_a_uniform_and_rejects(H):
    rng = np.random.default_rng(3)
    vocab = 4096
    row = rng.normal(0, 1.0, vocab); row[[10, 20, 30]] = [3.0, 2.9, 2.8]; row[40] = -6.0
    logits = step_rows(H, row)
    guess = [40, 1, 2, 10, 1, 2]                        # n-gram 0 proposes a token top-k removes
    rec, want = run_chain(H, logits, vocab, guess, 1.0, top_k=20,
                          offset=_offset_where(21, lambda u: u[1] < 0.02))
    assert want["checks"][0][2] == 0.0 and rec[3] == 10 and want["used"] >= 2


def test_chain_duplicate_candidate_gets_zero_probability(H):
    rng = np.random.default_rng(4)
    vocab = 4096
    row = rng.normal(0, 1.0, vocab); row[[10, 20]] = [8.0, 7.5]
    logits = step_rows(H, row)
    guess = [10, 1, 2, 10, 3, 4, 20, 5, 6]              # n-grams 0 and 1 both propose 10
    off = _offset_where(21, lambda u: u[0] > 0.5 and u[1] < 0.1 and u[2] < 0.1)
    rec, want = run_chain(H, logits, vocab, guess, 1.0, offset=off)
    assert want["checks"][1][2] == 0.0 and rec[3] == 20 and rec[R] == 2


def test_chain_all_rejected_then_residual_excludes_them(H):
    rng = np.random.default_rng(5)
    vocab = 4096
    row = rng.normal(0, 0.5, vocab); row[[10, 20, 30]] = [9.0, 8.8, 8.6]     # most of the mass on the candidates
    logits = step_rows(H, row)
    guess = [10, 1, 2, 20, 1, 2, 30, 1, 2]
    probs = SD.softmax_T(host_rows(logits, vocab)[0], 1.0)
    seen = set()
    for trial in range(6):
        p0 = probs[10]
        off = _offset_where(21 + trial, lambda u: u[0] > min(0.999, p0 + 0.01) and u[1] > 0.97 and u[2] > 0.9)
        rec, want = run_chain(H, logits, vocab, guess, 1.0, seed=21 + trial, offset=off)
        assert want["hits"] == [None] and rec[3] not in (10, 20, 30)
        seen.add(rec[3])
    assert len(seen) >= 2


def test_chain_full_acceptance_to_gs(H):
    rng = np.random.default_rng(6)
    vocab = 4096
    guess = [100, 101, 102, 200, 201, 202]
    row0 = _peak(vocab, 200, rng, 16.0)
    gr = {GS + i: _peak(vocab, 201 + i, rng, 16.0) for i in range(GS - 1)}
    logits = step_rows(H, row0, gr)
    off = _offset_where(21, lambda u: u[0] > 0.01 and max(u[1], u[2], u[3]) < 0.9)
    rec, want = run_chain(H, logits, vocab, guess, 1.0, offset=off)
    assert rec[1] == GS - 1 and rec[3:3 + GS] == [200, 201, 202] and rec[R] == 1


def test_chain_accept_at_later_ngram_and_position_picks_the_right_row(H):
    """n-grams 0 and 1 share position 0; at position 1 n-gram 0 is rejected and n-gram 1 accepted, so position 2 is
    decided by row 1 + WCAP + 1*GS + 1, the only row that makes 303 likely."""
    rng = np.random.default_rng(8)
    vocab = 4096
    guess = [300, 301, 302, 300, 311, 303, 300, 321, 322]
    row0 = _peak(vocab, 300, rng, 14.0)
    gr = {j: _peak(vocab, 900 + j, rng, 14.0) for j in range(3 * GS)}
    gr[0] = rng.normal(0, 1.0, vocab); gr[0][[301, 311]] = [10.0, 10.0]      # row after 300: 301 and 311 each ~1/2
    gr[GS + 1] = _peak(vocab, 303, rng, 14.0)
    logits = step_rows(H, row0, gr)
    off = _offset_where(21, lambda u: u[0] < 0.99 and u[1] > 0.7 and u[2] < 0.3 and u[3] < 0.99)
    rec, want = run_chain(H, logits, vocab, guess, 1.0, offset=off)
    assert rec[3:3 + GS] == [300, 311, 303] and rec[R] == 1 and rec[1] == GS - 1


# ---------------------------------------------------------------------------------------------- distribution
def enumerate_outcomes(rows, guess, T, top_k=0, top_p=1.0):
    """Exact float64 distribution of (emitted tokens, max_hit_idx) under the reference procedure."""
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
                        SD.softmax_T(rows[1 + WCAP + e * GS + i], T, top_k, top_p), h2, e, w * p)
            w *= 1.0 - p
            if w <= 0:
                return
            probs[d] = 0.0
            probs = probs / probs.sum()
        for t in np.nonzero(probs)[0]:
            add((hits + (int(t),), mhi if hits else 0), w * float(probs[t]))

    pos(0, list(range(n_ng)), SD.softmax_T(rows[0], T, top_k, top_p), (), 0, 1.0)
    return out


def _g_test(obs, exp_p, n):
    from scipy.stats import chi2
    keys = [k for k, p in exp_p.items() if n * p >= 5]
    o = np.array([obs.get(k, 0) for k in keys] + [n - sum(obs.get(k, 0) for k in keys)], dtype=np.float64)
    e = np.array([n * exp_p[k] for k in keys] + [n * (1.0 - sum(exp_p[k] for k in keys))])
    if e[-1] < 5:
        o, e = o[:-1], e[:-1]
    m = o > 0
    g = 2.0 * float((o[m] * np.log(o[m] / e[m])).sum())
    return g, len(o) - 1, chi2.sf(g, len(o) - 1)


def test_emitted_distribution_matches_exact_enumeration(H):
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
    exact = enumerate_outcomes(rows, guess, 1.0)
    assert abs(sum(exact.values()) - 1.0) < 1e-9
    n = 1 << 16
    meta = H.set_guess(guess)
    recs = torch.zeros(n, REC, dtype=torch.int32, device="cuda")
    H.seed(4242, 0)
    for j in range(n):
        H.launch(logits, vocab, meta, 1.0, rec=recs[j], dbg=False)
    rc = recs.cpu().numpy()
    obs = {}
    for r in rc:
        nh = int(r[1]) + 1
        key = (tuple(int(x) for x in r[3:3 + nh]), int(r[R]) if nh > 1 else 0)
        obs[key] = obs.get(key, 0) + 1
    assert set(obs) <= set(exact), f"outcomes the procedure cannot emit: {sorted(set(obs) - set(exact))[:3]}"
    g, df, p = _g_test(obs, exact, n)
    print(f"G = {g:.1f} on {df} dof, p = {p:.3g}; multi-token outcomes: "
          f"{sum(v for k, v in obs.items() if len(k[0]) > 1) / n:.3f}")
    assert p > 1e-6 and df >= 10
    first = {}
    for (hits, _), w in exact.items():
        first[hits[0]] = first.get(hits[0], 0.0) + w
    marg = SD.softmax_T(rows[0], 1.0)
    for t, w in first.items():
        assert abs(w - marg[t]) < 1e-9                     # the procedure's first token is exactly the softmax
    obs1 = {}
    for r in rc:
        obs1[int(r[3])] = obs1.get(int(r[3]), 0) + 1
    g1, df1, p1 = _g_test(obs1, {int(t): float(marg[t]) for t in np.nonzero(marg)[0]}, n)
    assert p1 > 1e-6 and df1 >= 5


# ---------------------------------------------------------------------------------------------- EOS, done, determinism
def test_eos_in_the_window_is_replaced_by_a_predicted_old_token(H):
    rng = np.random.default_rng(10)
    vocab = 4096
    row = _peak(vocab, 77, rng, 3.0)
    logits = step_rows(H, row)
    d = H.d
    old = list(range(500, 540))
    saved = H.st[d.off_old:d.off_old + len(old)].clone(), H.st[S_N_OLD].clone()
    H.st[d.off_old:d.off_old + len(old)] = torch.tensor(old, dtype=torch.int32)
    H.st[S_N_OLD] = len(old)
    am_saved = H.am.clone()
    win = [3, EOS, 8, EOS, EOS, 9, EOS]
    H.am[1:1 + W] = torch.tensor(win, dtype=torch.int32)
    try:
        for seed in (1, 2, 3):
            meta = H.set_guess([77, 1, 2, 78, 1, 2])
            H.seed(seed, 9)
            rec = H.launch(logits, vocab, meta, 1.0).cpu().tolist()
            us = H.exported()
            assert np.array_equal(bits_of(us), bits_of(PX.uniforms(seed, 9, len(us))))
            n_eos = win.count(EOS)
            tail = us[len(us) - n_eos:]
            want, k = [], 0
            for v in win:
                if v == EOS:
                    j = min(int(np.float32(tail[k]) * np.float32(len(old))), len(old) - 1)
                    want.append(old[j]); k += 1
                else:
                    want.append(v)
            assert rec[R + 1] & 2 and rec[R + 4:R + 4 + W] == want
            assert H.rng.cpu().tolist() == [seed, 9 + PX.advance(len(us))]
    finally:
        H.st[d.off_old:d.off_old + len(old)], H.st[S_N_OLD] = saved
        H.am.copy_(am_saved)


def test_finished_state_writes_a_zero_record_and_draws_nothing(H):
    logits = step_rows(H, np.zeros(4096))
    meta = H.set_guess([1, 2, 3])
    H.st[S_DONE] = 1
    try:
        H.seed(5, 13)
        rec = H.launch(logits, 4096, meta, 1.0)
        assert rec.cpu().tolist() == [0] * REC
        assert H.rng.cpu().tolist() == [5, 13]
    finally:
        H.st[S_DONE] = 0


def test_top_p_cut_near_a_bucket_edge_is_deterministic(H):
    rng = np.random.default_rng(12)
    vocab = 32000
    row = rng.normal(0, 0.3, vocab)
    logits = logits_tensor(H, row)
    s = host_rows(logits, vocab)[0]
    e = np.exp(s - s.max())
    vals = np.unique(s)
    cum = np.cumsum([e[s == v].sum() for v in vals])
    j = int(np.searchsorted(cum, 0.6 * cum[-1]))
    meta = H.plain_meta()
    for top_p in (1.0 - cum[j] / cum[-1], 1.0 - cum[j + 1] / cum[-1]):       # float64 cut on a boundary
        first = None
        for rep in range(100):
            H.seed(8, 0)
            recs = torch.zeros(8, REC, dtype=torch.int32, device="cuda")
            for o in range(8):
                H.launch(logits, vocab, meta, 1.0, 0, float(top_p), rec=recs[o], dbg=False)
            got = recs.cpu()
            if first is None:
                first = got
            assert torch.equal(got, first), f"top_p={top_p}: launch {rep} differs"
