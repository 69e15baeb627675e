"""Greedy logits processors on device (``lade_argmax_processed``) against HF's own processors run on the GPU.

* kernel exactness: a tiny engine's ctx serves direct launches; the test writes ``out_ids``, ``n_out``, the guess count
  and the guess tokens through a view of its device state.  Every lm slot must equal
  ``torch.argmax(processors(prefix[None], logits[slot].float()[None]))`` with the prefix the slot stands for (slot 0: the
  committed ids; verification slot of n-gram e, position u: the committed ids + the n-gram's tokens 0..u; window slots:
  plain argmax), for bf16 and fp16, vocab 32000 and 128256, padded rows, all -inf rows, and penalty ties where
  ``x / p`` and ``x * (1 / p)`` round differently.  With no processor active the output is lade_argmax_rows' bit for bit.
* end to end: lookahead (W15 N5 G15, pool from prompt) == the engine's own G = 0 run with the same processors, each
  alone and all combined; graph == eager, pipelined == synchronous; through the plugin, ``model.generate`` with
  repetition_penalty / no_repeat_ngram_size / min_new_tokens under USE_LADE=1 == HF's greedy.  A divergence is allowed
  only at a tie within 3 bf16 ulps of the processed fp32 oracle scores (oracle.llama_ref forward, then HF's
  processors)."""
import ctypes as C
import random

import numpy as np
import pytest
import torch
from transformers.generation.logits_process import (MinLengthLogitsProcessor, NoRepeatNGramLogitsProcessor,
                                                    RepetitionPenaltyLogitsProcessor)

pytestmark = pytest.mark.gpu

W, N, G = 7, 4, 7
GS, WCAP = N - 1, W + N - 3
LM_CAP = 1 + WCAP + G * GS
S_N_OUT, S_N_GUESS_TOK = 3, 9
DTYPES = [torch.bfloat16, torch.float16]


class _Dims(C.Structure):                  # lade::Dims (csrc/state.cuh)
    _fields_ = [(n, C.c_int32) for n in "W N G GS WCAP V cap pool_from_prompt n_eos D rank".split()] + \
               [("eos", C.c_int32 * 4), ("lm_cap", C.c_int32)] + \
               [(n, C.c_int32) for n in "off_win off_win_len off_guess off_out off_old off_cnt".split()] + \
               [("off_tup", C.c_int64), ("total_ints", C.c_int64)]


class _DevInts:
    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = dict(shape=(n,), typestr="<i4", data=(ptr, False), version=3)


def hf_processors(d):
    out = []
    if d.get("penalty") is not None:
        out.append(RepetitionPenaltyLogitsProcessor(float(d["penalty"]), d.get("prompt_ignore_length") or None))
    if d.get("ngram_size") is not None:
        out.append(NoRepeatNGramLogitsProcessor(int(d["ngram_size"])))
    if d.get("min_length") is not None and d.get("eos_token_id"):
        out.append(MinLengthLogitsProcessor(int(d["min_length"]), list(d["eos_token_id"]), device="cuda"))
    return out


def hf_scores(procs, prefix, row):
    s = row.float()[None].clone()
    ids = torch.tensor([prefix], dtype=torch.long, device="cuda")
    for p in procs:
        s = p(ids, s)
    return s[0]


class Harness:
    def __init__(self, dtype):
        from lookaheaddecoding_b200 import LookaheadEngine, _cabi
        from test_gpu_sampling_device import _prompt, peaked_periodic_model
        model = peaked_periodic_model()
        if dtype != torch.bfloat16:
            model = model.to(dtype)
        self.C, self.dtype = _cabi, dtype
        eng = LookaheadEngine(model, W, N, G, pool_from_prompt=True, max_total_len=256, use_cuda_graph=False)
        prompt = _prompt(24)
        eng.begin(prompt, 256, (), eng.draw_window(prompt, random.Random(3)))
        torch.cuda.synchronize()
        ctx = type("_Ctx", (C.Structure,), {"_fields_": [("cfg", _cabi.LadeConfig), ("d", _Dims),
                                                           ("state", C.c_void_p)]}).from_address(eng._ctx.value)
        d = ctx.d
        assert (d.W, d.N, d.G, d.GS, d.WCAP, d.lm_cap) == (W, N, G, GS, WCAP, LM_CAP), "ctx layout"
        self.eng, self.d = eng, d
        self.st = torch.as_tensor(_DevInts(ctx.state, int(d.total_ints)), device="cuda")
        self.am = torch.zeros(LM_CAP, dtype=torch.int32, device="cuda")
        self.proc = torch.zeros(C.sizeof(_cabi.LadeProcessors) // 4, dtype=torch.int32, device="cuda")

    def set_state(self, out_ids, guess):
        d = self.d
        self.st[S_N_OUT] = len(out_ids)
        self.st[S_N_GUESS_TOK] = len(guess)
        self.st[d.off_out:d.off_out + len(out_ids)] = torch.tensor(out_ids, dtype=torch.int32)
        if guess:
            self.st[d.off_guess:d.off_guess + len(guess)] = torch.tensor(guess, dtype=torch.int32)

    def launch(self, logits, vocab, procs):
        from lookaheaddecoding_b200.engine import processors_record
        stream = torch.cuda.current_stream().cuda_stream
        rec = processors_record(procs)
        self.C.check(self.eng.lib.lade_processors_upload(stream, C.byref(rec), self.proc.data_ptr()), "upload")
        self.am.fill_(-1)
        self.C.check(self.eng.k_argmax_processed(self.eng._ctx, stream, logits.data_ptr(), logits.shape[0], vocab,
                                                 logits.shape[1], self.proc.data_ptr(), self.am.data_ptr()),
                     "lade_argmax_processed")
        return self.am.cpu().tolist()

    def plain(self, logits, vocab):
        stream = torch.cuda.current_stream().cuda_stream
        am = torch.full((logits.shape[0],), -1, dtype=torch.int32, device="cuda")
        self.C.check(self.eng.k_argmax_rows(stream, logits.data_ptr(), logits.shape[0], vocab, logits.shape[1],
                                            am.data_ptr()), "lade_argmax_rows")
        return am.cpu().tolist()


@pytest.fixture(scope="module", params=DTYPES, ids=["bf16", "fp16"])
def H(request):
    h = Harness(request.param)
    yield h
    h.eng.close()


def to_dev(h, rows, ld=None, pad=None):
    vocab = rows.shape[1]
    ld = ld or vocab
    full = np.full((rows.shape[0], ld), torch.finfo(h.dtype).max if pad is None else pad, dtype=np.float32)
    full[:, :vocab] = rows
    return torch.tensor(full).to(h.dtype).cuda()


def slot_prefix(slot, out_ids, guess):
    """The prefix HF would hold for lm slot `slot`, or None for a plain-argmax slot."""
    if slot == 0:
        return list(out_ids)
    i = slot - 1 - WCAP
    if 0 <= i < len(guess):
        e, u = divmod(i, GS)
        return list(out_ids) + guess[e * GS:e * GS + u + 1]
    return None


def expected(h, logits, vocab, procs, out_ids, guess):
    hp = hf_processors(procs)
    want, changed = [], 0
    for s in range(logits.shape[0]):
        row = logits[s, :vocab]
        raw = int(torch.argmax(row.float()))
        pre = slot_prefix(s, out_ids, guess)
        got = raw if pre is None else int(torch.argmax(hf_scores(hp, pre, row)))
        changed += got != raw
        want.append(got)
    return want, changed


def check(h, logits, vocab, procs, out_ids, guess, what):
    h.set_state(out_ids, guess)
    got = h.launch(logits, vocab, procs)
    want, changed = expected(h, logits, vocab, procs, out_ids, guess)
    bad = [(s, got[s], want[s]) for s in range(len(want)) if got[s] != want[s]]
    assert not bad, f"{what}: slots (slot, kernel, HF) {bad[:6]}"
    return changed


def crafted_rows(rng, vocab, hot, n_rows=LM_CAP):
    """Random rows whose `hot` tokens (the prefix alphabet, eos ids) score around each row's maximum, both signs."""
    rows = rng.normal(0.0, 1.0, (n_rows, vocab)).astype(np.float32)
    top = rows.max(axis=1, keepdims=True)
    rows[:, hot] = top * rng.uniform(-1.4, 1.4, (n_rows, len(hot))).astype(np.float32)
    return rows


def _prefix_patterns(rng, alphabet, n_out):
    yield "mixed", [int(x) for x in rng.choice(alphabet[:4], n_out)]
    yield "aaaa", [alphabet[0]] * n_out


@pytest.mark.parametrize("vocab", [32000, 128256])
def test_every_slot_equals_hf_processors(H, vocab):
    rng = np.random.default_rng(vocab)
    alphabet = [5, 17, 300, vocab - 1, 4242, 77]
    eos = [alphabet[2], alphabet[5], vocab - 2]
    n_out = 40
    lg = 5 * GS                                         # 5 n-grams; verification slots past lg are never read
    changed_by = {}
    for pat, out_ids in _prefix_patterns(rng, alphabet, n_out):
        guess = [int(x) for x in rng.choice(alphabet[:4], lg)]
        configs = [("penalty", {"penalty": p}) for p in (1.3, 0.8, 1.0, 2.5)]
        configs += [("penalty", {"penalty": 1.3, "prompt_ignore_length": k}) for k in (17, n_out + 2)]
        configs += [("ngram", {"ngram_size": n}) for n in (1, 2, 3, 5)]
        configs += [("ngram", {"ngram_size": n_out + 2}), ("ngram", {"ngram_size": n_out + 3})]   # len + 1 < n edges
        configs += [("minlen", {"min_length": n_out + k, "eos_token_id": eos}) for k in range(-1, GS + 2)]
        configs += [("all", {"penalty": 1.2, "prompt_ignore_length": 3, "ngram_size": 3, "min_length": n_out + 2,
                             "eos_token_id": eos})]
        for kind, procs in configs:
            rows = crafted_rows(rng, vocab, alphabet + eos)
            if kind == "minlen":
                rows[:, eos] = np.abs(rows).max(axis=1, keepdims=True) * 2.0          # eos is the raw maximum
            ld, pad = (vocab + 16, None) if vocab == 32000 else (vocab + 8, float("nan"))
            logits = to_dev(H, rows, ld, pad)
            changed_by[kind] = changed_by.get(kind, 0) + check(H, logits, vocab, procs, out_ids, guess,
                                                               f"{pat} {procs}")
    for kind in ("penalty", "ngram", "minlen", "all"):
        assert changed_by[kind] > 0, f"no probe where {kind} changes the argmax"


def test_signed_zeros_all_minus_inf_rows_and_no_processor(H):
    vocab = 32000
    rng = np.random.default_rng(1)
    out_ids, guess = [9, 10, 11, 9, 10] * 4, [9, 12, 10, 11, 9, 13]
    rows = -np.abs(rng.normal(0, 1, (LM_CAP, vocab))).astype(np.float32) - 1.0
    rows[:, 9], rows[:, 10], rows[:, 12] = -0.0, 0.0, -0.0
    rows[3] = -np.inf
    rows[1 + WCAP + 2] = -np.inf                          # a verification row of n-gram 0 that accept reads
    logits = to_dev(H, rows)
    for procs in ({"penalty": 1.3}, {"penalty": 0.6}, {"ngram_size": 2}, {"penalty": 1.3, "ngram_size": 1}):
        check(H, logits, vocab, procs, out_ids, guess, f"zeros {procs}")
    assert H.launch(logits, vocab, {"ngram_size": 1})[1 + WCAP + 2] == 0
    for ld, pad in ((vocab, None), (vocab + 24, float("nan"))):
        lg = to_dev(H, crafted_rows(rng, vocab, [9, 10, 11]), ld, pad)
        H.set_state(out_ids, guess)
        assert H.launch(lg, vocab, {}) == H.plain(lg, vocab)
        assert H.launch(lg, vocab, {"min_length": 3, "eos_token_id": [9]}) == H.plain(lg, vocab)   # bound not reached


def test_token_only_in_a_guess_is_penalised_in_its_ngram_only(H):
    vocab = 32000
    rng = np.random.default_rng(2)
    X, Z = 31000, 20000                                   # X: only in n-gram 1; Z: in no prefix
    out_ids = [int(x) for x in rng.integers(3, 1000, 30)]
    guess = [int(x) for x in rng.integers(3, 1000, 3 * GS)]
    guess[GS + 1] = X                                     # n-gram 1, position 1
    rows = rng.normal(0, 1, (LM_CAP, vocab)).astype(np.float32)
    rows[:, X], rows[:, Z] = 6.0, 5.5
    logits = to_dev(H, rows)
    check(H, logits, vocab, {"penalty": 1.3}, out_ids, guess, "guess-only token")
    got = H.launch(logits, vocab, {"penalty": 1.3})
    ng1 = [1 + WCAP + GS + u for u in range(GS)]
    assert got[0] == X and got[ng1[0]] == X and got[ng1[1]] == Z and got[ng1[2]] == Z
    assert all(got[1 + WCAP + u] == X for u in range(GS)) and all(got[1 + WCAP + 2 * GS + u] == X for u in range(GS))


def _division_probe(dtype):
    """(penalty, x, y): x > 0 representable in `dtype`, y = fp32(x * fp32(1 / p)) also representable, and fp32(x / p)
    != y -- a penalised x then ties y under torch's CUDA reciprocal multiply but not under a true division."""
    bits = np.arange(0x0001, 0x7c00 if dtype == torch.float16 else 0x7f80, dtype=np.int64)
    xs = torch.tensor(bits.astype(np.int16)).view(dtype).float().numpy()
    xs = xs[(xs > 0.5) & (xs < 1000)]
    for p in np.float32(1.0) + np.arange(1, 400, dtype=np.float32) * np.float32(0.0025):
        inv = np.float32(1.0) / p
        a = xs * inv
        b = xs / p
        rep = torch.tensor(a).to(dtype).float().numpy() == a
        hit = np.nonzero((a != b) & rep)[0]
        if len(hit):
            k = hit[0]
            return float(p), float(xs[k]), float(a[k]), bool(b[k] > a[k])
    return None


def test_penalty_ties_follow_the_reciprocal_multiply(H):
    probe = _division_probe(H.dtype)
    assert probe is not None, "no x / p vs x * (1/p) rounding probe found"
    p, x, y, div_larger = probe
    vocab = 32000
    tx = 700
    ty = 600 if div_larger else 800                       # the tie goes to the lower index: y under the multiply
    out_ids = [tx, 5, 6]
    rows = np.full((LM_CAP, vocab), -4.0, dtype=np.float32)
    rows[:, tx], rows[:, ty] = x, y
    logits = to_dev(H, rows)
    h_ids = hf_processors({"penalty": p})
    s = hf_scores(h_ids, out_ids, logits[0, :vocab])
    assert s[tx].item() == y, "HF on the GPU does not compute x * fp32(1/p)"
    H.set_state(out_ids, [])
    got = H.launch(logits, vocab, {"penalty": p})[0]
    true_div = tx if div_larger else ty
    assert got == int(torch.argmax(s)) and got != true_div
    # penalty-made exact ties: 2x / 2 == x, lowest index wins either way round
    rows[:, tx], rows[:, ty] = 2.0, 1.0
    for other in (600, 800):
        rows2 = rows.copy()
        rows2[:, ty], rows2[:, other] = -4.0, 1.0
        check(H, to_dev(H, rows2), vocab, {"penalty": 2.0}, out_ids, [], f"exact tie at {other}")


def test_vocab_too_large_is_refused(H):
    big = torch.zeros(1, 160 * 1024 + 8, dtype=H.dtype, device="cuda")
    rc = H.eng.k_argmax_processed(H.eng._ctx, torch.cuda.current_stream().cuda_stream, big.data_ptr(), 1,
                                  big.shape[1], big.shape[1], H.proc.data_ptr(), H.am.data_ptr())
    assert rc == H.C.LADE_EUNSUPPORTED


# ------------------------------------------------------------------------------------------------ end to end
def _first_diff(a, b):
    return next((k for k in range(min(len(a), len(b))) if a[k] != b[k]), None)


@torch.no_grad()
def _oracle_scores(model, prefix, procs):
    """Processed fp32 scores of the next position after `prefix`: oracle.llama_ref's forward over the model's own weights
    (plain causal, no cache), then HF's processors."""
    from oracle import llama_ref as LR
    from test_gpu_sampling_device import TINY
    orc = LR.OracleLlama(TINY, {k: v.detach() for k, v in model.state_dict().items()}, device="cuda")
    n = len(prefix)
    logits = orc.forward_rows(prefix, list(range(n)), torch.tril(torch.ones(n, n, dtype=torch.bool)), 0)
    return hf_scores(hf_processors(procs), prefix, logits[-1])


def _assert_equal_up_to_a_tie(model, a, b, procs, what):
    """a == b, or the first differing position is a tie within 3 bf16 ulps of the oracle's processed scores."""
    i = _first_diff(a, b)
    if i is None:
        assert len(a) == len(b), what
        return
    s = _oracle_scores(model, a[:i], procs)
    top = s.max().item()
    ulp3 = 3 * 2.0 ** (np.floor(np.log2(abs(top))) - 7)
    assert top - s[a[i]].item() <= ulp3 and top - s[b[i]].item() <= ulp3, \
        f"{what}: diverged at {i} without a tie ({s[a[i]].item()}, {s[b[i]].item()}, top {top})"


def _repeats_3gram(ids, start):
    seen = {tuple(ids[j - 2:j + 1]) for j in range(2, start)}
    for k in range(start, len(ids)):
        g = tuple(ids[k - 2:k + 1])
        if g in seen:
            return True
        seen.add(g)
    return False


@pytest.mark.parametrize("scale", [30.0, 4.0])
def test_lookahead_equals_g0_run_with_the_same_processors(scale):
    from lookaheaddecoding_b200 import LookaheadEngine
    from test_gpu_sampling_device import _in_cycle_prompt, peaked_periodic_model
    model = peaked_periodic_model(scale=scale)
    prompt = _in_cycle_prompt(model, 32)
    P, M = len(prompt), 96
    la = LookaheadEngine(model, 15, 5, 15, pool_from_prompt=True, max_total_len=P + M)
    g0 = LookaheadEngine(model, 15, 5, 0, max_total_len=P + M)
    free = g0.generate(prompt, M, rng=random.Random(1))
    eos = [free[P + 3], free[P + 9]]
    configs = {"penalty": {"penalty": 1.3}, "ngram": {"ngram_size": 3},
               "minlen": {"min_length": P + 40, "eos_token_id": eos},
               "all": {"penalty": 1.3, "ngram_size": 3, "min_length": P + 40, "eos_token_id": eos}}
    best_rate = 0.0
    for name, procs in configs.items():
        e = eos if "min_length" in procs else ()
        ref = g0.generate(prompt, M, eos_token_ids=e, rng=random.Random(1), processors=procs)
        out = la.generate(prompt, M, eos_token_ids=e, rng=random.Random(1), processors=procs)
        best_rate = max(best_rate, (len(out) - P) / la.last_steps)
        _assert_equal_up_to_a_tie(model, out, ref, procs, f"scale {scale} {name}")
        if name == "all":
            assert not any(t in eos for t in out[P:P + 40])
            assert not _repeats_3gram(out, P) and _repeats_3gram(free, P)
            for graph, pipe in ((False, True), (True, False), (False, False)):
                other = LookaheadEngine(model, 15, 5, 15, pool_from_prompt=True, max_total_len=P + M,
                                        use_cuda_graph=graph, pipeline_host=pipe)
                assert other.generate(prompt, M, eos_token_ids=e, rng=random.Random(1), processors=procs) == out, \
                    f"graph={graph} pipelined={pipe}"
                other.close()
    # the engine switches back to plain argmax when a later call has no processors
    assert g0.generate(prompt, M, rng=random.Random(1)) == free
    print(f"scale {scale}: best tokens per step under processing {best_rate:.2f}")
    if scale == 30.0:
        assert best_rate > 1.3
    la.close()
    g0.close()


def test_plugin_generate_with_processors_equals_hf_greedy(monkeypatch):
    import lade
    from lookaheaddecoding_b200.decoding import FUNC_MAP
    from test_gpu_sampling_device import _in_cycle_prompt, peaked_periodic_model
    model = peaked_periodic_model(scale=30.0)
    prompt = _in_cycle_prompt(model, 32)
    P = len(prompt)
    ids = torch.tensor([prompt], device="cuda")
    model.generation_config.pad_token_id = 0
    lade.augment_all()
    try:
        lade.config_lade(LEVEL=5, WINDOW_SIZE=15, GUESS_SET_SIZE=15, DEBUG=0, POOL_FROM_PROMPT=True)
        kw = dict(attention_mask=torch.ones_like(ids), max_new_tokens=64, do_sample=False)
        monkeypatch.setenv("USE_LADE", "1")
        free = model.generate(ids, **kw)[0].tolist()
        eos = free[P + 5]
        model.generation_config.eos_token_id = eos
        pk = dict(kw, repetition_penalty=1.3, no_repeat_ngram_size=3, min_new_tokens=40)
        got = model.generate(ids, **pk)[0].tolist()
        monkeypatch.setenv("USE_LADE", "0")
        want = model.generate(ids, **pk)[0].tolist()
        assert "_sample" in FUNC_MAP
        procs = {"penalty": 1.3, "ngram_size": 3, "min_length": P + 40, "eos_token_id": [eos]}
        _assert_equal_up_to_a_tie(model, got, want, procs, "plugin vs HF greedy")
        assert eos not in got[P:P + 40] and not _repeats_3gram(got, P) and _repeats_3gram(free, P)
    finally:
        lade.restore_generate()
