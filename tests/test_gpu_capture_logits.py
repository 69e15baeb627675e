"""Per-token logits from lookahead generate(): lade_capture_rows inside the step, the engine's capture_logits and HF's
return_dict_in_generate / output_logits / output_scores on the plugin surface.

* slot exactness, lockstep: an eager engine one step at a time; after each step every captured row equals, bit for bit,
  eng.logits at the slot this test derives itself (greedy: the step record's max_hit_idx; sampling: the first n-gram
  of the step's guess rows that carries the hits), greedy with and without processors, sampling with T / top-k / top-p
  and with the min_p / eta cuts, bf16 and fp16, head_dim 128 and 64, and a Qwen3 model; rows past the last written one
  and past the buffer stay NaN, and a step on the finished state writes nothing;
* decisions replay from the captured rows alone: greedy argmax (scores under the processors), and the sampling
  verification restated (oracle/sampling_device.py) with the exported uniforms on guess rows that are NaN except where a
  row was captured;
* graph / eager / pipelined / synchronous give bit-identical rows, and capture on changes nothing but the one launch;
* edges: EOS inside a multi-token accept, max_new_tokens 1 and one that ends mid-accept, argument errors;
* against HF's own generate(): output types, shapes, dtype, device; logits within the tie tolerance where the ids agree;
  compute_transition_scores finite.

The "periodic with attention" Llama of test_gpu_step_fp64 (cyclic weights, a small random o_proj, lm_head scaled)
accepts guesses on many steps, so the slots past 0 really are exercised: each lockstep case asserts a minimum number of
steps with max_hit >= 2.
"""
import random

import numpy as np
import pytest
import torch

from oracle import sampling_device as SD

pytestmark = pytest.mark.gpu

PERIODIC = dict(hidden=256, layers=2, heads=2, kv_heads=2, inter=688, vocab=4096, max_pos=2048, rope_theta=10000.0,
                eps=1e-5)
PERIODIC_D64 = dict(PERIODIC, heads=4, kv_heads=2)
O_SCALE, LM_SCALE = 0.001, 30.0
W, N, G = 7, 4, 7
P, NEW = 24, 96
MIN_MULTI = 5                 # steps with max_hit >= 2 a periodic lockstep run must see


def periodic_model(shape=PERIODIC, dtype=torch.bfloat16):
    from bench import build_model
    model = build_model(shape, torch.device("cuda"), seed=0, weights="cyclic", dtype=dtype)
    g = torch.Generator(device="cuda").manual_seed(11)
    with torch.no_grad():
        model.lm_head.weight.mul_(LM_SCALE)
        for layer in model.model.layers:
            layer.self_attn.o_proj.weight.normal_(0.0, O_SCALE, generator=g)
    model.generation_config.pad_token_id = 0
    model.generation_config.eos_token_id = None
    return model


def _prompt(n=P, vocab=4096, seed=1):
    return torch.randint(3, vocab, (n,), generator=torch.Generator().manual_seed(seed)).tolist()


def _bits(t):
    return t.contiguous().view(torch.int16)


def _engine(model, max_total_len, **kw):
    from lookaheaddecoding_b200 import LookaheadEngine
    return LookaheadEngine(model, kw.pop("W", W), kw.pop("N", N), kw.pop("G", G), pool_from_prompt=True,
                           max_total_len=max_total_len, **kw)


def _set_sampling(eng, s):
    eng.sample_temperature, eng.sample_top_k, eng.sample_top_p = s.get("temperature", 1.0), s.get("top_k", 0), \
        s.get("top_p", 1.0)
    eng.sample_min_p, eng.sample_epsilon, eng.sample_eta = s.get("min_p", 0.0), s.get("epsilon", 0.0), s.get("eta", 0.0)


def lockstep(eng, prompt, new, sampling=None, processors=None, canary=3, tag=False):
    """Run `eng` (eager) one step at a time with capture on, checking every step's captured rows against eng.logits at
    the slots derived here.  Returns the per-step records (hits, guess tokens, captured rows, uniforms).
    `tag`: after each step's commit (its decisions made), the last column of every lm slot is overwritten with the slot's
    index, before the capture copies.  Guess rows with the same prefix have the same bits (every kernel of the step is
    row-independent), so without the tag a capture of the wrong n-gram's row would go unseen."""
    from lookaheaddecoding_b200 import _cabi
    from lookaheaddecoding_b200.engine import decided_slots
    n_p = len(prompt)
    commit = "sample" if sampling is not None else True
    rows = new + eng.GS
    big = torch.full((rows + canary, eng.V), float("nan"), dtype=eng.dt, device="cuda")
    eng.capture_buf = big[:rows]
    if sampling is not None:
        _set_sampling(eng, sampling)
        eng.debug_uniforms = torch.zeros(4 + eng.G * eng.GS + eng.W, dtype=torch.float32, device="cuda")
    eng.begin(prompt, n_p + new, (), eng.draw_window(prompt, random.Random(3)), processors, capture_logits=True)
    assert eng.capture_buf.data_ptr() == big.data_ptr()          # reused, canary rows behind it
    if tag:
        commit_stage = eng._commit
        slot_ids = torch.arange(eng.lm_cap, device="cuda").to(eng.dt)

        def tagged_commit(stream, commit_):
            n = commit_stage(stream, commit_)
            eng.logits[:, -1] = slot_ids
            return n
        eng._commit = tagged_commit
    if sampling is not None:
        eng.rng_state.copy_(torch.tensor([1234, 0], dtype=torch.int64))
    steps = []
    for step in range(new + eng.N + 4):
        eng.run_forward_step(step, n_p, commit=commit)
        torch.cuda.synchronize()
        res, meta = eng.res.cpu().tolist(), eng.meta.cpu().tolist()
        n_emit = res[_cabi.R_N_EMIT]
        hits = res[_cabi.R_HITS:_cabi.R_HITS + n_emit]
        q_len, lg = meta[_cabi.M_Q_LEN], meta[_cabi.M_N_GUESS_TOK]
        guess = eng.ids[q_len - lg:q_len].tolist() if lg else []
        slots = decided_slots(n_emit, hits, eng.WCAP, eng.GS, sampling is not None, res[_cabi.R_MAX_HIT_IDX], guess)
        base = res[_cabi.R_N_OUT] - n_emit - n_p
        for j, s in enumerate(slots):
            assert torch.equal(_bits(big[base + j]), _bits(eng.logits[s])), f"step {step} token {j} slot {s}"
            assert not tag or int(big[base + j, -1]) == s
        assert bool(big[base + n_emit:].isnan().all()), f"step {step}: a row past the step's tokens was written"
        uniforms = None
        if sampling is not None:
            dbg = eng.debug_uniforms.cpu().numpy()
            uniforms = dbg[1:1 + int(dbg[0])].tolist()
        steps.append(dict(hits=hits, max_hit=res[_cabi.R_MAX_HIT], guess=guess, slots=slots, uniforms=uniforms,
                          rows=big[base:base + n_emit].clone(), phase=meta[_cabi.M_PHASE]))
        if res[_cabi.R_DONE]:
            break
    before = big.clone()
    eng.run_forward_step(len(steps), n_p, commit=commit)         # a step on the finished state
    torch.cuda.synchronize()
    assert torch.equal(_bits(big), _bits(before)), "a step on the finished state wrote rows"
    return steps


# Low temperatures keep the sampled text close to the periodic one, so candidates keep being accepted; NEW_SAMPLING
# tokens give every sampling case several multi-token accepts (MIN_MULTI_SAMPLING).
SAMPLINGS = {"T": dict(temperature=0.5), "topk": dict(temperature=0.5, top_k=20), "topp": dict(temperature=0.5, top_p=0.8),
             "minp": dict(temperature=0.5, min_p=0.05), "eta": dict(temperature=0.5, eta=0.02)}
NEW_SAMPLING, MIN_MULTI_SAMPLING = 192, 3
PROCESSORS = dict(penalty=1.3, ngram_size=3, min_length=P + 8, eos_token_id=[5])


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("shape", ["d128", "d64"])
@pytest.mark.parametrize("mode", ["greedy", "greedy_proc"] + sorted(SAMPLINGS))
def test_captured_rows_are_the_deciding_slots(mode, shape, dtype):
    model = periodic_model(PERIODIC if shape == "d128" else PERIODIC_D64, dtype)
    sampling = SAMPLINGS.get(mode)
    new = NEW if sampling is None else NEW_SAMPLING
    eng = _engine(model, P + new, use_cuda_graph=False)
    assert eng.D == (128 if shape == "d128" else 64)
    prompt = _prompt()
    steps = lockstep(eng, prompt, new, sampling=sampling, processors=PROCESSORS if mode == "greedy_proc" else None,
                     tag=True)
    multi = sum(s["max_hit"] >= 2 for s in steps)
    print(f"{mode} {shape} {dtype}: {len(steps)} steps, {multi} with max_hit >= 2")
    assert multi >= (MIN_MULTI if sampling is None else MIN_MULTI_SAMPLING)
    eng.close()


@pytest.mark.parametrize("mode", ["greedy", "T", "minp"])
def test_captured_rows_qwen3(mode):
    from test_gpu_qwen3 import build_qwen3
    model = build_qwen3()
    eng = _engine(model, P + 48, W=15, N=5, G=15, use_cuda_graph=False)
    steps = lockstep(eng, _prompt(vocab=151936), 48, sampling=SAMPLINGS.get(mode), tag=True)
    assert sum(len(s["slots"]) for s in steps) >= 48
    eng.close()


def test_greedy_decisions_replay_from_captured_rows():
    """argmax of every captured row is the token emitted (lowest index on ties); with the processors, argmax of HF's
    scores built from the rows is."""
    from lookaheaddecoding_b200.decoding import generate_output
    from transformers.generation.logits_process import (LogitsProcessorList, MinNewTokensLengthLogitsProcessor,
                                                        NoRepeatNGramLogitsProcessor, RepetitionPenaltyLogitsProcessor)
    model = periodic_model()
    eng = _engine(model, P + NEW)
    prompt = _prompt()
    out = eng.generate(prompt, NEW, rng=random.Random(0), capture_logits=True)
    rows = eng.last_logits
    assert rows.shape == (NEW, eng.V) and rows.dtype == eng.dt
    assert rows.float().argmax(dim=-1).tolist() == out[P:]
    assert sum(r.max_hit >= 2 for r in eng.last_records) >= MIN_MULTI
    procs = LogitsProcessorList([RepetitionPenaltyLogitsProcessor(1.3), NoRepeatNGramLogitsProcessor(3),
                                 MinNewTokensLengthLogitsProcessor(P, 8, [5], device="cuda")])
    out = eng.generate(prompt, NEW, rng=random.Random(0), capture_logits=True,
                       processors=dict(penalty=1.3, prompt_ignore_length=0, ngram_size=3, min_length=P + 8,
                                       eos_token_id=[5]))
    seq = torch.tensor([out], device="cuda")
    o = generate_output(seq, P, eng.last_logits, procs, True, True)
    assert len(o.scores) == len(o.logits) == len(out) - P
    assert [int(s.argmax()) for s in o.scores] == out[P:]
    eng.close()


@pytest.mark.parametrize("mode", ["T", "topk", "topp"])
def test_sampling_decisions_replay_from_captured_rows(mode):
    """The restatement of the verification, given the kernel's uniforms and only the captured rows (every other guess
    row NaN), reproduces every step's hits: the chain never needs a row that was not captured."""
    s = SAMPLINGS[mode]
    T, top_k, top_p = s.get("temperature", 1.0), s.get("top_k", 0), s.get("top_p", 1.0)
    model = periodic_model()
    eng = _engine(model, P + NEW_SAMPLING, use_cuda_graph=False)
    steps = lockstep(eng, _prompt(), NEW_SAMPLING, sampling=s)
    GS, WCAP = eng.GS, eng.WCAP
    checked = accepted = 0
    for k, st in enumerate(steps):
        rows = st["rows"].float().cpu().numpy()
        guess = st["guess"] if st["phase"] == 2 and st["guess"] else None
        guess_rows = None
        if guess:
            guess_rows = np.full((len(guess), eng.V), np.nan, dtype=np.float32)
            for j, slot in enumerate(st["slots"][1:], start=1):
                guess_rows[slot - 1 - WCAP] = rows[j]
        with np.errstate(invalid="ignore"):      # a full accept warps the (NaN) row after the last token, unused
            want = SD.verify_given_uniforms(rows[0], guess_rows, guess, GS, T, st["uniforms"], top_k, top_p)
        if any(c[0] == "accept" and abs(c[1] - c[2]) < 1e-6 for c in want["checks"]):
            continue
        assert want["used"] == len(st["uniforms"]) and want["n_hits"] == len(st["hits"]), f"step {k}"
        draws = [c for c in want["checks"] if c[0] == "draw"]
        for j, h in enumerate(want["hits"] or [None]):
            if h is None:
                _, u, probs = draws[-1][:3]
                assert np.isfinite(probs).all() and SD.draw_is_consistent(u, probs, st["hits"][j]), f"step {k} draw"
            else:
                assert st["hits"][j] == h, f"step {k} token {j}"
        checked += 1
        accepted += st["max_hit"] >= 2
    print(f"{mode}: {checked} steps replayed, {accepted} with max_hit >= 2")
    assert checked >= len(steps) - 3 and accepted >= MIN_MULTI_SAMPLING
    eng.close()


def test_modes_agree_and_capture_changes_nothing_else():
    model = periodic_model()
    prompt = _prompt()
    runs = {}
    for name, kw in {"graph": {}, "eager": dict(use_cuda_graph=False), "sync": dict(pipeline_host=False),
                     "eager_sync": dict(use_cuda_graph=False, pipeline_host=False)}.items():
        eng = _engine(model, P + NEW, **kw)
        for sampling in (None, dict(temperature=0.8, top_k=20, seed=3)):
            res = {}
            for cap in (False, True, False):
                l0 = eng.launches
                out = eng.generate(prompt, NEW, rng=random.Random(0), sampling=sampling, capture_logits=cap)
                recs = [(r.n_emit, r.max_hit, tuple(r.hits), r.n_guess, r.kv_len, r.done) for r in eng.last_records]
                res.setdefault(cap, []).append((out, recs, eng.launches - l0, eng.last_steps,
                                                eng.last_logits.clone() if cap else None))
                assert (eng.last_logits is not None) == cap
            off, on, off2 = res[False][0], res[True][0], res[False][1]
            assert off[:3] == off2[:3] and on[:2] == off[:2]
            extra = on[2] - off[2]                                # one capture launch per step, the surplus one included
            assert extra in (on[3], on[3] + 1)
            if not kw.get("pipeline_host", True):
                assert extra == on[3]
            assert on[4].shape == (len(on[0]) - P, eng.V)
            runs[(name, sampling is None)] = on
        eng.close()
    for greedy in (True, False):
        ref = runs[("graph", greedy)]
        for name in ("eager", "sync", "eager_sync"):
            got = runs[(name, greedy)]
            assert got[0] == ref[0] and torch.equal(_bits(got[4]), _bits(ref[4])), (name, greedy)


def test_surplus_pipelined_step_writes_nothing():
    """A generation that ends early in the pipelined loop queues one step on the finished state; rows behind the last
    emitted token stay NaN."""
    model = periodic_model()
    prompt = _prompt()
    eng = _engine(model, P + NEW)
    ref = eng.generate(prompt, NEW, rng=random.Random(0), capture_logits=True)
    # end where a multi-token step crosses max_new_tokens: the loop did not know it was the last step
    total, new = 0, None
    for r in eng.last_records:
        if total > 4 and r.n_emit >= 2:
            new = total + 1
            break
        total += r.n_emit
    assert new is not None
    big = torch.full((new + eng.GS + 2, eng.V), float("nan"), dtype=eng.dt, device="cuda")
    eng.capture_buf = big[:new + eng.GS]
    l0 = eng.launches
    out = eng.generate(prompt, new, rng=random.Random(0), capture_logits=True)
    emitted = sum(r.n_emit for r in eng.last_records)
    assert out == ref[:P + new] and emitted > new
    assert not bool(big[:emitted].isnan().any()) and bool(big[emitted:].isnan().all())
    sync = _engine(model, P + NEW, pipeline_host=False)
    l1 = sync.launches
    sync.generate(prompt, new, rng=random.Random(0), capture_logits=True)
    print(f"pipelined launches {eng.launches - l0}, synchronous {sync.launches - l1}")
    assert torch.equal(_bits(sync.last_logits), _bits(eng.last_logits))
    eng.close()
    sync.close()


def test_edges_eos_inside_accept_and_short_budgets():
    model = periodic_model()
    prompt = _prompt()
    eng = _engine(model, P + NEW)
    ref = eng.generate(prompt, NEW, rng=random.Random(0), capture_logits=True)
    ref_rows = eng.last_logits.clone()
    gen = ref[P:]
    # EOS = the middle token of a multi-token accept that has not been emitted before
    pos = 0
    eos = None
    for r in eng.last_records:
        if r.max_hit >= 2 and r.hits[1] not in gen[:pos + 1] and r.hits[1] not in prompt:
            eos, cut = r.hits[1], pos + 2
            break
        pos += r.n_emit
    assert eos is not None
    out = eng.generate(prompt, NEW, eos_token_ids=[eos], rng=random.Random(0), capture_logits=True)
    assert out == ref[:P + cut] and out[-1] == eos
    assert eng.last_logits.shape[0] == cut and torch.equal(_bits(eng.last_logits), _bits(ref_rows[:cut]))
    out = eng.generate(prompt, 1, rng=random.Random(0), capture_logits=True)
    assert len(out) == P + 1 and eng.last_logits.shape[0] == 1
    assert torch.equal(_bits(eng.last_logits[0]), _bits(ref_rows[0]))
    total = 0
    eng.generate(prompt, NEW, rng=random.Random(0))
    for r in eng.last_records:
        if total > 3 and r.n_emit >= 3:
            break
        total += r.n_emit
    mid = total + 1                                               # ends one token into a multi-token accept
    out = eng.generate(prompt, mid, rng=random.Random(0), capture_logits=True)
    assert out == ref[:P + mid] and eng.last_logits.shape[0] == mid
    assert torch.equal(_bits(eng.last_logits), _bits(ref_rows[:mid]))
    eng.close()


def test_argument_errors_write_nothing():
    from lookaheaddecoding_b200 import _cabi
    model = periodic_model()
    eng = _engine(model, P + 16, use_cuda_graph=False)
    prompt = _prompt()
    eng.generate(prompt, 8, rng=random.Random(0), capture_logits=True)
    lib = eng.lib
    buf = torch.full((8, eng.V), float("nan"), dtype=eng.dt, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    p = lambda t: t.data_ptr()
    good = [eng._ctx, s, p(eng.logits), eng.V, eng.V, p(eng.ids), p(eng.lm_rows), p(eng.meta), p(eng.res), 0, p(buf),
            eng.V, 8]
    bad = {2: None, 3: eng.V - 1, 4: 0, 5: None, 6: None, 7: None, 8: None, 9: 2, 10: None, 11: eng.V - 1, 12: 0}
    for i, v in bad.items():
        args = list(good)
        args[i] = v
        assert lib.lade_capture_rows(*args) == _cabi.LADE_EINVAL, i
    args = list(good)
    args[10] = p(buf) + 1                                          # not aligned to its element
    assert lib.lade_capture_rows(*args) == _cabi.LADE_EINVAL
    assert lib.lade_capture_rows(None, *good[1:]) == _cabi.LADE_EINVAL
    torch.cuda.synchronize()
    assert bool(buf.isnan().all())
    eng.close()


def test_plugin_returns_hf_output_and_logits_agree_with_hf():
    import lade
    from transformers.generation.utils import GenerateDecoderOnlyOutput
    model = periodic_model()
    prompt = _prompt()
    ids = torch.tensor([prompt], device="cuda")
    kw = dict(attention_mask=torch.ones_like(ids), max_new_tokens=64, return_dict_in_generate=True, output_logits=True,
              output_scores=True)
    hf = model.generate(ids, do_sample=False, **kw)
    x = hf.sequences[:, :-1]
    tf = model(x).logits[0, P - 1:].float()                        # HF teacher-forced, for its self-inconsistency
    lade.augment_all()
    import os
    os.environ["USE_LADE"] = "1"
    try:
        lade.config_lade(LEVEL=N, WINDOW_SIZE=W, GUESS_SET_SIZE=G, DEBUG=0, POOL_FROM_PROMPT=True)
        out = model.generate(ids, do_sample=False, **kw)
        samp = model.generate(ids, do_sample=True, temperature=0.8, top_k=20, **kw)
        plain = model.generate(ids, do_sample=False, attention_mask=torch.ones_like(ids), max_new_tokens=8,
                               return_dict_in_generate=True)
    finally:
        os.environ["USE_LADE"] = "0"
        lade.restore_generate()
    for o in (out, samp):
        assert isinstance(o, GenerateDecoderOnlyOutput) and type(o) is type(hf)
        assert o.attentions is None and o.hidden_states is None and o.past_key_values is None
        assert len(o.logits) == len(o.scores) == o.sequences.shape[1] - P == 64
        for a, b in zip(o.logits + o.scores, hf.logits + hf.scores):
            assert a.shape == b.shape and a.dtype == b.dtype == torch.float32 and a.device == b.device
        ts = model.compute_transition_scores(o.sequences, o.scores, normalize_logits=True)
        assert ts.shape == (1, 64) and bool(torch.isfinite(ts).all())
    assert plain.scores is None and plain.logits is None and plain.sequences.shape == (1, P + 8)
    assert all(torch.equal(a, b) for a, b in zip(out.logits, out.scores))        # no processor: scores are the logits
    got, want = out.sequences[0, P:].tolist(), hf.sequences[0, P:].tolist()
    agree = next((j for j in range(64) if got[j] != want[j]), 64)
    hf_logits = torch.cat(hf.logits)
    top = torch.topk(hf_logits, 16, dim=-1).indices
    ulp = torch.pow(2.0, torch.floor(torch.log2(hf_logits.amax(dim=-1).abs())) - 7)[:, None]
    self_gap = float(((tf.gather(1, top) - hf_logits.gather(1, top)).abs() / ulp).max())
    mine = torch.cat(out.logits)
    diff = ((mine.gather(1, top) - hf_logits.gather(1, top)).abs() / ulp)[:agree]
    tol = max(3.0, self_gap)
    print(f"ids agree on {agree} of 64; worst top-16 logit gap {float(diff.max()):.2f} ulps (tol {tol:.2f})")
    assert agree >= 16 and float(diff.max()) <= tol


def test_refusals():
    from lookaheaddecoding_b200 import LadeError
    from lookaheaddecoding_b200.decoding import CONFIG_MAP, jacobi_greedy_search_multilevel
    model = periodic_model()
    eng = _engine(model, P + 16)
    eng.DW = 2
    prompt = _prompt()
    with pytest.raises(LadeError, match="DIST_WORKERS"):
        eng.begin(prompt, P + 8, (), prompt[:eng.WCAP], capture_logits=True)
    eng.DW = 1
    eng.close()
    ids = torch.tensor([_prompt()], device="cuda")
    for kw in (dict(output_attentions=True), dict(output_hidden_states=True)):
        with pytest.raises(LadeError, match="not supported"):
            jacobi_greedy_search_multilevel(model, ids, max_length=P + 8, return_dict_in_generate=True, **kw)
    CONFIG_MAP["DIST_WORKERS"] = 2
    try:
        with pytest.raises(LadeError, match="DIST_WORKERS"):
            jacobi_greedy_search_multilevel(model, ids, max_length=P + 8, return_dict_in_generate=True,
                                            output_logits=True)
    finally:
        CONFIG_MAP.pop("DIST_WORKERS")
