"""CPU: the host side of per-token logits capture.

* the first-matching-candidate rule (engine.first_matching_candidate, the rule lade_capture_rows follows on the
  sampling path) picks the candidate the sampling verification accepted: on every verification step of the oracle
  sampling runs pinned to the unmodified reference (tests/golden/sample_traces.json.gz), and at every position of
  crafted guess sets where one draft is carried by several n-grams and rejected;
* generate_output builds HF's logits / scores from (sequences, rows) with HF's own processor and warper objects, equal
  to running them position by position;
* output_logits reaches the decode loops through sample_entry_proxy; the refusals raise before any engine exists.
"""
import gzip
import json
import os
import random
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from lookaheaddecoding_b200.engine import decided_slots, first_matching_candidate
from oracle import lookahead as LA
from oracle import llama_ref as LR
from oracle import sampling_device as SD

GOLD = os.path.join(os.path.dirname(__file__), "golden")
with gzip.open(os.path.join(GOLD, "sample_traces.json.gz"), "rt") as f:
    TRACES = json.load(f)


def _warper(temperature, top_k, top_p):
    from test_oracle_sampling import make_warper
    return make_warper(temperature, top_k, top_p)


@pytest.mark.parametrize("name", sorted(TRACES))
def test_rule_picks_the_oracle_winner_on_golden_runs(name):
    """The oracle records the winner of the last accepted position (max_hit_idx).  That position is max_hit when the
    hits end on an accepted draft, else max_hit - 1 (the last hit was drawn from the residual); every earlier position
    has a carrying candidate too."""
    c = TRACES[name]
    w = LR.init_weights(c["model"], seed=c["weight_seed"], dtype=getattr(torch, c["dtype"]))
    om = LR.OracleLlama(c["model"], w)
    rng = random.Random(c["seed"])
    torch.manual_seed(c["seed"] + 1000)
    trace = []
    ids, _ = LA.sample_lookahead(c["prompt"], c["max_new"], c["W"], c["N"], c["G"], om,
                                 warper=_warper(c["temperature"], c["top_k"], c["top_p"]),
                                 pool_from_prompt=c["pool_from_prompt"], eos_token_id=c["eos_token_id"], rng=rng,
                                 trace=trace)
    assert ids == c["output_ids"]                       # the run is the pinned one
    GS = c["N"] - 1
    checked = 0
    for t in trace:
        if not t["guess_tokens"] or t["max_hit"] == 0:
            continue
        hits, mh = t["hits"], t["max_hit"]
        last = mh if first_matching_candidate(t["guess_tokens"], GS, hits, mh) >= 0 else mh - 1
        assert all(first_matching_candidate(t["guess_tokens"], GS, hits, i) >= 0 for i in range(last + 1))
        assert first_matching_candidate(t["guess_tokens"], GS, hits, last) == t["max_hit_idx"]
        checked += 1
    print(f"{name}: {checked} accepting verification steps")


def _winners_from_checks(want, guess, gs):
    """Per accepted position, the candidate that accepted: the restatement tests the alive candidates in order, one
    uniform each, and stops at the accepting one."""
    alive = list(range(len(guess) // gs))
    winners, k, checks = [], 0, want["checks"]
    for i in range(gs):
        n = 0
        while k < len(checks) and checks[k][0] == "accept":
            n += 1
            _, u, p, draft = checks[k]
            k += 1
            if u <= p:
                break
        else:
            return winners                               # a draw ended the chain
        e = alive[n - 1]
        winners.append(e)
        alive = [g for g in alive if guess[g * gs + i] == guess[e * gs + i]]
    return winners


def test_rule_on_crafted_guess_sets():
    """Random guess sets over a 5-token vocabulary (so drafts repeat across n-grams and get rejected for some of them),
    random rows and uniforms; the hand-made case rejects a draft carried by three n-grams at position 1."""
    rs = np.random.RandomState(0)
    gs, V = 3, 5
    n_rejected_shared = 0
    for trial in range(400):
        n_ng = rs.randint(1, 7)
        guess = rs.randint(0, V, size=n_ng * gs).tolist()
        out_row = rs.randn(V).astype(np.float32) * 2
        rows = rs.randn(n_ng * gs, V).astype(np.float32) * 2
        uniforms = rs.uniform(1e-6, 1.0, size=n_ng * gs + 2).tolist()
        want = SD.verify_given_uniforms(out_row, rows, guess, gs, 1.0, uniforms)
        winners = _winners_from_checks(want, guess, gs)
        hits = [-1 if h is None else h for h in want["hits"]]
        assert len(winners) == sum(h >= 0 for h in hits)
        for i, e in enumerate(winners):
            assert first_matching_candidate(guess, gs, hits, i) == e, (trial, i)
        n_rejected_shared += sum(1 for c in want["checks"] if c[0] == "accept" and c[2] == 0.0)
        slots = decided_slots(want["n_hits"], hits, 4, gs, True, 0, guess)
        assert slots[1:] == [1 + 4 + winners[j - 1] * gs + j - 1 for j in range(1, want["n_hits"])]
    assert n_rejected_shared > 50
    # 0 accepted at position 0 by n-gram 0; at position 1 draft 1 is rejected on n-gram 0, so n-gram 1, which carries
    # it too, is tested with p = 0; n-gram 2 carries 2 and accepts, and the rule picks it
    guess = [0, 1, 3, 0, 1, 4, 0, 2, 4, 0, 1, 2]
    rows = np.zeros((12, 5), dtype=np.float32)
    out_row = np.array([8, 0, 0, 0, 0], dtype=np.float32)
    rows[0] = [0, 3, 3, 0, 0]
    uniforms = [0.5, 0.99, 0.01, 0.02, 0.5, 0.5]
    want = SD.verify_given_uniforms(out_row, rows, guess, 3, 1.0, uniforms)
    assert want["checks"][1][2] < 0.99 and want["checks"][2][2] == 0.0 and want["hits"][:2] == [0, 2]
    assert _winners_from_checks(want, guess, 3)[:2] == [0, 2]
    assert [first_matching_candidate(guess, 3, want["hits"], i) for i in range(2)] == [0, 2]


def test_greedy_slots_follow_max_hit_idx():
    assert decided_slots(3, [7, 8, 9], 10, 4, False, max_hit_idx=2) == [0, 1 + 10 + 8, 1 + 10 + 9]
    assert decided_slots(1, [7], 10, 4, True, guess_tokens=[1, 2, 3, 4]) == [0]
    assert decided_slots(0, [], 10, 4, False) == []


def _hf_lists():
    from transformers.generation.logits_process import (LogitsProcessorList, MinNewTokensLengthLogitsProcessor,
                                                        MinPLogitsWarper, NoRepeatNGramLogitsProcessor,
                                                        RepetitionPenaltyLogitsProcessor, TemperatureLogitsWarper,
                                                        TopKLogitsWarper, TopPLogitsWarper)
    return {"none": LogitsProcessorList(),
            "processors": LogitsProcessorList([RepetitionPenaltyLogitsProcessor(1.3), NoRepeatNGramLogitsProcessor(2),
                                               MinNewTokensLengthLogitsProcessor(6, 3, [4])]),
            "warpers": LogitsProcessorList([TemperatureLogitsWarper(0.7), TopKLogitsWarper(20), TopPLogitsWarper(0.9),
                                            MinPLogitsWarper(0.05)])}


@pytest.mark.parametrize("kind", ["none", "processors", "warpers"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_generate_output_equals_hf_objects_position_by_position(kind, dtype):
    from transformers.generation.utils import GenerateDecoderOnlyOutput
    from lookaheaddecoding_b200.decoding import generate_output
    procs = _hf_lists()[kind]
    g = torch.Generator().manual_seed(3)
    P, new, V = 6, 9, 64
    seq = torch.randint(0, 8, (1, P + new), generator=g)               # small id range: repeats, n-gram bans
    rows = (torch.randn(new, V, generator=g) * 3).to(dtype)
    o = generate_output(seq, P, rows, procs, True, True)
    assert isinstance(o, GenerateDecoderOnlyOutput) and o.attentions is None and o.hidden_states is None
    assert len(o.logits) == len(o.scores) == new
    for j in range(new):
        want_logits = rows[j:j + 1].to(torch.float32)
        want_scores = procs(seq[:, :P + j], want_logits.clone())
        assert o.logits[j].dtype == torch.float32 and torch.equal(o.logits[j], want_logits)
        assert torch.equal(o.scores[j], want_scores), j
    if kind != "none":
        assert any(not torch.equal(a, b) for a, b in zip(o.logits, o.scores))
    only = generate_output(seq, P, rows, procs, False, True)
    assert only.logits is None and len(only.scores) == new
    none = generate_output(seq, P, None, procs, False, False)
    assert none.scores is None and none.logits is None and none.sequences is seq


def _fake_config(**kw):
    base = dict(do_sample=False, _eos_token_tensor=None, eos_token_id=None, _pad_token_tensor=None,
                output_attentions=False, output_hidden_states=False, output_scores=False, output_logits=False,
                return_dict_in_generate=False)
    base.update(kw)
    return SimpleNamespace(**base)


@pytest.mark.parametrize("do_sample", [False, True])
def test_output_logits_reaches_the_decode_loops(monkeypatch, do_sample):
    from lookaheaddecoding_b200 import decoding, sampling
    seen = {}

    def spy(self, input_ids, **kw):
        seen.update(kw)
        return "ok"
    monkeypatch.setenv("USE_LADE", "1")
    monkeypatch.setattr(decoding, "jacobi_greedy_search_multilevel", spy)
    monkeypatch.setattr(sampling, "jacobi_sample_multilevel", spy)
    cfg = _fake_config(do_sample=do_sample, output_logits=True, output_scores=True, return_dict_in_generate=True)
    assert decoding.sample_entry_proxy(None, torch.ones(1, 4, dtype=torch.long), None, None, cfg) == "ok"
    assert seen["output_logits"] is True and seen["output_scores"] is True and seen["return_dict_in_generate"] is True
    seen.clear()
    decoding.sample_entry_proxy(None, torch.ones(1, 4, dtype=torch.long), None, None, _fake_config(do_sample=do_sample))
    assert seen["output_logits"] is False


def test_refusals_before_any_engine():
    from lookaheaddecoding_b200 import LadeError
    from lookaheaddecoding_b200.decoding import CONFIG_MAP, jacobi_greedy_search_multilevel, wants_logits
    from lookaheaddecoding_b200.sampling import jacobi_sample_multilevel
    ids = torch.ones(1, 4, dtype=torch.long)
    for fn in (jacobi_greedy_search_multilevel, jacobi_sample_multilevel):
        for kw in (dict(output_attentions=True), dict(output_hidden_states=True)):
            with pytest.raises(LadeError, match="not supported"):
                fn(None, ids, max_length=8, return_dict_in_generate=True, **kw)
    CONFIG_MAP["DIST_WORKERS"] = 2
    try:
        for kw in (dict(output_logits=True), dict(output_scores=True)):
            with pytest.raises(LadeError, match="DIST_WORKERS"):
                jacobi_greedy_search_multilevel(None, ids, max_length=8, return_dict_in_generate=True, **kw)
    finally:
        CONFIG_MAP.pop("DIST_WORKERS")
    assert not wants_logits(False, True, True) and not wants_logits(True, False, False)
    assert wants_logits(True, True, False) and wants_logits(True, False, True)
