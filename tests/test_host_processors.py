"""CPU-only: HF greedy logits processors -> the engine's `processors` dict -> the device LadeProcessors record, and the
combinations that still raise (unsupported processors, sampling, lookahead parallelism)."""
import numpy as np
import pytest
import torch
from transformers.generation.logits_process import (LogitsProcessorList, MinLengthLogitsProcessor,
                                                    MinNewTokensLengthLogitsProcessor, NoBadWordsLogitsProcessor,
                                                    NoRepeatNGramLogitsProcessor, RepetitionPenaltyLogitsProcessor,
                                                    SuppressTokensLogitsProcessor)

from lookaheaddecoding_b200 import _cabi
from lookaheaddecoding_b200._cabi import LadeError
from lookaheaddecoding_b200.decoding import CONFIG_MAP, jacobi_greedy_search_multilevel, processors_from_hf
from lookaheaddecoding_b200.engine import LookaheadEngine, processors_record


def _f32_bits(x):
    return int(np.float32(x).view(np.uint32))


def _record(procs):
    r = processors_record(processors_from_hf(LogitsProcessorList(procs)))
    return dict(flags=r.flags, penalty_bits=r.penalty_bits, pil=r.prompt_ignore_length, n=r.ngram_size,
                eos_bound=r.eos_bound, eos=list(r.eos_token_id)[:r.n_eos])


def test_each_processor_translates():
    assert processors_from_hf(None) is None and processors_from_hf(LogitsProcessorList()) is None
    assert _record([RepetitionPenaltyLogitsProcessor(1.3)]) == dict(
        flags=_cabi.PROC_REPETITION_PENALTY, penalty_bits=_f32_bits(1.3), pil=0, n=0, eos_bound=0, eos=[])
    assert _record([RepetitionPenaltyLogitsProcessor(0.7, prompt_ignore_length=12)])["pil"] == 12
    assert _record([RepetitionPenaltyLogitsProcessor(0.7)])["penalty_bits"] == _f32_bits(0.7)
    for n in (1, 2, 3, 5):
        assert _record([NoRepeatNGramLogitsProcessor(n)]) == dict(
            flags=_cabi.PROC_NO_REPEAT_NGRAM, penalty_bits=0, pil=0, n=n, eos_bound=0, eos=[])
    assert _record([MinLengthLogitsProcessor(50, 2)]) == dict(
        flags=_cabi.PROC_MIN_LENGTH, penalty_bits=0, pil=0, n=0, eos_bound=50, eos=[2])
    assert _record([MinNewTokensLengthLogitsProcessor(17, 40, [2, 9, 4])]) == dict(
        flags=_cabi.PROC_MIN_LENGTH, penalty_bits=0, pil=0, n=0, eos_bound=57, eos=[2, 4, 9])


def test_combinations_translate_in_any_order():
    procs = [MinNewTokensLengthLogitsProcessor(10, 40, torch.tensor([3, 2])), NoRepeatNGramLogitsProcessor(3),
             RepetitionPenaltyLogitsProcessor(1.2, 4), MinLengthLogitsProcessor(60, [2, 3])]
    want = dict(flags=7, penalty_bits=_f32_bits(1.2), pil=4, n=3, eos_bound=60, eos=[2, 3])
    assert _record(procs) == want
    assert _record(procs[::-1]) == want
    # the eos bound is the larger of the two processors' bounds
    assert _record([MinLengthLogitsProcessor(30, 2), MinNewTokensLengthLogitsProcessor(10, 40, 2)])["eos_bound"] == 50


def test_unsupported_processors_are_named():
    for p in (NoBadWordsLogitsProcessor([[5]], eos_token_id=2), SuppressTokensLogitsProcessor([1, 2])):
        with pytest.raises(LadeError, match=type(p).__name__):
            processors_from_hf(LogitsProcessorList([RepetitionPenaltyLogitsProcessor(1.2), p]))
    with pytest.raises(LadeError, match="RepetitionPenaltyLogitsProcessor"):
        processors_from_hf([RepetitionPenaltyLogitsProcessor(1.2), RepetitionPenaltyLogitsProcessor(1.1)])
    with pytest.raises(LadeError, match="eos"):
        processors_from_hf([MinLengthLogitsProcessor(30, 2), MinNewTokensLengthLogitsProcessor(10, 40, 3)])


def test_record_limits():
    with pytest.raises(LadeError, match="no_repeat_ngram_size"):
        processors_record({"ngram_size": _cabi.PROC_MAX_NGRAM + 1})
    with pytest.raises(LadeError, match="eos"):
        processors_record({"min_length": 9, "eos_token_id": list(range(_cabi.PROC_MAX_EOS + 1))})
    with pytest.raises(LadeError, match="penalty"):
        processors_record({"penalty": 0.0})
    with pytest.raises(LadeError, match="unknown"):
        processors_record({"bad_words": [1]})
    assert processors_record({"min_length": 9}).flags == 0          # no eos id: nothing to suppress
    # the C-ABI rejects what the kernel cannot take, before any CUDA call
    lib = _cabi.load()
    r = _cabi.LadeProcessors()
    r.flags, r.ngram_size = _cabi.PROC_NO_REPEAT_NGRAM, 0
    assert lib.lade_processors_upload(None, r, None) == _cabi.LADE_EINVAL
    assert lib.lade_processors_upload(None, r, 16) == _cabi.LADE_EINVAL
    r.ngram_size, r.n_eos = 3, 9
    assert lib.lade_processors_upload(None, r, 16) == _cabi.LADE_EINVAL
    r.n_eos, r.flags = 0, 8
    assert lib.lade_processors_upload(None, r, 16) == _cabi.LADE_EINVAL
    assert lib.lade_argmax_processed(None, None, 16, 1, 32000, 32000, 16, 16) == _cabi.LADE_EINVAL


def _host_engine(dist_workers=1):
    eng = LookaheadEngine.__new__(LookaheadEngine)      # no model, no GPU: generate() raises before touching either
    eng.max_total_len, eng.DW = 4096, dist_workers
    return eng


def test_sampling_and_lookahead_parallelism_with_processors_raise():
    with pytest.raises(LadeError, match="greedy path only"):
        _host_engine().generate([1, 2, 3], 8, sampling={"temperature": 0.7}, processors={"penalty": 1.2})
    with pytest.raises(LadeError, match="lookahead parallelism"):
        _host_engine(2).generate([1, 2, 3], 8, processors={"ngram_size": 3})
    ids = torch.tensor([[1, 2, 3]])
    old = dict(CONFIG_MAP)
    try:
        CONFIG_MAP["DIST_WORKERS"] = 2
        with pytest.raises(LadeError, match="lookahead parallelism"):
            jacobi_greedy_search_multilevel(None, ids, logits_processor=LogitsProcessorList(
                [RepetitionPenaltyLogitsProcessor(1.2)]), max_length=8)
    finally:
        CONFIG_MAP.clear()
        CONFIG_MAP.update(old)
    from lookaheaddecoding_b200.sampling import jacobi_sample_multilevel
    with pytest.raises(LadeError):
        jacobi_sample_multilevel(None, ids, logits_processor=LogitsProcessorList([RepetitionPenaltyLogitsProcessor(1.2)]),
                                 max_length=8)
