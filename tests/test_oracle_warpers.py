"""CPU-only: the MinP / Epsilon / Eta cuts of the sampling path.

* ``warper_restatement.softmax_T`` (tests/) with min_p, epsilon and eta, alone and after temperature / top-k / top-p, equals
  HF's own warper chain run in float64 on tie-free rows at vocab 32000 and 128256;
* ``device_warper_params`` on the lists ``GenerationMixin._get_logits_processor`` builds, and None for the lists the
  device kernel does not implement;
* ``_check_warpers`` / ``split_warpers`` admit the three new warpers and nothing else;
* the C-ABI range checks of ``lade_sample_verify_warped`` (they precede any CUDA call);
* the engine's ``sampling=`` range checks."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import sampling_device as SD
import warper_restatement as WR


def _tie_free_row(seed, vocab, sigma, T):
    """A row whose fp32 scores row / T are pairwise distinct (HF's sort order inside a tie is undefined)."""
    rng = np.random.default_rng(seed)
    pool = rng.normal(0, sigma, 2 * vocab).astype(np.float32)
    _, first = np.unique(pool / np.float32(T), return_index=True)        # one value per distinct score
    row = rng.permutation(pool[first])[:vocab]
    assert row.size == vocab and np.unique(row / np.float32(T)).size == vocab
    return row.astype(np.float64)


def _hf_probs(row, T, top_k, top_p, min_p, epsilon, eta):
    """HF's chain: TemperatureLogitsWarper in fp32 (the dtype of the scores generate() warps), then TopK -> TopP ->
    MinP -> Epsilon -> Eta on float64 scores."""
    from transformers.generation.logits_process import (EpsilonLogitsWarper, EtaLogitsWarper, MinPLogitsWarper,
                                                        TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper)
    ids = torch.zeros(1, 1, dtype=torch.long)
    s = TemperatureLogitsWarper(T)(ids, torch.tensor(row, dtype=torch.float32)[None]).double()
    chain = []
    if top_k:
        chain.append(TopKLogitsWarper(top_k))
    if top_p < 1.0:
        chain.append(TopPLogitsWarper(top_p))
    if min_p:
        chain.append(MinPLogitsWarper(min_p))
    if epsilon:
        chain.append(EpsilonLogitsWarper(epsilon))
    if eta:
        chain.append(EtaLogitsWarper(eta))
    for w in chain:
        s = w(ids, s)
    return torch.softmax(s, dim=-1)[0].numpy()


CUTS = [dict(min_p=m) for m in (1e-3, 0.05, 0.1, 0.5, 1.0)] + \
       [dict(epsilon=e) for e in (1e-4, 3e-4, 0.9)] + \
       [dict(eta=e) for e in (1e-4, 2e-3, 0.5)] + \
       [dict(min_p=0.05, epsilon=3e-4), dict(min_p=1e-3, eta=2e-3), dict(epsilon=1e-4, eta=1e-4),
        dict(min_p=0.05, epsilon=1e-4, eta=2e-3)]
BASE = [(1.0, 0, 1.0), (0.7, 0, 1.0), (1.0, 400, 1.0), (1.0, 0, 0.9), (2.0, 1000, 0.95)]


@pytest.mark.parametrize("vocab,sigma", [(32000, 1.0), (128256, 2.5)])
@pytest.mark.parametrize("cut", CUTS, ids=lambda c: ",".join(f"{k}={v}" for k, v in c.items()))
def test_softmax_T_cuts_equal_hf_warpers(vocab, sigma, cut):
    effective = 0
    # the float64 top-p restatement walks the distinct scores one by one: at 128256 the top-p rows are left to 32000
    for i, (T, top_k, top_p) in enumerate(BASE if vocab <= 32000 else [b for b in BASE if b[2] == 1.0]):
        row = _tie_free_row(vocab + i, vocab, sigma, T)
        args = (cut.get("min_p", 0.0), cut.get("epsilon", 0.0), cut.get("eta", 0.0))
        want = _hf_probs(row, T, top_k, top_p, *args)
        got = WR.softmax_T(row, T, top_k, top_p, *args)
        assert np.array_equal(got > 0, want > 0), f"T={T} k={top_k} p={top_p}: kept sets differ " \
            f"({int((got > 0).sum())} vs {int((want > 0).sum())})"
        np.testing.assert_allclose(got, want, rtol=1e-10, atol=1e-300)
        base = WR.softmax_T(row, T, top_k, top_p)
        if cut in (dict(min_p=1.0), dict(epsilon=0.9)):
            assert (got > 0).sum() == 1                  # tie-free: only the maximum stays
        effective += int(1 < (got > 0).sum() < (base > 0).sum())
    if cut not in (dict(min_p=1.0), dict(epsilon=0.9)):
        assert effective >= 2, "the cut hardly ever left a proper subset"


def test_softmax_T_with_the_cuts_off_is_the_top_p_restatement():
    row = _tie_free_row(3, 4096, 1.0, 1.0)
    for args in [(1.0, 0, 1.0), (0.8, 50, 0.9)]:
        assert np.array_equal(SD.softmax_T(row, *args), WR.softmax_T(row, *args, 0.0, 0.0, 0.0))


def test_cuts_keep_a_tie_group_at_the_maximum_together():
    row = np.full(64, -3.0)
    row[[5, 9, 40]] = 2.0
    for kw in (dict(min_p=1.0), dict(epsilon=0.9), dict(eta=0.9 - 1e-9)):
        p = WR.softmax_T(row, 1.0, **kw)
        assert np.nonzero(p)[0].tolist() == [5, 9, 40], kw


# ---------------------------------------------------------------------------------------------- plugin
def _hf_list(**kw):
    from transformers import GenerationConfig
    from transformers.generation.utils import GenerationMixin

    class _Model(GenerationMixin):
        pass
    gc = GenerationConfig(do_sample=True, **kw)
    return _Model.__new__(_Model)._get_logits_processor(generation_config=gc, input_ids_seq_length=4,
                                                        encoder_input_ids=torch.zeros(1, 4, dtype=torch.long),
                                                        prefix_allowed_tokens_fn=None, logits_processor=None,
                                                        device="cpu")


@pytest.mark.parametrize("kw,want", [
    (dict(top_k=0, min_p=0.1), dict(min_p=0.1)),
    (dict(top_k=0, min_p=0.0), {}),
    (dict(temperature=0.7, top_k=50, top_p=0.9, min_p=0.05), dict(temperature=0.7, top_k=50, top_p=0.9, min_p=0.05)),
    (dict(top_k=0, epsilon_cutoff=3e-4), dict(epsilon=3e-4)),
    (dict(top_k=0, eta_cutoff=2e-3), dict(eta=float(np.float32(2e-3)))),
    (dict(temperature=0.8, top_k=40, top_p=0.95, min_p=0.02, epsilon_cutoff=1e-4, eta_cutoff=5e-4),
     dict(temperature=0.8, top_k=40, top_p=0.95, min_p=0.02, epsilon=1e-4, eta=float(np.float32(5e-4)))),
])
def test_device_warper_params_of_the_lists_generate_builds(kw, want):
    from lookaheaddecoding_b200.sampling import device_warper_params
    lp = _hf_list(**kw)
    got = device_warper_params(lp)
    full = {**dict(temperature=1.0, top_k=0, top_p=1.0, min_p=0.0, epsilon=0.0, eta=0.0), **want}
    assert got is not None and got.keys() == full.keys()
    for k, v in full.items():
        assert got[k] == pytest.approx(v, rel=1e-7), k
    assert isinstance(got["top_k"], int) and got["eta"] == full["eta"]     # the fp32 value of the eta tensor


def test_device_warper_params_rejects_what_the_kernel_does_not_implement():
    from transformers.generation.logits_process import (EpsilonLogitsWarper, EtaLogitsWarper, LogitsProcessorList,
                                                        MinPLogitsWarper, TemperatureLogitsWarper, TopKLogitsWarper,
                                                        TopPLogitsWarper, TypicalLogitsWarper)
    from lookaheaddecoding_b200.sampling import device_warper_params
    L = LogitsProcessorList
    assert device_warper_params(None) == dict(temperature=1.0, top_k=0, top_p=1.0, min_p=0.0, epsilon=0.0, eta=0.0)
    assert device_warper_params(L([MinPLogitsWarper(0.1), TopPLogitsWarper(0.9)])) is None          # out of order
    assert device_warper_params(L([EtaLogitsWarper(0.01), EpsilonLogitsWarper(0.01)])) is None
    assert device_warper_params(L([MinPLogitsWarper(0.1), MinPLogitsWarper(0.2)])) is None          # twice
    assert device_warper_params(L([TemperatureLogitsWarper(0.5), MinPLogitsWarper(0.1, min_tokens_to_keep=2)])) is None
    assert device_warper_params(L([EpsilonLogitsWarper(0.01, min_tokens_to_keep=2)])) is None
    assert device_warper_params(L([EtaLogitsWarper(0.01, filter_value=-1e4)])) is None
    assert device_warper_params(L([MinPLogitsWarper(0.1, filter_value=0.0)])) is None
    assert device_warper_params(L([MinPLogitsWarper(0.1), TypicalLogitsWarper(0.5)])) is None
    assert device_warper_params(_hf_list(top_k=0, min_p=0.1, epsilon_cutoff=1e-3, typical_p=0.9)) is None
    assert device_warper_params(L([TopKLogitsWarper(5), TopPLogitsWarper(0.5)]))["top_p"] == 0.5


def test_check_and_split_admit_the_threshold_warpers_only():
    from transformers.generation.logits_process import (EpsilonLogitsWarper, EtaLogitsWarper, LogitsProcessorList,
                                                        MinPLogitsWarper, RepetitionPenaltyLogitsProcessor,
                                                        TopKLogitsWarper, TypicalLogitsWarper)
    from lookaheaddecoding_b200 import LadeError
    from lookaheaddecoding_b200.sampling import _check_warpers, split_warpers
    lp = LogitsProcessorList([RepetitionPenaltyLogitsProcessor(1.1), TopKLogitsWarper(5), MinPLogitsWarper(0.1),
                              EpsilonLogitsWarper(1e-3), EtaLogitsWarper(1e-3)])
    procs, warpers = split_warpers(lp)
    assert [type(p).__name__ for p in procs] == ["RepetitionPenaltyLogitsProcessor"]
    assert [type(w).__name__ for w in warpers] == ["TopKLogitsWarper", "MinPLogitsWarper", "EpsilonLogitsWarper",
                                                   "EtaLogitsWarper"]
    _check_warpers(warpers)
    with pytest.raises(LadeError):
        _check_warpers(LogitsProcessorList([MinPLogitsWarper(0.1), TypicalLogitsWarper(0.5)]))


# ---------------------------------------------------------------------------------------------- range checks
def _warpers(**kw):
    from lookaheaddecoding_b200 import _cabi
    w = dict(temperature=1.0, top_k=0, top_p=1.0, min_p=0.0, epsilon=0.0, eta=0.0)
    w.update(kw)
    return _cabi.LadeWarpers(**w)


NAN = float("nan")
BAD = [dict(min_p=-1e-6), dict(min_p=1.0 + 1e-6), dict(min_p=NAN), dict(epsilon=1.0), dict(epsilon=-0.1),
       dict(epsilon=NAN), dict(eta=1.0), dict(eta=-1e-3), dict(eta=NAN), dict(temperature=0.0), dict(temperature=NAN),
       dict(top_k=-1), dict(top_p=0.0), dict(top_p=1.5), dict(top_p=NAN)]
GOOD = [{}, dict(min_p=1.0), dict(min_p=0.05, epsilon=0.9, eta=1e-4), dict(epsilon=1e-9), dict(eta=0.999)]


@pytest.mark.parametrize("sfx", ["", "_f16"])
def test_cabi_rejects_out_of_range_warpers_before_any_cuda_call(sfx):
    """A zeroed stand-in context: a valid record gets past the range checks to the context check (LADE_ESTATE: no
    sampling on a lookahead-parallel ctx, D = 0 here), an invalid one stops at LADE_EINVAL."""
    from lookaheaddecoding_b200 import _cabi
    fn = getattr(_cabi.load(), "lade_sample_verify_warped" + sfx)
    ctx = (C.c_char * 4096)()
    buf = (C.c_int32 * 64)()
    p = C.addressof(buf)

    def call(w, vocab=8, ld=8):
        return fn(C.addressof(ctx), None, p, ld, vocab, p, p, C.byref(w), p, p, None, None)
    for kw in GOOD:
        assert call(_warpers(**kw)) == _cabi.LADE_ESTATE, kw
    for kw in BAD:
        assert call(_warpers(**kw)) == _cabi.LADE_EINVAL, kw
    assert call(_warpers(), vocab=9) == _cabi.LADE_EINVAL                               # ld < vocab
    assert fn(C.addressof(ctx), None, p, 8, 8, p, p, None, p, p, None, None) == _cabi.LADE_EINVAL


def test_engine_sampling_ranges_match_the_cabi():
    """LookaheadEngine.generate checks the sampling dict before touching the device (engine built without __init__)."""
    from lookaheaddecoding_b200 import LadeError, LookaheadEngine
    eng = LookaheadEngine.__new__(LookaheadEngine)
    eng.max_total_len, eng.DW = 64, 1
    for kw in BAD[:9]:
        key = {"min_p": "min_p", "epsilon": "epsilon", "eta": "eta"}[next(iter(kw))]
        with pytest.raises(LadeError, match=key):
            eng.generate([1, 2, 3], 4, sampling=dict(kw, temperature=1.0))
