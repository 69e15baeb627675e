"""Host mirror of the reference's decode entry points (``lade/decoding.py``), driving the CUDA engine.

Same names and argument meaning as the reference so call sites and tests read alike:

  greedy_search_proxy / sample_proxy        lade/decoding.py:15-34   (env ``USE_LADE`` dispatch)
  jacobi_greedy_search_multilevel           lade/decoding.py:697     (greedy lookahead loop)
  CONFIG_MAP / FUNC_MAP                     lade/decoding.py:11-12

The reference patches ``GenerationMixin.greedy_search`` / ``.sample`` (transformers 4.36).  The
installed transformers (5.x) routes both through ``GenerationMixin._sample`` with
``generation_config.do_sample`` selecting the mode; ``sample_entry_proxy`` adapts that call to the
two reference-style entry points.  ``CHAT`` streaming / colour printing is UI and out of scope.
"""
from __future__ import annotations

import os
import random
from typing import Optional

import torch

from .engine import LookaheadEngine
from ._cabi import LadeError

FUNC_MAP = {}
CONFIG_MAP = {}


def _use_lade() -> bool:
    return bool(int(os.environ.get("USE_LADE", 0)))


def greedy_search_proxy(self, *args, **kwargs):
    """lade/decoding.py:15-26."""
    if _use_lade():
        return jacobi_greedy_search_multilevel(self, *args, chat=bool(int(os.environ.get("CHAT", 0))), **kwargs)
    return FUNC_MAP["greedy_search"](self, *args, **kwargs)


def sample_proxy(self, *args, **kwargs):
    """lade/decoding.py:28-34."""
    if _use_lade():
        from .sampling import jacobi_sample_multilevel
        return jacobi_sample_multilevel(self, *args, chat=bool(int(os.environ.get("CHAT", 0))), **kwargs)
    return FUNC_MAP["sample"](self, *args, **kwargs)


def sample_entry_proxy(self, input_ids, logits_processor=None, stopping_criteria=None, generation_config=None,
                       synced_gpus=False, streamer=None, **model_kwargs):
    """Replacement of transformers-5.x ``GenerationMixin._sample`` (the single greedy/sample entry)."""
    if not _use_lade():
        return FUNC_MAP["_sample"](self, input_ids, logits_processor, stopping_criteria, generation_config,
                                   synced_gpus=synced_gpus, streamer=streamer, **model_kwargs)
    do_sample = bool(getattr(generation_config, "do_sample", False))
    eos = getattr(generation_config, "_eos_token_tensor", None)
    eos_ids = eos.tolist() if eos is not None else getattr(generation_config, "eos_token_id", None)
    pad = getattr(generation_config, "_pad_token_tensor", None)
    common = dict(
        stopping_criteria=stopping_criteria, pad_token_id=pad, eos_token_id=eos_ids,
        output_attentions=bool(generation_config.output_attentions),
        output_hidden_states=bool(generation_config.output_hidden_states),
        output_scores=bool(generation_config.output_scores),
        return_dict_in_generate=bool(generation_config.return_dict_in_generate),
        synced_gpus=synced_gpus, streamer=streamer, **model_kwargs)
    if do_sample:
        from .sampling import jacobi_sample_multilevel, split_warpers
        processors, warpers = split_warpers(logits_processor)
        return jacobi_sample_multilevel(self, input_ids, logits_processor=processors, logits_warper=warpers, **common)
    return jacobi_greedy_search_multilevel(self, input_ids, logits_processor=logits_processor, **common)


def _max_length_from(stopping_criteria, max_length, init_len) -> int:
    best = None
    for crit in (stopping_criteria or []):
        ml = getattr(crit, "max_length", None)
        if ml is not None:
            best = ml if best is None else min(best, ml)
    if max_length is not None:
        best = init_len + max_length if best is None else min(best, init_len + max_length)
    if best is None:
        raise LadeError("no MaxLengthCriteria / max_length given: cannot bound the KV cache")
    return int(best)


def _extra_stopping_criteria(stopping_criteria):
    """Criteria beyond max-length / EOS (both handled on device).  The reference evaluates the whole list on every step
    (lade/decoding.py:1215, :646); anything else here is evaluated on the host after each step record."""
    from transformers.generation.stopping_criteria import MaxLengthCriteria
    try:
        from transformers.generation.stopping_criteria import EosTokenCriteria
    except ImportError:      # transformers 4.36 has no EosTokenCriteria
        EosTokenCriteria = ()
    handled = (MaxLengthCriteria,) + ((EosTokenCriteria,) if EosTokenCriteria else ())
    return [c for c in (stopping_criteria or []) if not isinstance(c, handled)]


def _host_stop_fn(extra, device, dtype):
    if not extra:
        return None

    def stop(ids) -> bool:
        t = torch.tensor([ids], dtype=dtype, device=device)
        for crit in extra:
            if bool(torch.as_tensor(crit(t, None)).all()):
                return True
        return False
    return stop


def processors_from_hf(logits_processor) -> Optional[dict]:
    """The engine's `processors` dict for a greedy LogitsProcessorList, read from the processors' own attributes.  Only
    processors that depend on nothing but the row's prefix are supported: RepetitionPenaltyLogitsProcessor,
    NoRepeatNGramLogitsProcessor, MinLengthLogitsProcessor and MinNewTokensLengthLogitsProcessor (the reference allows
    none, lade/decoding.py:968).  Anything else raises a LadeError naming its class."""
    from transformers.generation.logits_process import (MinLengthLogitsProcessor, MinNewTokensLengthLogitsProcessor,
                                                        NoRepeatNGramLogitsProcessor, RepetitionPenaltyLogitsProcessor)
    if not logits_processor:
        return None
    out, bounds, eos = {}, [], None
    for p in logits_processor:
        kind = type(p)
        if kind in (RepetitionPenaltyLogitsProcessor, NoRepeatNGramLogitsProcessor) and \
                ("penalty" if kind is RepetitionPenaltyLogitsProcessor else "ngram_size") in out:
            raise LadeError(f"{kind.__name__} given twice: not supported on the lookahead greedy path")
        if kind is RepetitionPenaltyLogitsProcessor:
            out["penalty"] = float(p.penalty)
            out["prompt_ignore_length"] = int(p.prompt_ignore_length or 0)
        elif kind is NoRepeatNGramLogitsProcessor:
            out["ngram_size"] = int(p.ngram_size)
        elif kind in (MinLengthLogitsProcessor, MinNewTokensLengthLogitsProcessor):
            ids = sorted({int(e) for e in torch.as_tensor(p.eos_token_id).reshape(-1).tolist()})
            if eos is not None and ids != eos:
                raise LadeError("the min-length logits processors name different eos ids: not supported")
            eos = ids
            bounds.append(int(p.min_length) if kind is MinLengthLogitsProcessor
                          else int(p.prompt_length_to_skip) + int(p.min_new_tokens))
        else:
            raise LadeError(f"logits processor {kind.__name__} is not supported on the lookahead greedy path "
                            "(supported: RepetitionPenaltyLogitsProcessor, NoRepeatNGramLogitsProcessor, "
                            "MinLengthLogitsProcessor, MinNewTokensLengthLogitsProcessor)")
    if bounds:
        out["min_length"] = max(bounds)
        out["eos_token_id"] = eos
    return out


def get_engine(model, **overrides) -> LookaheadEngine:
    """One engine per (model, lookahead config); reads CONFIG_MAP like lade/decoding.py:854-862."""
    W = CONFIG_MAP.get("WINDOW_SIZE", 60)
    G = CONFIG_MAP.get("GUESS_SET_SIZE", 60)
    N = CONFIG_MAP.get("LEVEL", 8)
    pool = bool(CONFIG_MAP.get("POOL_FROM_PROMPT", 0))
    overrides = {**CONFIG_MAP.get("ENGINE_OVERRIDES", {}), **overrides}
    # capacity: at least the request, and at least MAX_TOTAL_LEN (default 4096) so that a later, longer request does not
    # tear the engine down (KV cache + CUDA graphs) again
    cap = max(int(overrides.pop("max_total_len", 0)), int(CONFIG_MAP.get("MAX_TOTAL_LEN", 4096)))
    max_pos = int(getattr(model.config, "max_position_embeddings", cap) or cap)
    cap = max(int(overrides.pop("min_total_len", 0)), min(cap, max(max_pos, 1)))
    if CONFIG_MAP.get("DIST_WORKERS", 1) > 1:                         # lookahead parallelism (lade/utils.py:28-33)
        overrides.setdefault("dist_workers", CONFIG_MAP["DIST_WORKERS"])
        overrides.setdefault("rank", CONFIG_MAP.get("LOCAL_RANK", 0))
    key = (W, N, G, pool, tuple(sorted(overrides.items())))
    cache = model.__dict__.setdefault("_lade_engines", {})
    eng = cache.get(key)
    if eng is None or eng.max_total_len < cap:
        if eng is not None:          # drop the old engine (KV cache, graphs) BEFORE building the new one
            eng.close()
            del cache[key]
            eng = None
            torch.cuda.empty_cache()
        eng = LookaheadEngine(model, W, N, G, pool_from_prompt=pool, max_total_len=cap, **overrides)
        cache[key] = eng
    return eng


def jacobi_greedy_search_multilevel(self, input_ids: torch.LongTensor, logits_processor=None,
                                    stopping_criteria=None, max_length: Optional[int] = None,
                                    pad_token_id=None, eos_token_id=None, output_attentions=None,
                                    output_hidden_states=None, output_scores=None,
                                    return_dict_in_generate=None, synced_gpus: bool = False, streamer=None,
                                    chat: bool = False, stop_token: Optional[str] = None, **model_kwargs):
    """Greedy lookahead decoding on the H100 engine; drop-in for lade/decoding.py:697-1259.

    Logits processors: the prefix-only ones of ``processors_from_hf`` run on device (the reference allows none,
    :968); any other raises.  Inherited restrictions (fail loudly, as the reference asserts): batch size 1
    (modeling_llama.py:1448), ``return_dict_in_generate == False``
    (:967), ``ALWAYS_FWD_ONE == 1`` (:873), LEVEL >= 3 (:902).  ``stop_token`` / ``chat`` are
    accepted and ignored (UI only).
    """
    if input_ids.shape[0] != 1:
        raise LadeError("lookahead decoding supports batch size 1 only (modeling_llama.py:1448)")
    processors = processors_from_hf(logits_processor)
    if processors and CONFIG_MAP.get("DIST_WORKERS", 1) > 1:
        raise LadeError("logits processors are not supported with lookahead parallelism (DIST_WORKERS > 1)")
    if return_dict_in_generate:
        raise LadeError("return_dict_in_generate must be False (decoding.py:967)")
    if CONFIG_MAP.get("ALWAYS_FWD_ONE", 1) != 1:
        raise LadeError("ALWAYS_FWD_ONE must be 1 (decoding.py:873)")
    if output_attentions or output_hidden_states or output_scores:
        raise LadeError("output_attentions/hidden_states/scores are not supported")
    if isinstance(eos_token_id, int):
        eos_token_id = [eos_token_id]                                          # decoding.py:820-821
    if torch.is_tensor(eos_token_id):
        eos_token_id = eos_token_id.tolist()
    if eos_token_id is not None and pad_token_id is None:
        raise ValueError("If `eos_token_id` is defined, make sure that `pad_token_id` is defined.")   # :1028-1029
    init_len = input_ids.shape[1]
    total = _max_length_from(stopping_criteria, max_length, init_len)
    eng = get_engine(self, max_total_len=total, min_total_len=total)
    prompt = input_ids[0].tolist()
    stop_fn = _host_stop_fn(_extra_stopping_criteria(stopping_criteria), input_ids.device, input_ids.dtype)
    out = eng.generate(prompt, total - init_len, eos_token_ids=eos_token_id or (), rng=random, stop_fn=stop_fn,
                       processors=processors)
    if streamer is not None:
        streamer.put(torch.tensor(out[init_len:]))
        streamer.end()
    n_gen, steps = len(out) - init_len, eng.last_steps
    if CONFIG_MAP.get("DEBUG", 0) and CONFIG_MAP.get("LOCAL_RANK", 0) == 0:                           # :1231-1235
        print("\n==========================ACCELERATION===SUMMARY======================================")
        print("Generated tokens: ", n_gen, "Total steps: ", steps, " Compression ratio: ", round(n_gen / steps, 2))
        print("======================================================================================", end="")
        CONFIG_MAP.setdefault("log", []).append([n_gen, steps, round(n_gen / steps, 2)])
    return torch.tensor([out], dtype=input_ids.dtype, device=input_ids.device)
