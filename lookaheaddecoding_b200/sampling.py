"""Sampling lookahead decoding: ``jacobi_sample_multilevel`` (``lade/decoding.py:137-692``) on the CUDA engine.

Two ways to run the multi-candidate rejection-sampling verification (``decoding.py:484-540``, modified SpecInfer):

* **device (default for the warper lists HF builds from temperature / top_k / top_p / min_p / epsilon_cutoff /
  eta_cutoff)**: ``lade_sample_verify`` (``lade_sample_verify_warped`` with min_p, epsilon or eta) --
  temperature, top-k, top-p, min-p, epsilon and eta cut-offs, softmax, accept tests, zero-and-renormalise, residual multinomial draw and
  the EOS window filter in one kernel driven by a Philox stream -- followed by ``lade_commit_decision``; the whole step replays from one CUDA graph and the host loop is the
  pipelined greedy loop (``LookaheadEngine.generate(..., sampling=...)``).  Same distribution as the reference, its own
  random stream (seeded from torch's global generator, so ``torch.manual_seed`` makes a run reproducible).
* **host-RNG compatibility mode** (``sample_lookahead`` below; used when ``CONFIG_MAP["SAMPLING_ON_HOST"]`` is set
  or the warpers carry non-default filter values): the model forward, window / pool / KV bookkeeping and row-wise argmax
  run on the device; the verification runs here against device probability tensors, consuming python's
  ``random.random()`` for the accept tests and ``torch.multinomial`` for the residual draw in the reference's order,
  so that under fixed seeds the token stream follows the reference draw for draw (the fixed-seed golden tests).

Restrictions inherited from the reference: warpers within {Temperature, TopK, TopP} (``decoding.py:375-377``), to
which this port adds the threshold warpers {MinP, Epsilon, Eta} (each keeps every score at or above a cut, so lookahead
stays lossless: every verification row is warped as its own distribution, like the top-p cut); no other logits processors (``:412``), batch 1, ``return_dict_in_generate == False``; no lookahead
parallelism on this path (the reference has none either beyond the initial window broadcast).
"""
from __future__ import annotations

import ctypes as C
import random
from typing import List, Optional

import numpy as np
import torch

from . import _cabi
from ._cabi import LadeError, check


def _supported_warpers():
    """The warper classes of the sampling path, in HF's list order (GenerationMixin._get_logits_processor)."""
    from transformers.generation.logits_process import (EpsilonLogitsWarper, EtaLogitsWarper, MinPLogitsWarper,
                                                        TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper)
    return (TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper, MinPLogitsWarper, EpsilonLogitsWarper,
            EtaLogitsWarper)


def split_warpers(logits_processor):
    """transformers 5.x keeps the warpers inside the processor list; split them back out."""
    from transformers.generation.logits_process import LogitsProcessorList
    supported = _supported_warpers()
    procs, warpers = LogitsProcessorList(), LogitsProcessorList()
    for p in (logits_processor or []):
        (warpers if isinstance(p, supported) else procs).append(p)
    return procs, warpers


def _check_warpers(logits_warper):
    supported = _supported_warpers()
    for w in (logits_warper or []):
        if type(w) not in supported:
            raise LadeError(f"please set top_k=0.0 and top_p=1.0 {w}")                     # decoding.py:377


def device_sampling_params(logits_warper):
    """(temperature, top_k, top_p) when the warper list is what HF builds from generate(temperature=, top_k=, top_p=) --
    at most one TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper, in that order, -inf filter value,
    min_tokens_to_keep = 1 -- i.e. what the device kernel implements; else None (host-RNG compatibility loop)."""
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper
    order = {TemperatureLogitsWarper: 0, TopKLogitsWarper: 1, TopPLogitsWarper: 2}
    T, k, p, last = 1.0, 0, 1.0, -1
    for w in list(logits_warper or []):
        rank = order.get(type(w))
        if rank is None or rank <= last:
            return None
        last = rank
        if rank == 0:
            T = float(w.temperature)
        else:
            if getattr(w, "filter_value", -float("inf")) != -float("inf") or getattr(w, "min_tokens_to_keep", 1) != 1:
                return None
            if rank == 1:
                k = int(w.top_k)
            else:
                p = float(w.top_p)
    if not T > 0 or k < 0 or not 0.0 < p <= 1.0:
        return None
    return T, k, p


def device_warper_params(logits_warper):
    """dict(temperature, top_k, top_p, min_p, epsilon, eta) -- the LadeWarpers record -- when the warper list is what HF
    builds from generate(temperature=, top_k=, top_p=, min_p=, epsilon_cutoff=, eta_cutoff=): each warper at most once,
    in HF's order, -inf filter value, min_tokens_to_keep = 1; else None (host-RNG compatibility loop).  Values are read
    from the warpers' own attributes (EtaLogitsWarper holds its epsilon as an fp32 tensor)."""
    supported = _supported_warpers()
    rank_of = {cls: r for r, cls in enumerate(supported)}
    names = ("temperature", "top_k", "top_p", "min_p", "epsilon", "eta")
    attrs = ("temperature", "top_k", "top_p", "min_p", "epsilon", "epsilon")      # each warper's own attribute
    out = dict(temperature=1.0, top_k=0, top_p=1.0, min_p=0.0, epsilon=0.0, eta=0.0)
    last = -1
    for w in list(logits_warper or []):
        rank = rank_of.get(type(w))
        if rank is None or rank <= last:
            return None
        last = rank
        if rank > 0 and (getattr(w, "filter_value", -float("inf")) != -float("inf")
                         or getattr(w, "min_tokens_to_keep", 1) != 1):
            return None
        value = getattr(w, attrs[rank])
        out[names[rank]] = int(value) if rank == 1 else float(value.item() if torch.is_tensor(value) else value)
    ok = (out["temperature"] > 0 and out["top_k"] >= 0 and 0.0 < out["top_p"] <= 1.0 and 0.0 <= out["min_p"] <= 1.0
          and all(out[k] == 0.0 or 0.0 < out[k] < 1.0 for k in ("epsilon", "eta")))
    return out if ok else None


def device_temperature(logits_warper):
    """T if the warper list is empty or a single TemperatureLogitsWarper, else None (kept for callers of round 2's API)."""
    params = device_sampling_params(logits_warper)
    return params[0] if params is not None and params[1] == 0 and params[2] == 1.0 else None


@torch.no_grad()
def sample_lookahead(eng, prompt: List[int], max_new_tokens: int, logits_warper, eos_token_ids=(),
                     rng=None, window0=None, stop_fn=None) -> List[int]:
    """Drive one sampling generate() on `eng` (a LookaheadEngine). Returns prompt + sampled ids."""
    if eng.DW != 1:
        raise LadeError("the sampling path has no lookahead parallelism (reference: replicas only)")
    rnd = rng or random
    lib = eng.lib
    P = len(prompt)
    max_length = P + int(max_new_tokens)
    if max_length > eng.max_total_len:
        raise LadeError(f"prompt+max_new_tokens={max_length} exceeds engine capacity {eng.max_total_len}")
    eos = list(eos_token_ids or [])
    all_old_tokens = list(prompt)

    def set_token():                                                                       # copy_from, :336-337,:351
        return rnd.choice(all_old_tokens)

    eng.begin(prompt, max_length, eos, eng.draw_window(prompt, rnd, window0))
    stream = torch.cuda.current_stream(eng.dev).cuda_stream
    dev = eng.dev
    W, N, GS, WCAP = eng.W, eng.N, eng.GS, eng.WCAP
    R = eng.rec_ints
    dec_host = torch.zeros(R + 4 + W, dtype=torch.int32, pin_memory=True)
    dec_dev = torch.zeros(R + 4 + W, dtype=torch.int32, device=dev)
    warp = logits_warper if logits_warper is not None else (lambda ids, s: s)
    eos_t = torch.tensor(eos, device=dev) if eos else None

    out = list(prompt)
    input_ids = torch.tensor([out], device=dev)
    next_tokens = None            # the reference's `next_tokens` is only refreshed on some branches (sic)
    step = 0
    eng.last_records = []
    while True:
        eng.run_forward_step(step, P, commit=False)
        meta = eng.meta.cpu().tolist()                       # sync point (the reference has several per step)
        am = eng.am.cpu().tolist()
        phase, tiny, lg = meta[_cabi.M_PHASE], meta[_cabi.M_TINY], meta[_cabi.M_N_GUESS_TOK]
        inp_tokens = am[1:1 + tiny]
        next_token_logits = eng.logits[0:1].float()                                        # outputs.out_logits
        next_token_scores = warp(input_ids, next_token_logits)                             # :445
        max_hit, max_hit_idx = 0, 0
        new_results = list(inp_tokens)
        filtered = None
        if phase != 2 or lg == 0:                                                          # :458-480, :543-546
            probs = torch.nn.functional.softmax(next_token_scores, dim=-1)
            next_tokens = torch.multinomial(probs, num_samples=1).squeeze(1)
            hits = [next_tokens.item()]
        else:
            # Candidate verification with the HOST random streams (fixed-seed compatibility with the reference's
            # draws, decoding.py:484-540): a uniform from python's `random` per accept test, torch.multinomial for the
            # residual draw.  Probabilities stay on the device; only the probability of the token under test and the
            # drawn token cross to the host.
            q_len = meta[_cabi.M_Q_LEN]
            grams = np.asarray(eng.ids[q_len - lg:q_len].cpu().tolist(), dtype=np.int64).reshape(-1, GS)
            slot_probs = torch.nn.functional.softmax(warp(input_ids, eng.logits[1 + WCAP:1 + WCAP + lg].float()), dim=-1)
            dist = torch.nn.functional.softmax(next_token_scores, dim=-1)[0]      # distribution of the token being decided
            alive = np.ones(len(grams), dtype=bool)
            hits = []
            for pos in range(GS):
                winner = -1
                for cand in np.flatnonzero(alive):
                    tok = int(grams[cand, pos])
                    if rnd.random() < min(1, dist[tok].item()):                 # :505-508
                        winner = int(cand)
                        break
                    dist[tok] = 0                                               # :518-520
                    dist = dist / dist.sum()
                if winner < 0:
                    hits.append(torch.multinomial(dist, num_samples=1).item())  # :533-535
                    break
                tok = int(grams[winner, pos])
                hits.append(tok)
                max_hit_idx = winner
                alive &= grams[:, pos] == tok                                   # :513-516
                dist = slot_probs[winner * GS + pos]                            # :530
            max_hit = len(hits) - 1
        if phase == 2 and eos:                                                             # :578-580
            filtered = list(new_results)          # the pool was already fed the unfiltered row (:563)
            for i in range(len(filtered)):
                if filtered[i] == eos[0]:
                    filtered[i] = set_token()

        # stopping bookkeeping as :594-643 (all_old_tokens gets the *right* hit here, unlike the greedy path)
        n_emit = max_hit + 1
        finished = False
        for hit_ids in range(max_hit + 1):
            if eos and hits[hit_ids] == eos[0]:
                all_old_tokens.append(hits[hit_ids])
                next_tokens = eos_t
                n_emit = hit_ids + 1
                break
            all_old_tokens.append(hits[hit_ids])
        if eos_t is not None and next_tokens is not None:
            finished = bool(next_tokens.tile(eos_t.shape[0], 1).ne(eos_t.unsqueeze(1)).prod(dim=0).max() == 0)

        # hand the decision to the device state machine
        d = dec_host.zero_()
        d[0], d[1], d[2] = hits[0], max_hit, len(new_results)
        for i, h in enumerate(hits[:GS]):
            d[3 + i] = h
        for i, t in enumerate(new_results):
            d[3 + GS + i] = t
        d[R], d[R + 1], d[R + 2] = max_hit_idx, 1 | (2 if filtered is not None else 0), int(finished)
        if filtered is not None:
            for i, t in enumerate(filtered):
                d[R + 4 + i] = t
        dec_dev.copy_(dec_host, non_blocking=True)
        check(lib.lade_commit_decision(eng._ctx, stream, dec_dev.data_ptr(), eng.meta.data_ptr(), eng.res.data_ptr()),
              "lade_commit_decision")
        check(lib.lade_kv_compact(stream, eng.res.data_ptr(), eng.kv[0, 0].data_ptr(), eng.kv[0, 1].data_ptr(),
                                  eng.kv.stride(0), eng.L, eng.nkv, eng.kv_capacity, eng.D, max(GS - 1, 1)), "lade_kv_compact")
        eng.launches += 2
        rec = eng._read_result()
        eng.last_records.append(rec)
        out.extend(hits[:n_emit])
        input_ids = torch.tensor([out], device=dev)
        step += 1
        if rec.done or finished or len(out) >= max_length or (stop_fn is not None and stop_fn(out[:max_length])):
            break                                                                          # :636-646
        if step > max_new_tokens + N + 4:
            raise LadeError("sampling loop did not terminate")
    eng.last_steps = step
    return out[:max_length]


def jacobi_sample_multilevel(self, input_ids: torch.LongTensor, logits_processor=None, stopping_criteria=None,
                             logits_warper=None, max_length: Optional[int] = None, pad_token_id=None,
                             eos_token_id=None, output_attentions=None, output_hidden_states=None,
                             output_scores=None, return_dict_in_generate=None, synced_gpus: bool = False,
                             streamer=None, chat: bool = False, **model_kwargs):
    """Drop-in for lade/decoding.py:137 (same argument meaning; `chat` accepted and ignored)."""
    from .decoding import CONFIG_MAP, _max_length_from, get_engine

    if input_ids.shape[0] != 1:
        raise LadeError("lookahead decoding supports batch size 1 only (modeling_llama.py:1448)")
    if logits_processor is not None and len(logits_processor) != 0:
        raise LadeError("logits processors are not supported (decoding.py:412)")
    if return_dict_in_generate:
        raise LadeError("return_dict_in_generate must be False (decoding.py:411)")
    _check_warpers(logits_warper)
    if isinstance(eos_token_id, int):
        eos_token_id = [eos_token_id]
    if torch.is_tensor(eos_token_id):
        eos_token_id = eos_token_id.tolist()
    init_len = input_ids.shape[1]
    total = _max_length_from(stopping_criteria, max_length, init_len)
    saved = CONFIG_MAP.get("DIST_WORKERS")
    try:
        CONFIG_MAP.pop("DIST_WORKERS", None)      # sampling: replicas only
        eng = get_engine(self, max_total_len=total, min_total_len=total)
    finally:
        if saved is not None:
            CONFIG_MAP["DIST_WORKERS"] = saved
    from .decoding import _extra_stopping_criteria, _host_stop_fn
    stop_fn = _host_stop_fn(_extra_stopping_criteria(stopping_criteria), input_ids.device, input_ids.dtype)
    params = device_warper_params(logits_warper)
    if params is not None and not CONFIG_MAP.get("SAMPLING_ON_HOST", 0):
        seed = int(torch.randint(0, 2 ** 62, (1,)).item())          # reproducible under torch.manual_seed
        out = eng.generate(input_ids[0].tolist(), total - init_len, eos_token_ids=eos_token_id or (), rng=random,
                           stop_fn=stop_fn, sampling=dict(params, seed=seed))
    else:
        out = sample_lookahead(eng, input_ids[0].tolist(), total - init_len, logits_warper, eos_token_id or (), rng=random,
                               stop_fn=stop_fn)
    if streamer is not None:
        streamer.put(torch.tensor(out[init_len:]))
        streamer.end()
    n_gen, steps = len(out) - init_len, eng.last_steps
    if CONFIG_MAP.get("DEBUG", 0) and CONFIG_MAP.get("LOCAL_RANK", 0) == 0:                          # :662-666
        print("\n==========================ACCELERATION===SUMMARY======================================")
        print("Generated tokens: ", n_gen, "Total steps: ", steps, " Compression ratio: ", round(n_gen / steps, 2))
        print("======================================================================================", end="")
        CONFIG_MAP.setdefault("log", []).append([n_gen, steps, round(n_gen / steps, 2)])
    return torch.tensor([out], dtype=input_ids.dtype, device=input_ids.device)
