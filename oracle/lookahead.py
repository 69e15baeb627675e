"""TEST INFRASTRUCTURE ONLY -- CPU restatement of lade's lookahead/verification state machine.

Plain Python/numpy restatement of the integer side of the hot path of
hao-ai-lab/LookaheadDecoding (citations are ``/root/reference/...`` file:line).  It is the
*checker* for the CUDA path: only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s
``cpu_baseline`` / ``--impl reference`` legs may import it.  The product package
(``lookaheaddecoding_b200``) never does.

Parity status: PINNED.  The reference ships no tests or golden vectors (SURVEY.md section 4), so this
restatement is pinned against the reference *itself*, executed unmodified through
``baseline/ref_loader.py`` (``oracle/ref_shim.py`` is its old import path): per-step traces (step rows,
position ids, masks, argmax tokens, hits, pool contents, final ids) are committed under ``tests/golden/`` by
``tests/golden/gen_golden*.py`` and checked by ``tests/test_oracle_golden.py``, ``test_oracle_edge.py``,
``test_oracle_pool.py``, ``test_oracle_sampling.py`` and ``test_lp_gloo.py``.

Vocabulary follows the reference: LEVEL (N), WINDOW_SIZE (W), GUESS_SET_SIZE (G), guess size = N-1,
``past_tokens`` = the 2-D lookahead window (N-1 levels), ``token_map`` = the n-gram pool,
``hits`` / ``max_hit`` = the accepted tokens of a step.
"""
from __future__ import annotations

import random
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np

# Row classes of a step (used by the mask predicate and mirrored by the CUDA row descriptors).
ROW_PREFIX = 0   # re-fed input tokens (+ the L0 prefix a rank does not own under LP): causal
ROW_WINDOW = 1   # lookahead window row (level, column)
ROW_GUESS = 2    # verification-branch row (n-gram, index in n-gram)
ROW_PAD = 3      # padding row of the fixed-shape device layout: sees only itself


# --------------------------------------------------------------------------------------------
# n-gram pool  (lade/decoding.py:37-127)
# --------------------------------------------------------------------------------------------
def pool_insert(token_map: Dict[int, list], key: int, tup: Tuple[int, ...], G: int) -> None:
    """One LRU insertion (lade/decoding.py:39-49 and the identical blocks at :52-63, :86-96, :112-122).

    Present -> move to the end; room -> append; full -> drop the oldest, append.
    """
    assert G != -1, "GUESS_SET_SIZE=-1 (unbounded python set) is not supported by the device path"
    lst = token_map.setdefault(key, [])
    if tup in lst:
        lst.remove(tup)
        lst.append(tup)
    elif len(lst) < G:
        lst.append(tup)
    else:
        assert len(lst) == G
        token_map[key] = lst[1:] + [tup]


def update_token_map(token_map, lst_token, past_tokens, new_results, N, W, G) -> None:
    """lade/decoding.py:37-63: W insertions, column i keyed by the token left of the diagonal start."""
    for i in range(W):
        key = lst_token if i == 0 else past_tokens[0][i - 1]
        tup = tuple(past_tokens[ll][i] for ll in range(1, N - 1)) + (new_results[i],)
        pool_insert(token_map, key, tup, G)


def append_new_generated_pool(tokens, token_map, N, G) -> None:
    """lade/decoding.py:80-96 (no-op unless exactly N tokens are given)."""
    if len(tokens) != N:
        return
    pool_insert(token_map, tokens[0], tuple(tokens[1:]), G)


def fill_pool_with_prompt(prompt, token_map, N, G) -> None:
    """lade/decoding.py:104-122: every N-gram of the prompt, in order."""
    for s in range(len(prompt) - N + 1):
        pool_insert(token_map, prompt[s], tuple(prompt[s + 1:s + N]), G)


# --------------------------------------------------------------------------------------------
# step layout: token rows + position ids  (lade/models/modeling_llama.py:1458-1511)
# --------------------------------------------------------------------------------------------
@dataclass
class StepLayout:
    ids: List[int]              # token id of every step row
    pos: List[int]              # position id of every step row
    row_type: List[int]         # ROW_*
    row_blk: List[int]          # prefix: 0 ; window: level ; guess: n-gram index
    row_idx: List[int]          # prefix: i ; window: column ; guess: index in n-gram
    level_sizes: List[int]
    n_input: int                # number of re-fed input rows (1 + guess_skip_dist)
    n_guess_tok: int            # len(guess_tokens)
    is_prefill: bool
    # derived mask scalars (modeling_llama.py:136-137,188)
    level_offset: int = 0
    dist_offset: int = 0
    tiny: int = 0               # level_sizes[-1]

    @property
    def q_len(self) -> int:
        return len(self.ids)


def build_step_layout(input_tail: Sequence[int], lst_id: int, past_tokens_inp, fill_level: int,
                      guess_tokens: Optional[Sequence[int]], N: int, is_first: bool) -> StepLayout:
    """Token/position rows of one step.

    ``input_tail`` are the input rows fed this step (the whole prompt on the first step, otherwise
    the last ``1+guess_skip_dist`` ids, lade/decoding.py:938-942); ``lst_id`` is the position id of
    the last of them (modeling_llama.py:1466).  Mirrors modeling_llama.py:1487-1511.
    """
    ids = list(input_tail)
    n_in = len(ids)
    pos = list(range(lst_id - n_in + 1, lst_id + 1))
    level_sizes = []
    win_ids, win_pos = [], []
    for ll in range(fill_level + 1):
        lvl = past_tokens_inp[ll]
        win_ids += list(lvl)
        level_sizes.append(len(lvl))
        if ll == 0:
            win_pos += list(range(lst_id + 1, lst_id + 1 + len(lvl)))                    # :1494
        else:
            off = len(past_tokens_inp[0]) + 1 - len(lvl)                                 # :1496
            win_pos += list(range(lst_id + ll + off, lst_id + ll + off + len(lvl)))      # :1497
    g = list(guess_tokens) if guess_tokens is not None else []
    gs = N - 1
    g_pos = list(range(lst_id + 1, lst_id + 1 + gs)) * (len(g) // gs)                    # :1501
    ids = ids + win_ids + g
    pos = pos + win_pos + g_pos

    is_prefill = past_tokens_inp[1] is None                                              # :1527
    lay = StepLayout(ids=ids, pos=pos, row_type=[], row_blk=[], row_idx=[],
                     level_sizes=level_sizes, n_input=n_in, n_guess_tok=len(g), is_prefill=is_prefill)
    classify_rows(lay, len(ids), gs)
    return lay


def classify_rows(lay: StepLayout, q: int, gs: int) -> None:
    """Row classes + mask scalars from (q, level_sizes, n_guess_tok); modeling_llama.py:132-138."""
    lay.row_type, lay.row_blk, lay.row_idx = [0] * q, [0] * q, [0] * q
    if lay.is_prefill:
        for r in range(q):
            lay.row_type[r], lay.row_idx[r] = ROW_PREFIX, r
        return
    ng = lay.n_guess_tok
    tiny = lay.level_sizes[-1]
    level_offset = q - (sum(lay.level_sizes) + 1) - ng                                   # :136
    dist_offset = 1 + lay.level_sizes[0] - tiny                                          # :137
    assert level_offset >= 0 and dist_offset >= 0
    a = level_offset + dist_offset
    lay.level_offset, lay.dist_offset, lay.tiny = level_offset, dist_offset, tiny
    for r in range(q):
        if r < a:
            lay.row_type[r], lay.row_blk[r], lay.row_idx[r] = ROW_PREFIX, 0, r
        elif r < q - ng:
            lay.row_type[r] = ROW_WINDOW
            lay.row_blk[r], lay.row_idx[r] = divmod(r - a, tiny)
        else:
            lay.row_type[r] = ROW_GUESS
            lay.row_blk[r], lay.row_idx[r] = divmod(r - (q - ng), gs)


def layout_from_shape(level_sizes, n_input: int, n_guess_tok: int, gs: int, is_prefill=False) -> StepLayout:
    """A layout carrying only the mask-relevant shape (for mask-only checks, incl. LP shapes)."""
    q = n_input + sum(level_sizes) + n_guess_tok
    lay = StepLayout(ids=[0] * q, pos=[0] * q, row_type=[], row_blk=[], row_idx=[],
                     level_sizes=list(level_sizes), n_input=n_input, n_guess_tok=n_guess_tok,
                     is_prefill=is_prefill)
    classify_rows(lay, q, gs)
    return lay


def row_sees(lay: StepLayout, r: int, c: int) -> bool:
    """Mask predicate over step-local (row, column); SURVEY.md App. B == modeling_llama.py:115-207.

    This is the function the CUDA attention kernel evaluates in registers from the row descriptors.
    Columns of the committed KV cache are visible to every row (modeling_llama.py:205-206) and are
    not part of this predicate.
    """
    tr, tc = lay.row_type[r], lay.row_type[c]
    if tr == ROW_PAD:
        return r == c
    if tr == ROW_PREFIX:                         # causal prefix (:124-130 prefill, :189-192)
        return tc == ROW_PREFIX and lay.row_idx[c] <= lay.row_idx[r]
    if tr == ROW_WINDOW:
        if tc == ROW_PREFIX:                     # :195
            return True
        if tc == ROW_WINDOW:
            if lay.row_blk[c] == 0:              # level-0 block, causal in the column index (:201)
                return lay.row_idx[c] <= lay.row_idx[r]
            return lay.row_blk[c] <= lay.row_blk[r] and lay.row_idx[c] == lay.row_idx[r]   # :202-203
        return False
    # guess row: the true input token(s) = absolute step columns <= level_offset (:184), whatever
    # their class (on one GPU the input token is column 0 of the level-0 block)
    if c <= lay.level_offset:
        return True
    if tc == ROW_GUESS:                          # :141-181 block-lower-triangular per n-gram
        return lay.row_blk[c] == lay.row_blk[r] and lay.row_idx[c] <= lay.row_idx[r]
    return False


def step_mask(lay: StepLayout) -> np.ndarray:
    """Boolean [q, q] visibility matrix of the step block."""
    q = lay.q_len
    m = np.zeros((q, q), dtype=bool)
    for r in range(q):
        for c in range(q):
            m[r, c] = row_sees(lay, r, c)
    return m


# --------------------------------------------------------------------------------------------
# verification / accept  (lade/decoding.py:1032-1084)
# --------------------------------------------------------------------------------------------
def verify_guesses(first_guess: int, guess_tokens: Sequence[int], guess_results: Sequence[int], N: int):
    """Longest-prefix accept; returns (max_hit, max_hit_idx, hits) as lade/decoding.py:1071-1084."""
    gs = N - 1
    max_hit, max_hit_idx = 0, 0
    hits = [first_guess] + [0] * (gs - 1)
    for eg in range(len(guess_results) // gs):
        egx = eg * gs
        correct = [first_guess] + list(guess_results[egx:egx + gs])
        myguess = list(guess_tokens[egx:egx + gs])
        gg = 0
        for gg in range(len(myguess)):
            if myguess[gg] != correct[gg]:
                break
        if gg > max_hit:
            max_hit, max_hit_idx = gg, eg
            hits[:max_hit + 1] = correct[:max_hit + 1]
    return max_hit, max_hit_idx, hits


# --------------------------------------------------------------------------------------------
# the greedy loop  (lade/decoding.py:697-1259), model abstracted as a callable
# --------------------------------------------------------------------------------------------
@dataclass
class StepTrace:
    ids: List[int]
    pos: List[int]
    level_sizes: List[int]
    guess_tokens: Optional[List[int]]
    kv_len: int
    first_guess: int = -1
    inp_tokens: List[int] = field(default_factory=list)
    guess_results: List[int] = field(default_factory=list)
    hits: List[int] = field(default_factory=list)
    max_hit: int = 0
    max_hit_idx: int = 0
    kv_src: int = -1            # first cache row copied on accept (decoding.py:1156), -1 if none


# StepFn(layout, kv_len) -> (out_tok, inp_toks[window], guess_toks[lguess]) ; the model must append
# the step rows to its KV cache at rows [kv_len, kv_len+q) and keep the first n_input of them.
StepFn = Callable[[StepLayout, int], Tuple[int, List[int], List[int]]]
# CompactFn(dst_row, src_row, n, new_len): move accepted guess rows, then truncate the cache.
CompactFn = Callable[[int, int, int, int], None]


class LocalComm:
    """Single-worker stand-in for the LP collectives (lade/decoding.py:906,1024,1045,1057,1090,1096,1106)."""
    world = 1
    rank = 0

    def broadcast(self, obj, src):
        return obj

    def all_gather(self, obj):
        return [obj]


class TorchDistComm:
    """The same collectives over torch.distributed (gloo on CPU, nccl on GPUs) with object pickling."""

    def __init__(self):
        import torch.distributed as dist
        self.dist = dist
        self.world = dist.get_world_size()
        self.rank = dist.get_rank()

    def broadcast(self, obj, src):
        box = [obj]
        self.dist.broadcast_object_list(box, src=src)
        return box[0]

    def all_gather(self, obj):
        out = [None] * self.world
        self.dist.all_gather_object(out, obj)
        return out


def lp_window_slice(window_len: int, D: int, rank: int):
    """Window columns [ws, we) owned by `rank` (lade/decoding.py:974-977)."""
    split = (window_len + D - 1) // D
    return min(split * rank, window_len), min(split * (rank + 1), window_len)


def step_state(step, lay, kv_len, past_tokens, fill_level, token_map, all_old, out_ids, first_guess, inp_tokens,
               new_tokens, hits, max_hit, max_hit_idx, kv_src, kv_dst, kv_len_new, skip, n_emit, finished, filtered,
               local) -> dict:
    """What ``on_step`` receives after step ``step`` (1-based) has updated the loop state.

    ``past_tokens``, ``token_map``, ``all_old`` and ``out_ids`` are the loop's live objects (read-only; copy what must
    outlive the call).  ``layout`` / ``kv_len`` describe the step's rows and the committed cache before it;
    ``inp_tokens`` are this worker's outputs on the newest window level, ``new_tokens`` the (gathered) row the window
    took from them; ``hits`` / ``max_hit`` / ``max_hit_idx`` the decision every worker applied, and ``local`` =
    (max_hit, max_hit_idx, hits) of this worker's own verification before the LP reduction.  ``kv_src`` (-1: no copy),
    ``kv_dst``, ``kv_len_new`` the cache compaction, ``skip`` the tokens re-fed next step, ``n_emit`` the tokens
    appended to ``out_ids``, ``filtered`` the newest window level after the sampling loop's EOS filter (None when
    no filter ran) and ``finished`` the stop condition."""
    return dict(step=step, layout=lay, kv_len=kv_len, past_tokens=past_tokens, fill_level=fill_level,
                token_map=token_map, all_old=all_old, out_ids=out_ids, first_guess=first_guess,
                inp_tokens=list(inp_tokens), new_tokens=list(new_tokens), hits=list(hits), max_hit=max_hit,
                max_hit_idx=max_hit_idx, kv_src=kv_src, kv_dst=kv_dst, kv_len_new=kv_len_new, skip=skip,
                n_emit=n_emit, finished=bool(finished), filtered=filtered, local=local)


def greedy_lookahead(prompt: Sequence[int], max_new: int, W: int, N: int, G: int, step_fn: StepFn,
                     compact_fn: CompactFn, pool_from_prompt: bool = False,
                     eos_token_id=None, rng: Optional[random.Random] = None,
                     trace: Optional[List[StepTrace]] = None, token_map_out: Optional[dict] = None,
                     comm=None, on_step: Optional[Callable[[dict], None]] = None):
    """Restatement of jacobi_greedy_search_multilevel, incl. lookahead parallelism. Returns (ids, steps).

    `comm` = None/LocalComm for one worker, TorchDistComm under LP (DIST_WORKERS = comm.world).
    `on_step(state)`, if given, is called after every step's state update with the dict ``step_state`` documents.
    """
    assert N >= 3, "LEVEL must be >= 3 (past_tokens[1] must exist, decoding.py:902)"
    comm = comm or LocalComm()
    D, RANK = comm.world, comm.rank
    rng = rng or random
    if isinstance(eos_token_id, int):
        eos_token_id = [eos_token_id]                                                    # :820-821
    all_old = list(prompt)
    init_len = len(all_old)
    out_ids = list(prompt)
    max_length = init_len + max_new
    past_tokens: List[Optional[List[int]]] = [[rng.choice(all_old) for _ in range(W + N - 3)]] + [None] * (N - 2)  # :902
    if D > 1:
        past_tokens = comm.broadcast(past_tokens, 0)                                     # :906
    fill_level = 0
    token_map: Dict[int, list] = token_map_out if token_map_out is not None else {}
    steps = 0
    lst_token = None
    guess_skip_dist = 0
    if pool_from_prompt:
        fill_pool_with_prompt(all_old, token_map, N, G)                                  # :915-916
    kv_len = 0
    first = True
    GS = N - 1
    while True:
        tail = out_ids if first else out_ids[-1 - guess_skip_dist:]                      # :938-942
        lst_id = len(out_ids) - 1
        if past_tokens[N - 2] is not None and lst_token in token_map and G > 0:          # :948
            guess_tokens = [t for tup in token_map[lst_token] for t in tup]
            if D > 1:                                                                    # :956-963
                cnt = (len(guess_tokens) // GS + D - 1) // D
                guess_tokens = guess_tokens[GS * cnt * RANK: GS * cnt * (RANK + 1)]
            if len(guess_tokens) == 0:
                guess_tokens = None
        else:
            guess_tokens = None
        if D > 1:                                                                        # :973-984
            window_len = len(past_tokens[0]) + 1
            ws, we = lp_window_slice(window_len, D, RANK)
            past_inp = [past_tokens[0][: we - 1]] + [t[ws:we] if t is not None else None for t in past_tokens[1:]]
        else:
            past_inp = past_tokens
        lay = build_step_layout(tail, lst_id, past_inp, fill_level, guess_tokens, N, first)
        out_tok, inp_toks, guess_res = step_fn(lay, kv_len)
        steps += 1
        tr = StepTrace(ids=list(lay.ids), pos=list(lay.pos), level_sizes=list(lay.level_sizes),
                       guess_tokens=list(guess_tokens) if guess_tokens is not None else None,
                       kv_len=kv_len, first_guess=out_tok, inp_tokens=list(inp_toks),
                       guess_results=list(guess_res))
        kvcache_len = kv_len + lay.n_input                                               # modeling :1570
        step_len = kv_len + lay.q_len                                                    # modeling :1571
        first_guess = out_tok
        if D > 1:
            first_guess = comm.broadcast(first_guess, 0)                                 # :1024
        max_hit, max_hit_idx = 0, 0
        hits = [first_guess] + [0] * (N - 2)
        local = (max_hit, max_hit_idx, list(hits))
        if past_tokens[1] is None:                                                       # :1038
            past_tokens[0] = past_tokens[0][1:]
            past_tokens[1] = list(inp_toks)
            if D > 1:
                past_tokens[1] = comm.broadcast(past_tokens[1], D - 1)                   # :1045
            new_tokens = past_tokens[1]
            fill_level += 1
        elif past_tokens[N - 2] is None:                                                 # :1049
            for level in range(fill_level + 1):
                past_tokens[level] = past_tokens[level][1:]
            current = list(inp_toks)
            if D > 1:
                current = sum(comm.all_gather(current), [])                              # :1057-1058
            past_tokens[fill_level + 1] = current[1:]
            new_tokens = current
            fill_level += 1
        else:
            if guess_tokens is not None:
                max_hit, max_hit_idx, hits = verify_guesses(first_guess, guess_tokens, guess_res, N)
            local = (max_hit, max_hit_idx, list(hits))
            if D > 1:                                                                    # :1088-1097
                all_hits = comm.all_gather(max_hit)
                max_hit = max(all_hits)
                winner = all_hits.index(max_hit)
                if max_hit > 0:
                    hits = comm.broadcast(hits, winner)
            new_results = list(inp_toks)
            if D > 1:
                new_results = sum(comm.all_gather(new_results), [])                      # :1106-1107
            assert len(past_tokens[N - 2]) == W and len(new_results) == W                # :1114
            new_tokens = new_results
            update_token_map(token_map, lst_token, past_tokens, new_results, N, W, G)    # :1116
            past_tokens[0] = past_tokens[1][1:]                                          # :1120
            for level in range(1, N - 2):
                past_tokens[level] = past_tokens[level + 1][:]
            past_tokens[N - 2] = new_results
        # KV handling (:1145-1163)
        if D > 1 and max_hit > 0:
            guess_skip_dist = max_hit              # accepted tokens are re-fed next step, no KV copy
            compact_fn(kvcache_len, 0, 0, kvcache_len)
            kv_len = kvcache_len
        else:
            guess_skip_dist = 0
            if max_hit > 0:
                src = step_len - len(guess_tokens) + max_hit_idx * GS
                tr.kv_src = src
                compact_fn(kvcache_len, src, max_hit, kvcache_len + max_hit)
            else:
                compact_fn(kvcache_len, 0, 0, kvcache_len)
            kv_len = kvcache_len + max_hit
        lst_token = hits[max_hit]                                                        # :1165
        n_emit = max_hit + 1
        for hit_idx in range(max_hit + 1):                                               # :1168-1177
            if eos_token_id is not None and hits[hit_idx] == eos_token_id[0]:
                all_old.append(hits[hit_idx])
                n_emit = hit_idx + 1
                finished = True
                break
            else:
                all_old.append(hits[max_hit])      # (sic) reference appends the LAST hit each time
                if pool_from_prompt:
                    append_new_generated_pool(all_old[-N:], token_map, N, G)
        else:
            # :1205-1212 -- next_tokens (= first_guess) is also tested against *every* eos id
            finished = eos_token_id is not None and first_guess in eos_token_id
        tr.hits, tr.max_hit, tr.max_hit_idx = list(hits), max_hit, max_hit_idx
        if trace is not None:
            trace.append(tr)
        out_ids = out_ids + hits[:n_emit]                                                # :1196
        first = False
        if on_step is not None:
            on_step(step_state(steps, lay, tr.kv_len, past_tokens, fill_level, token_map, all_old, out_ids,
                               first_guess, inp_toks, new_tokens, hits, max_hit, max_hit_idx, tr.kv_src, kvcache_len,
                               kv_len, guess_skip_dist, n_emit, finished, None, local))
        if finished or len(out_ids) >= max_length:                                       # :1205-1219
            break
    out_ids = out_ids[:max_length]                                                       # :1221-1225
    return out_ids, steps


# --------------------------------------------------------------------------------------------
# the sampling loop  (lade/decoding.py:137-692), single worker
# --------------------------------------------------------------------------------------------
def sample_lookahead(prompt: Sequence[int], max_new: int, W: int, N: int, G: int, model, warper=None,
                     pool_from_prompt: bool = False, eos_token_id=None, rng: Optional[random.Random] = None,
                     trace: Optional[list] = None, on_step: Optional[Callable[[dict], None]] = None):
    """Restatement of jacobi_sample_multilevel.  `model` provides step_fn / compact_fn / last_logits
    (oracle.llama_ref.OracleLlama); `warper(input_ids, scores)` is the HF LogitsProcessorList of
    temperature / top-k / top-p warpers.  Consumes python `random` and the global torch RNG exactly like the
    reference (random.random() per accept test :507, torch.multinomial :462,:472,:533,:545, random.choice in
    filter_window :578-580).  Returns (ids, steps).  `on_step` as in greedy_lookahead."""
    import torch

    rng = rng or random
    if isinstance(eos_token_id, int):
        eos_token_id = [eos_token_id]
    warp = warper if warper is not None else (lambda ids, s: s)
    GS = N - 1
    all_old = list(prompt)
    init_len = len(all_old)
    out_ids = list(prompt)
    max_length = init_len + max_new

    def set_token():
        return rng.choice(all_old)

    past_tokens = [[set_token() for _ in range(W + N - 3)]] + [None] * (N - 2)          # :353
    fill_level = 0
    token_map: Dict[int, list] = {}
    steps = 0
    lst_token = None
    if pool_from_prompt:
        fill_pool_with_prompt(all_old, token_map, N, G)
    kv_len = 0
    first = True
    next_tokens = None
    eos_t = torch.tensor(eos_token_id) if eos_token_id is not None else None
    while True:
        tail = out_ids if first else out_ids[-1:]
        lst_id = len(out_ids) - 1
        if past_tokens[N - 2] is not None and lst_token in token_map and G > 0:         # :394
            guess_tokens = [t for tup in token_map[lst_token] for t in tup]
        else:
            guess_tokens = None
        lay = build_step_layout(tail, lst_id, past_tokens, fill_level, guess_tokens, N, first)
        _, inp_toks, _ = model.step_fn(lay, kv_len)
        logits = model.last_logits
        dev = logits.device
        if eos_t is not None:
            eos_t = eos_t.to(dev)
        input_ids_t = torch.tensor([out_ids], device=dev)
        steps += 1
        q, lg = lay.q_len, lay.n_guess_tok
        kvcache_len = kv_len + lay.n_input
        step_len = kv_len + q
        next_token_scores = warp(input_ids_t, logits[lay.n_input - 1:lay.n_input])      # :445
        max_hit, max_hit_idx = 0, 0
        filtered = None
        if past_tokens[1] is None:                                                       # :458-468
            probs = torch.nn.functional.softmax(next_token_scores, dim=-1)
            next_tokens = torch.multinomial(probs, num_samples=1).squeeze(1)
            hits = [next_tokens.item()]
            past_tokens[0] = past_tokens[0][1:]
            past_tokens[1] = list(inp_toks)
            fill_level += 1
        elif past_tokens[N - 2] is None:                                                 # :469-480
            probs = torch.nn.functional.softmax(next_token_scores, dim=-1)
            next_tokens = torch.multinomial(probs, num_samples=1).squeeze(1)
            hits = [next_tokens.item()]
            for level in range(fill_level + 1):
                past_tokens[level] = past_tokens[level][1:]
            past_tokens[fill_level + 1] = list(inp_toks)[1:]
            fill_level += 1
        else:
            if guess_tokens is not None:                                                 # :484-540
                probs_next = torch.nn.functional.softmax(next_token_scores, dim=-1)[0]
                hits = []
                guess_logits = warp(input_ids_t, logits[q - lg:])
                guess_probs = torch.nn.functional.softmax(guess_logits, dim=-1)
                guess_indices = list(range(lg // GS))
                for idx_in_ngram in range(GS):
                    g_idx = 0
                    is_accept = False
                    while g_idx < len(guess_indices):
                        guess_idx = guess_indices[g_idx]
                        guess_offset = guess_idx * GS
                        draft_guess = guess_tokens[guess_offset + idx_in_ngram]
                        prob_accept = min(1, probs_next[draft_guess].item())
                        sample_prob = rng.random()
                        if sample_prob < prob_accept:
                            hits.append(draft_guess)
                            is_accept = True
                            max_hit_idx = guess_idx
                            guess_indices = [gi for gi in guess_indices
                                             if guess_tokens[gi * GS + idx_in_ngram] == draft_guess]
                            break
                        else:
                            probs_next[draft_guess] = 0
                            probs_next = probs_next / probs_next.sum()
                            g_idx += 1
                    if is_accept:
                        probs_next = guess_probs[guess_offset + idx_in_ngram]
                        continue
                    else:
                        hits.append(torch.multinomial(probs_next, num_samples=1).item())
                        break
                max_hit = len(hits) - 1
            else:                                                                        # :543-546
                probs_next = torch.nn.functional.softmax(next_token_scores, dim=-1)
                next_tokens = torch.multinomial(probs_next, num_samples=1).squeeze(1)
                hits = [next_tokens.item()]
            new_results = list(inp_toks)
            assert len(past_tokens[N - 2]) == W and len(new_results) == W                # :551
            update_token_map(token_map, lst_token, past_tokens, new_results, N, W, G)    # :553
            past_tokens[0] = past_tokens[1][1:]
            for level in range(1, N - 2):
                past_tokens[level] = past_tokens[level + 1][:]
            past_tokens[N - 2] = new_results
            if eos_token_id is not None:                                                 # :578-580
                for idx in range(len(past_tokens[N - 2])):
                    if past_tokens[N - 2][idx] == eos_token_id[0]:
                        past_tokens[N - 2][idx] = set_token()
                filtered = list(past_tokens[N - 2])
        src = -1
        if max_hit > 0:                                                                  # :583-590
            src = step_len - len(guess_tokens) + max_hit_idx * GS
            model.compact_fn(kvcache_len, src, max_hit, kvcache_len + max_hit)
        else:
            model.compact_fn(kvcache_len, 0, 0, kvcache_len)
        kv_len = kvcache_len + max_hit
        lst_token = hits[max_hit]                                                        # :592
        n_emit = max_hit + 1
        for hit_ids in range(max_hit + 1):                                               # :594-603
            if eos_token_id is not None and hits[hit_ids] == eos_token_id[0]:
                all_old.append(hits[hit_ids])
                next_tokens = eos_t
                n_emit = hit_ids + 1
                break
            else:
                all_old.append(hits[hit_ids])
                if pool_from_prompt:
                    append_new_generated_pool(all_old[-N:], token_map, N, G)
        if trace is not None:
            trace.append(dict(ids=list(lay.ids), hits=list(hits), max_hit=max_hit, max_hit_idx=max_hit_idx,
                              guess_tokens=list(guess_tokens) if guess_tokens else None))
        out_ids = out_ids + hits[:n_emit]                                                # :625
        first = False
        finished = False
        if eos_t is not None:                                                            # :636-643
            finished = bool(next_tokens.to(dev).tile(eos_t.shape[0], 1).ne(eos_t.unsqueeze(1)).prod(dim=0).max() == 0)
        if on_step is not None:
            on_step(step_state(steps, lay, kvcache_len - lay.n_input, past_tokens, fill_level, token_map, all_old,
                               out_ids, hits[0], inp_toks, inp_toks, hits, max_hit, max_hit_idx, src, kvcache_len,
                               kv_len, 0, n_emit, finished, filtered, (max_hit, max_hit_idx, list(hits))))
        if finished or len(out_ids) >= max_length:
            break
    return out_ids[:max_length], steps
