"""CPU side of tests/test_gpu_state_scale.py: the oracle's ``on_step`` hook, the fakes and prompt builders, the
oracle-side LP and sampling traces, the vectorised step mask, and the admitted configuration edges of the C-ABI."""
import ctypes as C
import random

import numpy as np
import pytest
import torch

import state_scale as SS
from oracle import lookahead as LA


def _small():
    m = SS.CycleModel(4096, 3, n_ids=120, dev_per_mille=150)
    return m, SS.walk_prompt(m, 160, 3)


@pytest.mark.parametrize("W,N,G,pool,eos", [(15, 5, 15, True, None), (7, 4, 3, False, None), (5, 3, 8, True, 17)])
def test_on_step_leaves_the_greedy_loop_unchanged(W, N, G, pool, eos):
    m, prompt = _small()
    if eos is not None:
        eos = int(m.cycles[0][2])
    plain_trace, hooked_trace, pool_a, pool_b, states = [], [], {}, {}, []
    a = LA.greedy_lookahead(prompt, 150, W, N, G, m.step_fn, lambda *x: None, pool_from_prompt=pool, eos_token_id=eos,
                            rng=random.Random(1), trace=plain_trace, token_map_out=pool_a)
    b = LA.greedy_lookahead(prompt, 150, W, N, G, m.step_fn, lambda *x: None, pool_from_prompt=pool, eos_token_id=eos,
                            rng=random.Random(1), trace=hooked_trace, token_map_out=pool_b,
                            on_step=lambda s: states.append(SS.snapshot(s, ())))
    assert a == b and pool_a == pool_b and [vars(t) for t in plain_trace] == [vars(t) for t in hooked_trace]
    assert len(states) == a[1] and [s["step"] for s in states] == list(range(1, a[1] + 1))
    out = list(prompt)
    for s, nxt, t in zip(states, states[1:] + [None], plain_trace):
        assert s["ids"] == t.ids and s["hits"] == t.hits and s["max_hit"] == t.max_hit and s["kv_src"] == t.kv_src
        out += s["hits"][:s["n_emit"]]
        assert s["n_out"] == len(out)
        if nxt is not None:       # the window / cache left by a step is what the next step is built from
            assert nxt["kv_len"] == s["kv_len_new"] and nxt["n_input"] == 1 + s["skip"]
            lv = nxt["level_sizes"]
            assert sum(lv) == sum(len(s["window"][l]) for l in range(len(lv)))
            assert nxt["ids"][nxt["n_input"]:nxt["n_input"] + sum(lv)] == sum(s["window"][:len(lv)], [])
    assert out[:len(a[0])] == a[0]
    assert states[-1]["finished"] or states[-1]["n_out"] >= len(prompt) + 150


def test_on_step_leaves_the_sampling_loop_unchanged():
    m, prompt = _small()
    pm = SS.PeakedModel(m)
    eos = [int(m.cycles[0][1])]
    torch.manual_seed(5)
    a = LA.sample_lookahead(prompt, 120, 15, 5, 15, pm, pool_from_prompt=True, eos_token_id=eos, rng=random.Random(5))
    torch.manual_seed(5)
    states = []
    b = LA.sample_lookahead(prompt, 120, 15, 5, 15, pm, pool_from_prompt=True, eos_token_id=eos, rng=random.Random(5),
                            on_step=lambda s: states.append(SS.snapshot(s, set(range(1, 1000)))))
    assert a == b and len(states) == a[1]
    for s in states:
        if s["filtered"] is not None:     # the EOS filter replaced exactly the EOS tokens of the row the pool was fed
            assert len(s["filtered"]) == len(s["new_tokens"]) == 15
            assert all((f == t) == (t != eos[0]) for f, t in zip(s["filtered"], s["new_tokens"])), s
            assert s["window"][-1] == s["filtered"]


def test_sampling_traces_exercise_accepts_rejects_and_the_eos_filter():
    for seed in (51, 52):
        V, W, N, G = 512, 15, 5, 15
        cm = SS.CycleModel(V, seed, n_ids=120, dev_per_mille=80)
        eos = [int(cm.cycles[0][1]), int(cm.cycles[1][1])]
        ids, snaps = SS.run_sampling(cm, SS.walk_prompt(cm, 120, seed), 200, W, N, G, eos, seed, seed)
        rejects = sum(s["n_guess_tok"] > 0 and s["max_hit"] < N - 2 for s in snaps)
        multi = sum(s["max_hit"] > 0 and len(set(s["hits"][:s["max_hit"] + 1])) > 1 for s in snaps)
        filtered = sum(s["filtered"] is not None and s["filtered"] != s["new_tokens"] for s in snaps)
        assert multi >= 5 and rejects >= 5 and filtered >= 1, (seed, multi, rejects, filtered)


def test_cycle_model_and_prompts():
    m = SS.CycleModel(151936, 1)
    assert len(set(m.ids.tolist())) == 300 and m.ids.max() > 100000           # scattered over the vocabulary
    toks = np.arange(0, 151936, 7)
    nxt = m.next(toks, toks * 3)
    assert np.isin(nxt, m.ids).all()                                          # every id leads into a cycle id
    cyc = m.cycles[0]
    assert m.continuation(int(cyc[0]), len(cyc))[-1] == int(cyc[0])
    rate = SS.CycleModel(32000, 2, dev_per_mille=100)
    pos = np.arange(20000)
    dev = (rate.next(np.full(20000, rate.cycles[0][0]), pos) != rate.succ[rate.cycles[0][0]]).mean()
    assert 0.07 < dev < 0.13
    hub_m = SS.CycleModel(128256, 2, dev_per_mille=100)
    prompt, ha, hb = SS.hub_prompt(hub_m, 4, 2)
    tm = {}
    LA.fill_pool_with_prompt(prompt, tm, 5, 200)
    assert len(tm[ha]) > 128 and len(tm[hb]) > 128
    c = tuple(hub_m.continuation(ha, 4))
    assert tm[ha].index(c) > 128                                              # the full match sits past candidate 128


@pytest.mark.parametrize("name", SS.CASES)
def test_scale_cases_exercise_their_paths(name):
    m, prompt, W, N, G, max_new, eos, seed, mins, ids, snaps, st = SS.oracle_case(name)
    for k, v in mins.items():
        assert st[k] >= v, (name, k, st[k], v)
    SS.check_hub(name, snaps, st)
    if "eos1" in name:
        assert any(eos[1] in s["hits"][1:s["n_emit"]] for s in snaps) and not snaps[-1]["finished"]


def test_mask_from_rows_is_the_step_mask():
    rnd = random.Random(0)
    m, prompt = _small()
    lays = []
    LA.greedy_lookahead(prompt, 60, 7, 5, 9, m.step_fn, lambda *x: None, pool_from_prompt=True, rng=random.Random(2),
                        on_step=lambda s: lays.append(s["layout"]))
    for D in (2, 3):
        for r in range(D):
            lays.append(LA.layout_from_shape([6, 5, 5, 5], rnd.randint(1, 4), 4 * rnd.randint(0, 5), 4))
    for lay in lays:
        if lay.is_prefill:
            continue
        assert np.array_equal(SS.layout_mask(lay), LA.step_mask(lay))


def test_lp_oracle_traces_over_gloo_are_lossless():
    m = SS.CycleModel(32000, 43, dev_per_mille=60)
    prompt = SS.walk_prompt(m, 200, 43)
    spec = dict(V=32000, model_seed=43, model_kw=dict(dev_per_mille=60), prompt=prompt, max_new=80, W=16, N=5, G=20,
                pool=True, seed=40)
    ranks = SS.run_lp(spec, 3)
    single, _, _ = SS.run_greedy(m, prompt, 80, 16, 5, 20, seed=40)
    assert all(rk["ids"] == single for rk in ranks)
    assert all(rk["pool"] == ranks[0]["pool"] for rk in ranks)               # the pool is replicated
    s0 = ranks[0]["snaps"]
    assert sum(a["skip"] > 0 and b["skip"] > 0 for a, b in zip(s0, s0[1:])) >= 2
    for i in range(len(s0)):
        assert len({tuple(rk["snaps"][i]["hits"]) for rk in ranks}) == 1
        assert len({str(rk["snaps"][i]["window"]) for rk in ranks}) == 1


def test_admitted_edges_of_the_state_config():
    """One past each admitted edge is refused before anything is allocated; the edges themselves are accepted by
    the host-side sizing, and lade_step_rows_bound at D = 64 is the largest row count the oracle's layout reaches."""
    from helpers import make_lade_config
    from lookaheaddecoding_b200 import _cabi
    lib = _cabi.load()
    for (W, N, G, D), rc in [((7, 34, 16, 1), _cabi.LADE_EUNSUPPORTED), ((1025, 3, 8, 1), _cabi.LADE_EUNSUPPORTED),
                             ((7, 5, 4097, 1), _cabi.LADE_EUNSUPPORTED), ((200, 5, 8, 65), _cabi.LADE_EINVAL)]:
        cfg = make_lade_config(W, N, G, 64, 1000)
        cfg.dist_workers, cfg.rank = D, 0
        out = C.c_void_p()
        assert lib.lade_ctx_create(C.byref(cfg), C.byref(out)) == rc and out.value is None, (W, N, G, D)
    W, N, G, D = 1000, 5, 100, 64
    GS = N - 1
    cfg = make_lade_config(W, N, G, 64, 1000)
    cfg.dist_workers = D
    assert lib.lade_lp_record_ints(C.byref(cfg)) == 3 + GS + W + N - 3
    for r in range(D):
        cfg.rank = r
        for k in range(N + 1):
            fill = min(k, N - 2)
            wl = W + N - 2 - fill
            ws, we = LA.lp_window_slice(wl, D, r)
            if k and ws == we:        # a rank without window columns (the oracle cannot lay out its step)
                continue
            levels = [[0] * (we - 1)] + [[0] * (we - ws)] * fill
            per = (G + D - 1) // D
            n_ng = max(0, min(per * (r + 1), G) - per * r) if k >= N - 2 else 0
            tail = [0] * (40 if k == 0 else 1 + (N - 2 if k >= N - 2 else 0))
            lay = LA.build_step_layout(tail, 50, levels + [None] * (N - 2 - fill), fill, [0] * (n_ng * GS) or None, N,
                                       k == 0)
            assert lib.lade_step_rows_bound(C.byref(cfg), 40, k) >= lay.q_len, (r, k)
            if r == 0:
                assert lib.lade_step_rows_bound(C.byref(cfg), 40, k) == lay.q_len, (r, k)


def _next_layout(s, N, G):
    """The rows of the step after the one `s` describes (greedy_lookahead's layout code, one worker): what the step
    generate() queues before it knows that this step ends the generation runs on."""
    past, out = s["past_tokens"], s["out_ids"]
    lst = s["hits"][s["max_hit"]]
    guess = None
    if past[N - 2] is not None and lst in s["token_map"] and G > 0:
        guess = [t for tup in s["token_map"][lst] for t in tup] or None
    return LA.build_step_layout(out[-1 - s["skip"]:], len(out) - 1, past, s["fill_level"], guess, N, False)


def _launched_rows(m, prompt, max_new, W, N, G):
    """kv_len + q_len of every step the engine's pipelined generate() launches, in order, and whether the last one
    is the surplus step: step k + 1 is queued while step k runs unless the tokens out before step k already make step
    k the last (engine.generate's `certainly_last`)."""
    P, states = len(prompt), []

    def on_step(s):
        states.append(dict(rows=s["kv_len"] + s["layout"].q_len, n_out=len(s["out_ids"]), kv_new=s["kv_len_new"],
                           nxt=_next_layout(s, N, G).q_len))

    LA.greedy_lookahead(prompt, max_new, W, N, G, m.step_fn, lambda *a: None, pool_from_prompt=True,
                        rng=random.Random(0), on_step=on_step)
    rows = [s["rows"] for s in states]
    n_out_before_last = states[-2]["n_out"] if len(states) > 1 else P
    surplus = (n_out_before_last - P) + 1 < max_new
    if surplus:
        rows.append(states[-1]["kv_new"] + states[-1]["nxt"])
    return rows, surplus, states[-1]["kv_new"]


def test_reference_order_attention_bound_covers_the_surplus_step():
    """attn_impl=3 traps when kv_len + q_len of a launched step exceeds its kv_bound.  A final multi-token accept
    leaves the cache past max_length, and generate() has already queued one more step on that finished state: the
    engine's bound must cover it.  Driven over every max_new_tokens of a range, on a model that accepts often."""
    from helpers import make_lade_config
    from lookaheaddecoding_b200 import _cabi
    from lookaheaddecoding_b200.engine import attn_kv_bound
    lib = _cabi.load()
    W, N, G = 15, 5, 15
    cfg = make_lade_config(W, N, G, 4096, 4096, pool=True)
    q_nonprefill = max(lib.lade_step_rows_bound(C.byref(cfg), 1, k) for k in range(1, N - 1))
    assert q_nonprefill == 120
    # the model's own continuations are always right, and a prompt of many jumps and foreign ids fills every key's
    # pool to G candidates: every steady step is a full accept of the full 120 rows
    m = SS.CycleModel(4096, 5, n_ids=24, dev_per_mille=0)
    prompt = SS.walk_prompt(m, 600, 5, jump=0.3, foreign=0.3)
    worst_over, worst_kv, n_surplus = -10 ** 9, -10 ** 9, 0
    for max_new in range(30, 50):
        max_length = len(prompt) + max_new
        rows, surplus, kv_last = _launched_rows(m, prompt, max_new, W, N, G)
        assert max(rows) <= attn_kv_bound(max_length, q_nonprefill, N), (max_new, max(rows))
        assert kv_last <= max_length + N - 3, max_new                     # the bound's argument
        n_surplus += surplus
        worst_over = max(worst_over, max(rows) - (max_length + q_nonprefill))
        worst_kv = max(worst_kv, kv_last - max_length)
    # a final full accept from max_length - 1 tokens out leaves kv_len = max_length + N - 3 (no step follows it in
    # generate(), but the bound covers one); from max_length - 2 tokens out, the most that still queues the surplus
    # step, it leaves max_length + N - 4, and the surplus step runs the full 120 rows on that: N - 4 = 1 row past
    # the bound of max_length + q_nonprefill the engine used to pass
    assert n_surplus > 0 and worst_kv == N - 3 and worst_over == N - 4, (n_surplus, worst_kv, worst_over)
