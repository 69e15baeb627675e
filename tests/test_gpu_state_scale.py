"""The device state machine (state.cu) held to the oracle at production shapes, every step.

The model is ``state_scale.CycleModel``, a deterministic next-token function that accepts often at any vocabulary, so
the float side stays out of the loop.  The oracle (``oracle.lookahead``, pinned to the reference by the CPU suite) runs
first with an ``on_step`` hook; the device is then driven step by step through ``lade_step_layout`` and
``lade_accept_update`` (greedy), ``lade_lp_verify`` / ``lade_lp_commit`` (lookahead parallelism, D contexts on one GPU,
oracle traces from D gloo CPU workers) or ``lade_commit_decision`` (the sampling path, fed the oracle's decisions).
After every step: every meta field, the ids / position ids, the row descriptors and the rowmask bits against the step
mask, the lm rows, q_len <= ``lade_step_rows_bound``, every result slot (and every LP record), and the window through
``lade_ctx_window_snapshot``; the pool (counts and LRU order) at a few steps and at the end, and the output ids through
``lade_ctx_output_ids``.

Shapes: vocabularies of 4096 to 151936, prompts of up to 3000 tokens, W up to 1024, N up to 33 (GS = 32 fills result
slot 47), G up to 4096, hub keys with more than 128 candidates (the winner past candidate 128, ties across the
128-thread rounds of the verification), D in {2, 3, 5, 8, 16}.  Planted faults, made through a view of the device
state, must each fail the check they target."""
import ctypes as C
import random

import numpy as np
import pytest
import torch

import state_scale as SS
from helpers import make_lade_config
from oracle import lookahead as LA

pytestmark = pytest.mark.gpu

S_SKIP = 10


class Checked(AssertionError):
    pass


def _cabi():
    from lookaheaddecoding_b200 import _cabi
    return _cabi, _cabi.load()


def _state_view(ctx):
    """int32 view of a context's device state block and its lade::Dims (csrc/state.cuh)."""
    from test_gpu_sampling_kernel import _DevInts, _Dims
    from lookaheaddecoding_b200._cabi import LadeConfig
    fields = [("cfg", LadeConfig), ("d", _Dims), ("state", C.c_void_p)]
    c = type("_Ctx", (C.Structure,), {"_fields_": fields}).from_address(ctx.value)
    return torch.as_tensor(_DevInts(c.state, int(c.d.total_ints)), device="cuda"), c.d


class Device:
    """D contexts of one configuration (D = 1: no lookahead parallelism) and their step buffers."""

    def __init__(self, W, N, G, V, P, max_length, D=1, pool=True, eos=()):
        self.C, self.lib = _cabi()
        self.W, self.N, self.G, self.V, self.P, self.D = W, N, G, V, P, D
        self.GS, self.WCAP = N - 1, W + N - 3
        self.max_length = max_length
        self.cfgs, self.ctxs = [], []
        for r in range(D):
            cfg = make_lade_config(W, N, G, V, max_length + N + 8, pool=pool, eos=list(eos))
            cfg.dist_workers, cfg.rank = D, r
            ctx = C.c_void_p()
            self.C.check(self.lib.lade_ctx_create(C.byref(cfg), C.byref(ctx)), "create")
            self.cfgs.append(cfg)
            self.ctxs.append(ctx)
        self.stream = torch.cuda.current_stream().cuda_stream
        self.lm_cap = 1 + self.WCAP + G * self.GS
        self.rec_ints = self.lib.lade_lp_record_ints(C.byref(self.cfgs[0]))
        i32 = dict(dtype=torch.int32, device="cuda")
        self.meta = [torch.zeros(self.C.META_INTS, **i32) for _ in range(D)]
        self.res = [torch.zeros(self.C.RES_INTS, **i32) for _ in range(D)]
        self.lm_rows = [torch.zeros(self.lm_cap, **i32) for _ in range(D)]
        self.recs = torch.zeros(D * self.rec_ints, **i32)

    def reset(self, prompt, win0, max_length=None):
        pr = np.asarray(prompt, dtype=np.int32)
        w0 = np.asarray(win0, dtype=np.int32)
        self.P = len(prompt)
        self.max_length = max_length or self.max_length
        for ctx in self.ctxs:
            self.C.check(self.lib.lade_ctx_reset(ctx, self.stream, pr.ctypes.data, len(pr), w0.ctypes.data, self.WCAP,
                                                 self.max_length), "reset")
        torch.cuda.synchronize()

    def close(self):
        for ctx in self.ctxs:
            self.lib.lade_ctx_destroy(ctx)

    # ------------------------------------------------------------------------------------------------ reads
    def window(self, r=0):
        win = np.zeros((self.N - 1) * self.WCAP, dtype=np.int32)
        ln = np.zeros(self.N - 1, dtype=np.int32)
        self.C.check(self.lib.lade_ctx_window_snapshot(self.ctxs[r], self.stream, win.ctypes.data, ln.ctypes.data))
        win = win.reshape(self.N - 1, self.WCAP)
        return [win[l, :ln[l]].tolist() for l in range(self.N - 1)]

    def pool(self, r=0):
        cnt = np.zeros(self.V, dtype=np.int32)
        tup = np.zeros((self.V, max(self.G, 1), self.GS), dtype=np.int32)
        self.C.check(self.lib.lade_ctx_pool_snapshot(self.ctxs[r], self.stream, cnt.ctypes.data, tup.ctypes.data))
        return {int(k): [tuple(x) for x in tup[k, :cnt[k]].tolist()] for k in np.nonzero(cnt)[0]}

    def output_ids(self, n, r=0):
        out = np.zeros(n, dtype=np.int32)
        self.C.check(self.lib.lade_ctx_output_ids(self.ctxs[r], self.stream, out.ctypes.data, n))
        return out.tolist()

    # ------------------------------------------------------------------------------------------------ one step
    def layout(self, r, i, s):
        """lade_step_layout of rank r for step i, checked against the oracle's snapshot s; returns (meta, lm_rows)."""
        Cb = self.C
        q = len(s["ids"])
        bound = self.lib.lade_step_rows_bound(C.byref(self.cfgs[r]), self.P, i)
        _expect(q <= bound, "rows bound", i, f"q_len {q} > lade_step_rows_bound {bound}")
        q_pad = bound
        mw = (q_pad + 31) // 32
        i32 = dict(dtype=torch.int32, device="cuda")
        ids, pos, rd = (torch.full((q_pad,), -9, **i32) for _ in range(3))
        rowmask = torch.full((q_pad * mw,), -1, **i32)
        Cb.check(self.lib.lade_step_layout(self.ctxs[r], self.stream, q_pad, ids.data_ptr(), pos.data_ptr(),
                                           rd.data_ptr(), self.lm_rows[r].data_ptr(), self.meta[r].data_ptr(),
                                           rowmask.data_ptr(), mw), "layout")
        m = self.meta[r].cpu().numpy()
        ls, lg, n_in = s["level_sizes"], s["n_guess_tok"], s["n_input"]
        lo = q - (sum(ls) + 1) - lg
        phase = 0 if s["is_prefill"] else (2 if len(ls) == self.N - 1 else 1)
        want = {Cb.M_Q_LEN: q, Cb.M_KV_LEN: s["kv_len"], Cb.M_N_INPUT: n_in, Cb.M_LEVEL_OFFSET: lo,
                Cb.M_ALL_OFFSET: lo + 1 + ls[0] - ls[-1], Cb.M_TINY: ls[-1], Cb.M_N_LEVELS: len(ls),
                Cb.M_N_GUESS_TOK: lg, Cb.M_IS_PREFILL: int(phase == 0), Cb.M_PHASE: phase, Cb.M_Q_PAD: q_pad,
                Cb.M_DONE: 0, Cb.M_STEP: i}
        got = {k: int(m[k]) for k in want}
        _expect(got == want, "meta", i, f"rank {r}: {got} != {want}")
        _expect(ids[:q].cpu().tolist() == s["ids"], "ids", i, f"rank {r}")
        _expect(pos[:q].cpu().tolist() == s["pos"], "pos", i, f"rank {r}")
        rdh = rd.cpu().numpy().astype(np.int64) & 0xFFFFFFFF
        cls, blk, idx = (rdh >> 30) & 3, (rdh >> 15) & 0x7FFF, rdh & 0x7FFF
        _expect((cls[q:] == LA.ROW_PAD).all(), "rowdesc", i, f"rank {r}: padding rows")
        if phase == 0:          # every prefill row is a causal prefix row
            _expect((cls[:q] == LA.ROW_PREFIX).all() and (idx[:q] == np.arange(q) & 0x7FFF).all(), "rowdesc mask", i,
                    f"rank {r}")
        else:
            want_mask = SS.mask_from_rows(s["cls"], s["blk"], s["idx"], lo)
            got_mask = SS.mask_from_rows(cls[:q], blk[:q], idx[:q], lo)
            _expect(np.array_equal(got_mask, want_mask), "rowdesc mask", i, f"rank {r}")
            wd = rowmask.cpu().numpy().view(np.uint32).reshape(q_pad, mw)
            bits = np.unpackbits(wd.view(np.uint8).reshape(q_pad, mw * 4), axis=-1, bitorder="little").astype(bool)
            _expect(np.array_equal(bits[:q, :q], want_mask), "rowmask", i, f"rank {r}")
            _expect(not bits[q:].any() and not bits[:, q:].any(), "rowmask", i, f"rank {r}: bits past q_len")
        lmr = self.lm_rows[r].cpu().numpy()
        tiny = ls[-1]
        want_lm = np.full(self.lm_cap, n_in - 1)
        want_lm[1:1 + tiny] = np.arange(q - lg - tiny, q - lg)
        want_lm[1 + self.WCAP:1 + self.WCAP + lg] = np.arange(q - lg, q)
        _expect(np.array_equal(lmr, want_lm), "lm_rows", i, f"rank {r}")
        return m, lmr

    def argmax_slots(self, model, s, lmr):
        outs = model.next(s["ids"], s["pos"])
        return torch.from_numpy(outs[lmr].astype(np.int32)).cuda()

    def check_result(self, r, i, s, last, lp=False):
        Cb = self.C
        res = self.res[r].cpu().numpy()
        GS = self.GS
        want = {Cb.R_N_EMIT: s["n_emit"], Cb.R_MAX_HIT: s["max_hit"], Cb.R_MAX_HIT_IDX: 0 if lp else s["max_hit_idx"],
                Cb.R_KV_SRC: s["kv_src"], Cb.R_KV_DST: s["kv_dst"], Cb.R_KV_LEN: s["kv_len_new"],
                Cb.R_DONE: int(last), Cb.R_N_OUT: s["n_out"], Cb.R_STEPS: i + 1,
                Cb.R_N_GUESS: s["n_guess_tok"] // GS}
        got = {k: int(res[k]) for k in want}
        _expect(got == want, "result", i, f"rank {r}: {got} != {want}")
        hits = (list(s["hits"]) + [0] * GS)[:GS]
        _expect(res[Cb.R_HITS:Cb.R_HITS + GS].tolist() == hits, "result hits", i, f"rank {r}")
        _expect(not res[10:Cb.R_HITS].any() and not res[Cb.R_HITS + GS:].any(), "result", i, "unused slots")
        if s["max_hit"] > 0 and s["kv_src"] >= 0:
            _expect(res[Cb.R_KV_SRC] - res[Cb.R_KV_DST] >= res[Cb.R_MAX_HIT], "kv overlap", i, "src - dst < max_hit")

    def check_window(self, i, s, r=0):
        _expect(self.window(r) == s["window"], "window", i, f"rank {r}")

    def check_pool(self, i, pool, r=0):
        got = self.pool(r)
        if got != pool:
            keys = sorted(set(got) | set(pool))
            bad = [k for k in keys if got.get(k) != pool.get(k)]
            what = "pool counts" if any(len(got.get(k, [])) != len(pool.get(k, [])) for k in bad) else "pool LRU order"
            _expect(False, what, i, f"rank {r}: {len(bad)} keys differ, first {bad[:3]}")


def _expect(ok, what, step, detail=""):
    if not ok:
        raise Checked(f"{what} at step {step}: {detail}")


def drive_greedy(dev, model, prompt, win0, snaps, ref_ids, plant=None, max_length=None):
    """Lockstep single-context greedy run against the oracle snapshots; `plant(step, dev)` edits the device state."""
    dev.reset(prompt, win0, max_length)
    results = []
    for i, s in enumerate(snaps):
        m, lmr = dev.layout(0, i, s)
        am = dev.argmax_slots(model, s, lmr)
        dev.C.check(dev.lib.lade_accept_update(dev.ctxs[0], dev.stream, am.data_ptr(), dev.meta[0].data_ptr(),
                                               dev.res[0].data_ptr()), "accept")
        dev.check_result(0, i, s, i == len(snaps) - 1)
        results.append(dev.res[0].cpu().tolist())
        if plant is not None:
            plant(i, dev)
        dev.check_window(i, s)
        if "pool" in s:
            dev.check_pool(i, s["pool"])
    n_out = snaps[-1]["n_out"]
    out = dev.output_ids(min(n_out, dev.max_length + dev.N + 8))
    _expect(out[:dev.max_length] == ref_ids, "output ids", len(snaps))
    return results


def _report(name, st, extra=""):
    print(f"{name}: {st['steps']} steps, {st['accepts']} accepts ({st['full_accepts']} full, {st['accepted_tokens']} "
          f"tokens), {st['evictions']} evictions, largest pool count {st['max_pool_count']}, largest candidate list "
          f"{st['max_candidates']}, largest winning e {st['max_win_e']} (of a key with > 128 candidates: "
          f"{st['max_win_e_of_big_key']}){extra}")


# ---------------------------------------------------------------------------------------------------- greedy cases
@pytest.mark.parametrize("name", SS.CASES)
def test_state_machine_scale(name):
    m, prompt, W, N, G, max_new, eos, seed, mins, ids, snaps, st = SS.oracle_case(name)
    for k, v in mins.items():
        assert st[k] >= v, f"{name}: {k} {st[k]} < {v}: the case no longer exercises what it is for"
    SS.check_hub(name, snaps, st)
    if "eos0" in name:     # eos_token_id[0] inside an accepted n-gram ends the run
        assert snaps[-1]["finished"] and snaps[-1]["n_emit"] >= 2 and snaps[-1]["hits"][snaps[-1]["n_emit"] - 1] == eos[0]
    if "eos1" in name:     # the second eos id stops only as the step's first token (decoding.py:1168-1173, :1205-1212)
        inside = [s for s in snaps if eos[1] in s["hits"][1:s["n_emit"]]]
        assert inside and not snaps[-1]["finished"]
    dev = Device(W, N, G, m.V, len(prompt), len(prompt) + max_new, pool=True, eos=eos or ())
    try:
        drive_greedy(dev, m, prompt, SS.window0(prompt, W + N - 3, seed), snaps, ids)
    finally:
        dev.close()
    _report(name, st, f", WCAP {W + N - 3}, GS {N - 1}")


def test_max_length_inside_a_multi_token_accept():
    m, prompt, W, N, G, max_new, eos, seed, mins, ids, snaps, st = SS.oracle_case("v32000_w7n33g16")
    P = len(prompt)
    cut = next(s for s in snaps if s["n_emit"] >= 4 and s["n_out"] - s["n_emit"] > P + 10)
    new = cut["n_out"] - cut["n_emit"] + 2 - P              # max_length falls two tokens into the accept
    _, _, _, _, _, _, _, _, _, ids2, snaps2, _ = SS.oracle_case("v32000_w7n33g16", max_new=new)
    assert snaps2[-1]["n_out"] > P + new and len(ids2) == P + new
    dev = Device(W, N, G, m.V, P, P + new, pool=True)
    try:
        drive_greedy(dev, m, prompt, SS.window0(prompt, W + N - 3, seed), snaps2, ids2)
    finally:
        dev.close()


def test_context_reuse_matches_a_fresh_context():
    """generate() resets one context per call: a used context must give what a fresh one gives, bit for bit."""
    W, N, G, V = 15, 5, 40, 32000
    ma, mb = SS.CycleModel(V, 21), SS.CycleModel(V, 22, dev_per_mille=150)
    pa, pb = SS.walk_prompt(ma, 900, 21), SS.walk_prompt(mb, 200, 22)
    ida, sa, _ = SS.run_greedy(ma, pa, 300, W, N, G, seed=21)
    idb, sb, stb = SS.run_greedy(mb, pb, 200, W, N, G, seed=22)
    assert stb["accepts"] > 10
    used = Device(W, N, G, V, 900, 1200, pool=True)
    fresh = Device(W, N, G, V, 200, 1200, pool=True)
    try:
        drive_greedy(used, ma, pa, SS.window0(pa, W + N - 3, 21), sa, ida)
        got = drive_greedy(used, mb, pb, SS.window0(pb, W + N - 3, 22), sb, idb, max_length=400)
        want = drive_greedy(fresh, mb, pb, SS.window0(pb, W + N - 3, 22), sb, idb, max_length=400)
        assert got == want
        assert used.pool() == fresh.pool() == sb[-1]["pool"]
        assert used.window() == fresh.window()
    finally:
        used.close()
        fresh.close()


def test_pool_at_the_guess_set_limit():
    """G = 4096 (the largest admitted) at N = 3: one key holds all 4096 continuations of a 64-id vocabulary."""
    V, W, N, G = 64, 4, 3, 4096
    m = SS.CycleModel(V, 34, n_ids=16, dev_per_mille=50)
    hub = int(next(c for c in m.cycles if len(c) % 2)[0])     # odd cycle: two tokens a step still land on the hub
    rnd = random.Random(34)
    pairs = [(a, b) for a in range(V) for b in range(V)]
    rnd.shuffle(pairs)
    prompt = [t for a, b in pairs for t in (hub, a, b)] + m.continuation(hub, 40)
    ids, snaps, st = SS.run_greedy(m, prompt, 40, W, N, G, seed=34, n_pool_checks=1)
    assert st["max_pool_count"] == 4096 and st["max_candidates"] == 4096
    dev = Device(W, N, G, V, len(prompt), len(prompt) + 40, pool=True)
    try:
        drive_greedy(dev, m, prompt, SS.window0(prompt, W + N - 3, 34), snaps, ids)
    finally:
        dev.close()
    _report("v64_w4n3g4096", st)


# ---------------------------------------------------------------------------------------------------- planted faults
def _fault_case():
    m, prompt, W, N, G, max_new, eos, seed, mins, ids, snaps, st = SS.oracle_case("v32000_w7n33g16")
    return m, prompt, W, N, G, max_new, seed, ids, snaps


def _planted(edit):
    m, prompt, W, N, G, max_new, seed, ids, snaps = _fault_case()
    at = next(i for i, s in enumerate(snaps) if "pool" in s and i > 10)
    dev = Device(W, N, G, m.V, len(prompt), len(prompt) + max_new, pool=True)

    def plant(i, d):
        if i == at:
            st, dims = _state_view(d.ctxs[0])
            edit(st, dims, snaps[i])
            torch.cuda.synchronize()
    try:
        with pytest.raises(Checked) as e:
            drive_greedy(dev, m, prompt, SS.window0(prompt, W + N - 3, seed), snaps, ids, plant=plant)
    finally:
        dev.close()
    return str(e.value), at


def test_planted_lru_swap_fails_the_pool_order_check():
    def edit(st, d, s):
        key = next(k for k, v in s["pool"].items() if len(v) >= 2 and v[0] != v[1])
        base = int(d.off_tup) + key * d.G * d.GS
        a, b = st[base:base + d.GS].clone(), st[base + d.GS:base + 2 * d.GS].clone()
        st[base:base + d.GS], st[base + d.GS:base + 2 * d.GS] = b, a
    msg, at = _planted(edit)
    assert msg.startswith(f"pool LRU order at step {at}"), msg


def test_planted_pool_count_fails_the_pool_count_check():
    def edit(st, d, s):
        key = next(k for k, v in s["pool"].items() if len(v) >= 2)
        st[int(d.off_cnt) + key] -= 1
    msg, at = _planted(edit)
    assert msg.startswith(f"pool counts at step {at}"), msg


def test_planted_window_token_fails_the_window_check():
    def edit(st, d, s):
        st[int(d.off_win) + 2 * d.WCAP + 3] += 1        # level 2, column 3
    msg, at = _planted(edit)
    assert msg.startswith(f"window at step {at}"), msg


# ---------------------------------------------------------------------------------------------------- LP
LP_CASES = [  # D, W, N, G, V, prompt, max_new
    (2, 15, 5, 15, 32000, 300, 160),
    (3, 16, 5, 20, 32000, 300, 160),       # window_len % D != 0 at most steps
    (5, 23, 5, 30, 128256, 400, 160),
    (8, 57, 5, 12, 32000, 300, 120),       # fewer n-grams than ranks on some steps
    (16, 61, 5, 8, 4096, 300, 100),        # at most 8 n-grams for 16 ranks
]


def drive_lp(dev, model, prompt, ranks, plant=None):
    D = dev.D
    dev.reset(prompt, ranks[0]["win0"])
    n_steps = ranks[0]["steps"]
    refeeds = 0
    for i in range(n_steps):
        metas = []
        for r in range(D):
            s = ranks[r]["snaps"][i]
            m, lmr = dev.layout(r, i, s)
            am = dev.argmax_slots(model, s, lmr)
            dev.C.check(dev.lib.lade_lp_verify(dev.ctxs[r], dev.stream, am.data_ptr(), dev.meta[r].data_ptr(),
                                               dev.recs[r * dev.rec_ints:].data_ptr()), "lp_verify")
            rec = dev.recs[r * dev.rec_ints:(r + 1) * dev.rec_ints].cpu().tolist()
            lmh, _, lhits = s["local"]
            want = [s["first_guess"], lmh, len(s["inp_tokens"])] + (list(lhits) + [0] * dev.GS)[:dev.GS] + \
                (list(s["inp_tokens"]) + [0] * dev.WCAP)[:dev.WCAP]
            _expect(rec == want, "lp record", i, f"rank {r}")
        for r in range(D):
            dev.C.check(dev.lib.lade_lp_commit(dev.ctxs[r], dev.stream, dev.recs.data_ptr(), dev.meta[r].data_ptr(),
                                               dev.res[r].data_ptr()), "lp_commit")
        for r in range(D):
            s = ranks[r]["snaps"][i]
            dev.check_result(r, i, s, i == n_steps - 1, lp=True)
            dev.check_window(i, s, r)
        refeeds += ranks[0]["snaps"][i]["skip"] > 0
        if plant is not None:
            plant(i, dev)
    for r in range(D):
        dev.check_pool(n_steps, ranks[r]["pool"], r)
        _expect(dev.output_ids(dev.max_length, r) == ranks[r]["ids"], "output ids", n_steps, f"rank {r}")
    return refeeds


def _lp_oracle(D, W, N, G, V, P, max_new, seed=40):
    m = SS.CycleModel(V, seed + D, dev_per_mille=60)
    prompt = SS.walk_prompt(m, P, seed + D)
    spec = dict(V=V, model_seed=seed + D, model_kw=dict(dev_per_mille=60), prompt=prompt, max_new=max_new, W=W, N=N,
                G=G, pool=True, seed=seed)
    ranks = SS.run_lp(spec, D)
    w0 = SS.window0(prompt, W + N - 3, seed)               # rank 0's draws are broadcast (decoding.py:906)
    for rk in ranks:
        rk["win0"] = w0
    return m, prompt, ranks


@pytest.mark.parametrize("D,W,N,G,V,P,max_new", LP_CASES)
def test_lp_state_machine_scale(D, W, N, G, V, P, max_new):
    assert SS.lp_window_ok(W, N, D)
    m, prompt, ranks = _lp_oracle(D, W, N, G, V, P, max_new)
    single, _, _ = SS.run_greedy(m, prompt, max_new, W, N, G, seed=40)
    assert all(rk["ids"] == single for rk in ranks)            # lossless: LP emits the single-worker ids
    snaps = ranks[0]["snaps"]
    consecutive = sum(a["skip"] > 0 and b["skip"] > 0 for a, b in zip(snaps, snaps[1:]))
    starved = sum(any(rk["snaps"][i]["n_guess_tok"] == 0 for rk in ranks) and
                  any(rk["snaps"][i]["n_guess_tok"] for rk in ranks) for i in range(len(snaps)))
    uneven = sum((s["level_sizes"][0] + 1) % D != 0 for s in ranks[-1]["snaps"])   # the last rank's L0 = window_len - 1
    assert consecutive >= 3, "re-fed accepts on consecutive steps"
    if D >= 8:
        assert starved >= 1, "a step where some ranks verify no n-gram"
    dev = Device(W, N, G, V, P, P + max_new, D=D, pool=True)
    try:
        refeeds = drive_lp(dev, m, prompt, ranks)
    finally:
        dev.close()
    print(f"LP D{D} W{W} N{N} G{G} V{V}: {len(snaps)} steps, {refeeds} re-fed accepts ({consecutive} back to back), "
          f"{starved} steps with ranks lacking n-grams, {uneven} steps with window_len % D != 0")


def test_planted_skip_fails_the_lp_meta_check():
    D, W, N, G, V, P, max_new = LP_CASES[0]
    m, prompt, ranks = _lp_oracle(D, W, N, G, V, P, max_new)
    at = next(i for i, s in enumerate(ranks[0]["snaps"]) if s["skip"] > 0 and i + 1 < len(ranks[0]["snaps"]))
    dev = Device(W, N, G, V, P, P + max_new, D=D, pool=True)

    def plant(i, d):
        if i == at:
            st, _ = _state_view(d.ctxs[1])
            st[S_SKIP] += 1
            torch.cuda.synchronize()
    try:
        with pytest.raises(Checked) as e:
            drive_lp(dev, m, prompt, ranks, plant=plant)
    finally:
        dev.close()
    assert str(e.value).startswith(f"meta at step {at + 1}: rank 1"), str(e.value)


# ---------------------------------------------------------------------------------------------------- sampling commit
@pytest.mark.parametrize("seed", [51, 52])
def test_sampling_commit_matches_the_oracle(seed):
    """lade_commit_decision fed each step's oracle decision in the record of sampling.py: result, window and pool."""
    V, W, N, G = 512, 15, 5, 15
    cm = SS.CycleModel(V, seed, n_ids=120, dev_per_mille=80)
    eos = [int(cm.cycles[0][1]), int(cm.cycles[1][1])]
    prompt = SS.walk_prompt(cm, 120, seed)
    ids, snaps = SS.run_sampling(cm, prompt, 200, W, N, G, eos, seed, seed)
    GS, WCAP = N - 1, W + N - 3
    rejects = sum(s["n_guess_tok"] > 0 and s["max_hit"] < GS - 1 for s in snaps)
    distinct_accepts = sum(s["max_hit"] > 0 and len(set(s["hits"][:s["max_hit"] + 1])) > 1 for s in snaps)
    filtered = sum(s["filtered"] is not None and s["filtered"] != s["new_tokens"] for s in snaps)
    assert distinct_accepts >= 5 and rejects >= 5 and filtered >= 1, (distinct_accepts, rejects, filtered)
    dev = Device(W, N, G, V, len(prompt), len(prompt) + 200, pool=True, eos=eos)
    R = dev.rec_ints
    try:
        dev.reset(prompt, SS.window0(prompt, WCAP, seed))
        for i, s in enumerate(snaps):
            dev.layout(0, i, s)
            d = np.zeros(R + 4 + W, dtype=np.int32)
            d[0], d[1], d[2] = s["hits"][0], s["max_hit"], len(s["new_tokens"])
            d[3:3 + min(len(s["hits"]), GS)] = s["hits"][:GS]
            d[3 + GS:3 + GS + len(s["new_tokens"])] = s["new_tokens"]
            d[R], d[R + 1], d[R + 2] = s["max_hit_idx"], 1 | (2 if s["filtered"] is not None else 0), int(s["finished"])
            if s["filtered"] is not None:
                d[R + 4:R + 4 + W] = s["filtered"]
            dd = torch.from_numpy(d).cuda()
            dev.C.check(dev.lib.lade_commit_decision(dev.ctxs[0], dev.stream, dd.data_ptr(), dev.meta[0].data_ptr(),
                                                     dev.res[0].data_ptr()), "commit")
            dev.check_result(0, i, s, i == len(snaps) - 1)
            dev.check_window(i, s)
            dev.check_pool(i, s["pool"])
        _expect(dev.output_ids(len(ids)) == ids, "output ids", len(snaps))
    finally:
        dev.close()
    print(f"sampling V{V} seed {seed}: {len(snaps)} steps, {distinct_accepts} multi-token accepts, {rejects} rejections, "
          f"{filtered} EOS-filtered window rows, finished by EOS: {snaps[-1]['finished']}")
