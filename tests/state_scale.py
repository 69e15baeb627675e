"""Fakes and oracle runs for holding the device state machine to ``oracle.lookahead`` at production shapes.

* ``CycleModel``: a deterministic next-token function that accepts often at any vocabulary size.  A few hundred ids
  scattered over the vocabulary form short cycles; every other id leads into one.  A position-hashed deviation at a
  controlled rate (per mille) breaks a continuation now and then, which gives partial accepts, and optional EOS rules
  make a token's successor an EOS id from a position on.
* prompt builders: ``walk_prompt`` (the model's own continuations with random jumps and foreign tokens) and
  ``hub_prompt`` (keys followed by more than 128 distinct continuations, the winning or tying candidates placed on
  both sides of candidate 128).
* ``run_greedy`` / ``run_lp`` / ``run_sampling``: the oracle loop with an ``on_step`` hook that copies what the device
  must equal after every step; ``run_lp`` runs D gloo CPU workers.
* ``mask_from_rows``: the step mask (``LA.row_sees``) vectorised over row classes, for step blocks of thousands of rows.
"""
from __future__ import annotations

import json
import os
import random
import tempfile

import numpy as np

from oracle import lookahead as LA

M32 = (1 << 32) - 1


def _mix(t, p, salt):
    x = (t.astype(np.uint64) * np.uint64(0x9E3779B1) + p.astype(np.uint64) * np.uint64(0x85EBCA77)
         + np.uint64(salt)) & np.uint64(M32)
    x ^= x >> np.uint64(15)
    x = (x * np.uint64(0x2C1B3C6D)) & np.uint64(M32)
    x ^= x >> np.uint64(12)
    return x


class CycleModel:
    """next(tok, pos) over a vocabulary of V ids; see the module docstring."""

    def __init__(self, V, seed, n_ids=300, dev_per_mille=20, eos_rules=(), min_cycle=3, max_cycle=12):
        rng = np.random.default_rng(seed)
        self.V, self.seed, self.rate = V, seed, dev_per_mille
        self.ids = rng.choice(V, size=min(n_ids, V), replace=False).astype(np.int64)
        n = len(self.ids)
        self.succ = self.ids[rng.integers(0, n, size=V)]          # every id leads into the cycle ids
        self.cycles = []
        i = 0
        while i < n:
            L = int(rng.integers(min_cycle, max_cycle + 1))
            cyc = self.ids[i:i + L]
            if len(cyc) < 2:
                self.succ[cyc] = self.cycles[-1][0]
                break
            self.succ[cyc] = np.roll(cyc, -1)
            self.cycles.append(cyc)
            i += L
        self.eos_rules = [tuple(int(x) for x in r) for r in eos_rules]   # (token, first position, eos id)

    def next(self, toks, pos):
        t = np.asarray(toks, dtype=np.int64)
        p = np.asarray(pos, dtype=np.int64)
        out = self.succ[t]
        h = _mix(t, p, self.seed)
        dev = (h % np.uint64(1000)).astype(np.int64) < self.rate
        jump = self.ids[((h >> np.uint64(10)) % np.uint64(len(self.ids))).astype(np.int64)]
        out = np.where(dev, jump, out)
        for tok, p0, e in self.eos_rules:
            out = np.where((t == tok) & (p >= p0), e, out)
        return out

    def continuation(self, tok, n):
        out = []
        for _ in range(n):
            tok = int(self.succ[tok])
            out.append(tok)
        return out

    def step_fn(self, lay, kv_len):
        outs = self.next(lay.ids, lay.pos).tolist()
        q, lg, win = lay.q_len, lay.n_guess_tok, lay.level_sizes[-1]
        return outs[lay.n_input - 1], outs[q - lg - win:q - lg], outs[q - lg:]


def walk_prompt(model, P, seed, jump=0.04, foreign=0.05):
    """P tokens that follow the model, with random jumps to cycle ids and foreign ids from the whole vocabulary."""
    rnd = random.Random(seed)
    tok = int(model.ids[rnd.randrange(len(model.ids))])
    out = [tok]
    while len(out) < P:
        u = rnd.random()
        if u < foreign:
            tok = rnd.randrange(model.V)
        elif u < foreign + jump:
            tok = int(model.ids[rnd.randrange(len(model.ids))])
        else:
            tok = int(model.next([tok], [len(out) - 1])[0])
        out.append(tok)
    return out


def hub_prompt(model, GS, seed, n_cand=170, tail=240):
    """Two hub keys on one cycle, each followed by `n_cand` distinct GS-token continuations, then a walk on the cycle.

    Hub A: the only candidate matching the model's continuation to full length sits at e = 140; shorter matches (two
    tokens) sit at e = 10 and e = 150, on both sides of e = 128.  Hub B: two equal-length matches at e = 20 and e = 150
    (the earliest must win).  Every other candidate matches at most the first token."""
    rnd = random.Random(seed)
    cyc = max(model.cycles, key=len)
    assert len(cyc) >= 6
    hub_a, hub_b = int(cyc[0]), int(cyc[3])
    cyc_set = set(int(x) for x in model.ids)

    def foreign():
        while True:
            t = rnd.randrange(model.V)
            if t not in cyc_set:
                return t

    out = []
    for hub, full, part in ((hub_a, {140}, {10, 150}), (hub_b, {20, 150}, set())):
        c = model.continuation(hub, GS)
        for e in range(n_cand):
            if e in full:
                tup = c[:GS - 1] + ([foreign()] if hub == hub_b else c[GS - 1:])
            elif e in part:
                tup = c[:2] + [foreign() for _ in range(GS - 2)]
            elif e % 2:
                tup = c[:1] + [foreign() for _ in range(GS - 1)]
            else:
                tup = [foreign() for _ in range(GS)]
            out += [hub] + tup
    tok = hub_a
    for i in range(tail):
        out.append(tok)
        tok = int(model.succ[tok])
    return out, hub_a, hub_b


# ---------------------------------------------------------------------------------------------------------- masks
def mask_from_rows(cls, blk, idx, level_offset):
    """LA.row_sees over every (row, column) of a step block, from the row classes / blocks / indices."""
    cls, blk, idx = (np.asarray(a, dtype=np.int64) for a in (cls, blk, idx))
    q = len(cls)
    r_cls, c_cls = cls[:, None], cls[None, :]
    r_blk, c_blk = blk[:, None], blk[None, :]
    r_idx, c_idx = idx[:, None], idx[None, :]
    cols = np.arange(q)[None, :]
    prefix = (c_cls == LA.ROW_PREFIX) & (c_idx <= r_idx)
    window = (c_cls == LA.ROW_PREFIX) | ((c_cls == LA.ROW_WINDOW) & np.where(
        c_blk == 0, c_idx <= r_idx, (c_blk <= r_blk) & (c_idx == r_idx)))
    guess = (cols <= level_offset) | ((c_cls == LA.ROW_GUESS) & (c_blk == r_blk) & (c_idx <= r_idx))
    pad = np.eye(q, dtype=bool)
    return np.select([r_cls == LA.ROW_PREFIX, r_cls == LA.ROW_WINDOW, r_cls == LA.ROW_GUESS], [prefix, window, guess],
                     pad)


def layout_mask(lay):
    return mask_from_rows(lay.row_type, lay.row_blk, lay.row_idx, lay.level_offset)


# ---------------------------------------------------------------------------------------------------------- oracle runs
class CountingPool(dict):
    """token_map that counts LRU evictions: pool_insert assigns a key only when it drops the oldest tuple."""
    evictions = 0

    def __setitem__(self, k, v):
        self.evictions += 1
        super().__setitem__(k, v)


def copy_pool(token_map):
    return {int(k): [tuple(t) for t in v] for k, v in token_map.items() if len(v)}


def snapshot(s, pool_steps):
    lay = s["layout"]
    snap = dict(step=s["step"], ids=list(lay.ids), pos=list(lay.pos), cls=list(lay.row_type), blk=list(lay.row_blk),
                idx=list(lay.row_idx), level_sizes=list(lay.level_sizes), n_input=lay.n_input,
                n_guess_tok=lay.n_guess_tok, is_prefill=lay.is_prefill, kv_len=s["kv_len"],
                window=[list(x) if x is not None else [] for x in s["past_tokens"]],
                inp_tokens=s["inp_tokens"], new_tokens=s["new_tokens"], first_guess=s["first_guess"],
                hits=s["hits"], max_hit=s["max_hit"], max_hit_idx=s["max_hit_idx"], kv_src=s["kv_src"],
                kv_dst=s["kv_dst"], kv_len_new=s["kv_len_new"], skip=s["skip"], n_emit=s["n_emit"],
                n_out=len(s["out_ids"]), finished=s["finished"], filtered=s["filtered"], local=list(s["local"]),
                n_keys_max=max((len(v) for v in s["token_map"].values()), default=0))
    if s["step"] in pool_steps:
        snap["pool"] = copy_pool(s["token_map"])
    return snap


def stats(snaps, GS, evictions):
    acc = [s for s in snaps if s["max_hit"] > 0]
    win = [(s["max_hit_idx"], s["n_guess_tok"] // GS) for s in acc]
    return dict(steps=len(snaps), accepts=len(acc), full_accepts=sum(s["max_hit"] == GS - 1 for s in acc),
                accepted_tokens=sum(s["max_hit"] for s in acc), evictions=evictions,
                max_pool_count=max(s["n_keys_max"] for s in snaps),
                max_candidates=max(s["n_guess_tok"] // GS for s in snaps),
                max_win_e=max((e for e, _ in win), default=-1),
                max_win_e_of_big_key=max((e for e, n in win if n > 128), default=-1))


def window0(prompt, WCAP, seed):
    r = random.Random(seed)
    return [r.choice(prompt) for _ in range(WCAP)]        # the draws of decoding.py:902, in the oracle's order


def run_greedy(model, prompt, max_new, W, N, G, pool=True, eos=None, seed=0, n_pool_checks=3):
    """Oracle greedy run; returns (ids, per-step snapshots, stats).  Pools are copied at a few steps and the last."""
    probe = []
    LA.greedy_lookahead(prompt, max_new, W, N, G, model.step_fn, lambda *a: None, pool_from_prompt=pool,
                        eos_token_id=eos, rng=random.Random(seed), on_step=lambda s: probe.append(s["step"]))
    n = len(probe)
    pool_steps = {max(1, n * k // (n_pool_checks + 1)) for k in range(1, n_pool_checks + 1)} | {n}
    snaps, tm = [], CountingPool()
    ids, steps = LA.greedy_lookahead(prompt, max_new, W, N, G, model.step_fn, lambda *a: None, pool_from_prompt=pool,
                                     eos_token_id=eos, rng=random.Random(seed), token_map_out=tm,
                                     on_step=lambda s: snaps.append(snapshot(s, pool_steps)))
    assert steps == n == len(snaps)
    return ids, snaps, stats(snaps, N - 1, tm.evictions)


# ---------------------------------------------------------------------------------------------------------- greedy cases
def case(name):
    """(model, prompt, W, N, G, max_new, eos, seed, minimum stats)."""
    if name == "v151936_w60n8g60_p3000":
        m = CycleModel(151936, 1, dev_per_mille=300)
        return m, walk_prompt(m, 3000, 1), 60, 8, 60, 500, None, 1, dict(accepts=60, full_accepts=8, evictions=1)
    if name.startswith("v128256_w15n5g200_hub"):
        seed = int(name[-1])
        m = CycleModel(128256, seed, dev_per_mille=100)
        prompt, _, _ = hub_prompt(m, 4, seed)
        return m, prompt, 15, 5, 200, 500, None, seed, dict(accepts=60, full_accepts=30, max_candidates=129)
    if name == "v32000_w7n33g16":
        m = CycleModel(32000, 11)
        return m, walk_prompt(m, 500, 11), 7, 33, 16, 300, None, 11, dict(accepts=20, full_accepts=1, evictions=20)
    if name == "v4096_w1024n3g8":
        m = CycleModel(4096, 12)
        return m, walk_prompt(m, 1500, 12), 1024, 3, 8, 200, None, 12, dict(accepts=50, full_accepts=50,
                                                                              evictions=100)
    if name.startswith("v4096_w129n5g300_eos"):
        m0 = CycleModel(4096, 13)
        prompt = walk_prompt(m0, 1500, 13)
        ids, _, _ = run_greedy(m0, prompt, 400, 129, 5, 300, seed=13)
        e0, e1 = [t for t in range(4096) if t not in set(m0.ids.tolist())][:2]
        x = ids[1600]         # from position 1600 on, the token generated there is followed by an EOS id
        m = CycleModel(4096, 13, eos_rules=[(x, 1600, e0 if name.endswith("0") else e1)])
        return m, prompt, 129, 5, 300, 400, [e0, e1], 13, dict(accepts=10, full_accepts=5)
    raise KeyError(name)


CASES = ["v151936_w60n8g60_p3000", "v128256_w15n5g200_hub2", "v128256_w15n5g200_hub5", "v32000_w7n33g16",
         "v4096_w1024n3g8", "v4096_w129n5g300_eos0", "v4096_w129n5g300_eos1"]


def check_hub(name, snaps, st):
    """hub2: a key with more than 128 candidates is won past e = 128.  hub5: two full-length matches at e ~ 20 and
    e ~ 150 tie across the 128-thread rounds of the verification, and the earlier one wins."""
    if name.endswith("hub2"):
        assert st["max_win_e_of_big_key"] > 128
    if name.endswith("hub5"):
        assert any(s["n_guess_tok"] // 4 > 128 and s["max_hit"] == 3 and s["max_hit_idx"] < 128 for s in snaps)


def oracle_case(name, max_new=None):
    m, prompt, W, N, G, mx, eos, seed, mins = case(name)
    max_new = max_new or mx
    ids, snaps, st = run_greedy(m, prompt, max_new, W, N, G, eos=eos, seed=seed)
    return m, prompt, W, N, G, max_new, eos, seed, mins, ids, snaps, st


# ---------------------------------------------------------------------------------------------------------- LP (gloo)
def _lp_worker(rank, D, spec, init_file, out_dir):
    import torch
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method=f"file://{init_file}", rank=rank, world_size=D)
    torch.set_num_threads(1)
    model = CycleModel(spec["V"], spec["model_seed"], **spec.get("model_kw", {}))
    snaps, tm = [], CountingPool()
    ids, steps = LA.greedy_lookahead(spec["prompt"], spec["max_new"], spec["W"], spec["N"], spec["G"], model.step_fn,
                                     lambda *a: None, pool_from_prompt=spec["pool"],
                                     rng=random.Random(spec["seed"] + 100 * rank), token_map_out=tm,
                                     comm=LA.TorchDistComm(), on_step=lambda s: snaps.append(snapshot(s, ())))
    pool = copy_pool(tm)
    with open(os.path.join(out_dir, f"{rank}.json"), "w") as f:
        json.dump(dict(ids=ids, steps=steps, snaps=snaps, evictions=tm.evictions,
                       pool={str(k): [list(t) for t in v] for k, v in pool.items()}), f)
    dist.barrier()
    dist.destroy_process_group()


def run_lp(spec, D):
    """D gloo CPU workers run the oracle's LP loop on the same fake model; returns the per-rank records."""
    import torch.multiprocessing as mp
    with tempfile.TemporaryDirectory() as td:
        mp.spawn(_lp_worker, args=(D, spec, os.path.join(td, "init"), td), nprocs=D, join=True)
        out = []
        for r in range(D):
            with open(os.path.join(td, f"{r}.json")) as f:
                rec = json.load(f)
            rec["pool"] = {int(k): [tuple(t) for t in v] for k, v in rec["pool"].items()}
            out.append(rec)
    return out


def lp_window_ok(W, N, D):
    """Every rank owns at least one window column at every step (the window shrinks from W+N-2 to W columns)."""
    return all(LA.lp_window_slice(wl, D, D - 1)[0] < wl and
               all(LA.lp_window_slice(wl, D, r)[1] > LA.lp_window_slice(wl, D, r)[0] for r in range(D))
               for wl in range(W, W + N - 1))


# ---------------------------------------------------------------------------------------------------------- sampling
class PeakedModel:
    """CycleModel whose logits rows peak at next(tok, pos) with a position-hashed height: accepts and rejects."""

    def __init__(self, cm, heights=(2.0, 5.0, 9.0)):
        self.cm, self.heights = cm, np.asarray(heights)
        self.last_logits = None

    def step_fn(self, lay, kv_len):
        import torch
        nxt = self.cm.next(lay.ids, lay.pos)
        h = self.heights[(_mix(np.asarray(lay.ids), np.asarray(lay.pos), 7) % np.uint64(len(self.heights))).astype(np.int64)]
        logits = torch.zeros(len(nxt), self.cm.V, dtype=torch.float32)
        logits[torch.arange(len(nxt)), torch.from_numpy(nxt)] = torch.from_numpy(h).float()
        self.last_logits = logits
        outs = nxt.tolist()
        q, lg, win = lay.q_len, lay.n_guess_tok, lay.level_sizes[-1]
        return outs[lay.n_input - 1], outs[q - lg - win:q - lg], outs[q - lg:]

    def compact_fn(self, *a):
        pass


def run_sampling(cm, prompt, max_new, W, N, G, eos, seed, torch_seed):
    import torch
    torch.manual_seed(torch_seed)
    snaps = []
    every = set(range(1, 10 ** 6))
    ids, steps = LA.sample_lookahead(prompt, max_new, W, N, G, PeakedModel(cm), pool_from_prompt=True,
                                     eos_token_id=eos, rng=random.Random(seed),
                                     on_step=lambda s: snaps.append(snapshot(s, every)))
    return ids, snaps
