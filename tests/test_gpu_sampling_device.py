"""Sampling verification ON DEVICE (lade_sample_verify + lade_commit_decision inside the step graph).

* exactness: every decision of the kernel (accepted tokens, winning n-gram, residual / plain draw) equals the
  restatement of the reference's control flow (oracle/sampling_device.py, decoding.py:445-546) replayed with the
  uniforms the kernel exported, on logits read back from the device -- a uniform within 1e-6 of its threshold is
  skipped, a draw must be the inverse-CDF token within float rounding;
* distribution: the first sampled token over 1200 seeds follows softmax(logits / T) (chi-square on the top tokens);
* T -> 0 reproduces the greedy ids (accept with probability 1, multi-token steps, KV compaction);
* graph replay == eager launches; the plugin surface routes temperature-only sampling here and is reproducible under
  torch.manual_seed."""
import random

import numpy as np
import pytest
import torch

from oracle import sampling_device as SD

pytestmark = pytest.mark.gpu
TINY = dict(hidden=256, layers=2, heads=2, kv_heads=2, inter=688, vocab=4096, max_pos=2048, rope_theta=10000.0, eps=1e-5)


def peaked_periodic_model(scale=30.0, seed=0):
    """Tiny model whose next token is a function of the last one (o_proj / down_proj zeroed: periodic text, n-gram
    hits) with a peaked output distribution (lm_head scaled), so that candidates really get accepted."""
    from bench import build_model
    m = build_model(TINY, torch.device("cuda"), seed=seed, weights="cyclic")
    with torch.no_grad():
        m.lm_head.weight.mul_(scale)
    return m


def _prompt(n, seed=1, vocab=4096):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(3, vocab, (n,), generator=g).tolist()


@pytest.mark.parametrize("T,top_k,top_p", [(0.7, 0, 1.0), (0.9, 20, 1.0), (1.0, 0, 0.8), (0.8, 50, 0.9)])
def test_device_decisions_match_restatement_given_the_same_uniforms(T, top_k, top_p):
    from lookaheaddecoding_b200 import LookaheadEngine, _cabi
    W, N, G = 7, 4, 7
    GS, WCAP = N - 1, W + N - 3
    model = peaked_periodic_model()
    prompt = _prompt(24)
    # long enough that every parameter set meets multi-token accept steps whatever the GPU's GEMM rounding does to the
    # sampled trajectory
    eng = LookaheadEngine(model, W, N, G, pool_from_prompt=True, max_total_len=24 + 192, use_cuda_graph=False)
    eng.debug_uniforms = torch.zeros(4 + G * GS + W, dtype=torch.float32, device="cuda")
    eng.sample_temperature, eng.sample_top_k, eng.sample_top_p = T, top_k, top_p
    eng.begin(prompt, 24 + 192, (), eng.draw_window(prompt, random.Random(3)))
    eng.rng_state.copy_(torch.tensor([1234, 0], dtype=torch.int64))
    n_accept_steps = n_draws = 0
    for step in range(192):
        eng.run_forward_step(step, 24, commit="sample")
        torch.cuda.synchronize()
        meta = eng.meta.cpu().tolist()
        res = eng.res.cpu().tolist()
        if res[_cabi.R_DONE] and res[_cabi.R_N_EMIT] == 0:
            break
        phase, lg, q_len = meta[_cabi.M_PHASE], meta[_cabi.M_N_GUESS_TOK], meta[_cabi.M_Q_LEN]
        logits = eng.logits.float().cpu().numpy()
        dbg = eng.debug_uniforms.cpu().numpy()
        uniforms = dbg[1:1 + int(dbg[0])].tolist()
        guess_tokens = eng.ids[q_len - lg:q_len].cpu().tolist() if (phase == 2 and lg) else None
        guess_rows = logits[1 + WCAP:1 + WCAP + lg] if guess_tokens else None
        want = SD.verify_given_uniforms(logits[0], guess_rows, guess_tokens, GS, T, uniforms, top_k, top_p)
        n_emit, max_hit = res[_cabi.R_N_EMIT], res[_cabi.R_MAX_HIT]
        hits = res[_cabi.R_HITS:_cabi.R_HITS + max_hit + 1]
        ambiguous = any(c[0] == "accept" and abs(c[1] - c[2]) < 1e-6 for c in want["checks"])
        if ambiguous:
            continue
        assert want["used"] == len(uniforms), f"step {step}: kernel drew {len(uniforms)}, restatement {want['used']}"
        assert want["n_hits"] == max_hit + 1, f"step {step}"
        if want["hits"] is None:                               # plain draw
            (kind, u, probs), = [c for c in want["checks"] if c[0] == "draw"]
            assert SD.draw_is_consistent(u, probs, hits[0]), f"step {step}: plain draw"
            n_draws += 1
        else:
            for k, h in enumerate(want["hits"]):
                if h is None:
                    kind, u, probs = [c for c in want["checks"] if c[0] == "draw"][-1][:3]
                    assert SD.draw_is_consistent(u, probs, hits[k]), f"step {step}: residual draw"
                    n_draws += 1
                else:
                    assert hits[k] == h, f"step {step}: accepted token {k}"
            if max_hit > 0:
                assert res[_cabi.R_MAX_HIT_IDX] == want["max_hit_idx"], f"step {step}"
                n_accept_steps += 1
        if res[_cabi.R_DONE]:
            break
    print(f"T={T} top_k={top_k} top_p={top_p}: steps with accepted candidates: {n_accept_steps}, draws checked: {n_draws}")
    assert n_accept_steps >= 2 and n_draws >= 8
    eng.close()


def test_first_token_follows_the_softmax_distribution():
    from lookaheaddecoding_b200 import LookaheadEngine
    model = peaked_periodic_model(scale=12.0)
    prompt = _prompt(16, seed=5)
    eng = LookaheadEngine(model, 5, 3, 3, max_total_len=16 + 8, use_cuda_graph=False)
    T = 0.9
    n = 1200
    counts = {}
    for s in range(n):
        out = eng.generate(prompt, 1, rng=random.Random(0), sampling={"temperature": T, "seed": s})
        counts[out[-1]] = counts.get(out[-1], 0) + 1
    probs = SD.softmax_T(eng.logits[0].float().cpu().numpy(), T)
    top = np.argsort(-probs)[:8]
    chi2 = 0.0
    for t in top:
        exp = n * probs[t]
        if exp >= 5:
            chi2 += (counts.get(int(t), 0) - exp) ** 2 / exp
    rest_exp = n * (1 - probs[top].sum())
    rest_obs = n - sum(counts.get(int(t), 0) for t in top)
    if rest_exp >= 5:
        chi2 += (rest_obs - rest_exp) ** 2 / rest_exp
    print(f"chi2 over top-8 + rest = {chi2:.2f}; p(top) = {probs[top[:3]]}")
    assert chi2 < 35.0          # 9 cells: P(chi2_8 > 35) ~ 3e-5
    eng.close()


def _in_cycle_prompt(model, n=64):
    """A prompt that is itself a trajectory of the model's next-token map, long enough to have entered its cycle: the
    pool filled from it holds true continuations, so candidates are verified (and accepted) from the first steps on."""
    from lookaheaddecoding_b200 import LookaheadEngine
    eng = LookaheadEngine(model, 5, 3, 0, max_total_len=8 + 400)
    traj = eng.generate(_prompt(8, seed=2), 400, rng=random.Random(0))
    eng.close()
    return traj[-n:]


def _assert_equal_up_to_a_tie(model, a, b, what):
    """a == b, or the first differing position is an exact / 1-ulp bf16 tie of the model's own logits there (bf16 logits
    of a 4096-word vocabulary tie at a few percent of the positions: greedy takes the lowest index, T -> 0 sampling
    either)."""
    n = min(len(a), len(b))
    i = next((k for k in range(n) if a[k] != b[k]), None)
    if i is None:
        assert len(a) == len(b), what
        return None
    with torch.no_grad():
        logits = model(torch.tensor([a[:i]], device="cuda")).logits[0, -1].float()
    top = logits.max().item()
    ulp = 2.0 ** (np.floor(np.log2(abs(top))) - 7)
    assert top - logits[a[i]].item() <= ulp and top - logits[b[i]].item() <= ulp, \
        f"{what}: diverged at {i} without a tie ({logits[a[i]].item()}, {logits[b[i]].item()}, top {top})"
    return i


def test_low_temperature_reproduces_greedy_and_graph_equals_eager():
    from lookaheaddecoding_b200 import LookaheadEngine
    model = peaked_periodic_model(scale=30.0)
    prompt = _in_cycle_prompt(model, 32)
    outs = {}
    for graph in (False, True):
        eng = LookaheadEngine(model, 7, 4, 7, pool_from_prompt=True, max_total_len=32 + 64, use_cuda_graph=graph)
        greedy = eng.generate(prompt, 64, rng=random.Random(1))
        steps_g = eng.last_steps
        cold = eng.generate(prompt, 64, rng=random.Random(1), sampling={"temperature": 0.02, "seed": 7})
        steps_s = eng.last_steps
        warm = eng.generate(prompt, 64, rng=random.Random(1), sampling={"temperature": 0.8, "seed": 7})
        warm2 = eng.generate(prompt, 64, rng=random.Random(1), sampling={"temperature": 0.8, "seed": 7})
        other = eng.generate(prompt, 64, rng=random.Random(1), sampling={"temperature": 0.8, "seed": 8})
        tie = _assert_equal_up_to_a_tie(model, cold, greedy, f"graph={graph}")
        assert steps_g < 64 and steps_s < 64        # multi-token steps happened (candidates accepted with p = 1)
        if tie is None:
            assert steps_s == steps_g
        assert warm == warm2 and warm != other and len(warm) == 32 + 64
        outs[graph] = (cold, warm)
        eng.close()
    assert outs[False] == outs[True]


def test_eos_stops_sampling_and_window_is_filtered():
    from lookaheaddecoding_b200 import LookaheadEngine
    model = peaked_periodic_model(scale=30.0)
    prompt = _prompt(32, seed=2)
    eng = LookaheadEngine(model, 7, 4, 7, pool_from_prompt=True, max_total_len=32 + 64)
    full = eng.generate(prompt, 64, rng=random.Random(1), sampling={"temperature": 0.02, "seed": 7})
    assert len(set(full[32:])) > 21, "test premise: the first 21 generated tokens must contain a fresh one"
    eos = full[32 + 20]
    first = next(i for i in range(32, len(full)) if full[i] == eos)
    cut = eng.generate(prompt, 64, eos_token_ids=[eos], rng=random.Random(1), sampling={"temperature": 0.02, "seed": 7})
    # EOS ends the run at its first occurrence (the emission loop of the commit kernel truncates the hits there,
    # decoding.py:594-603); at T -> 0 the trajectory up to that point is the one of the run without EOS
    gen = cut[32:]
    assert cut[-1] == eos and gen.count(eos) == 1 and len(cut) <= first + 1
    _assert_equal_up_to_a_tie(model, cut, full[:len(cut)], "eos run vs free run")
    eng.close()


def test_generate_do_sample_temperature_only_runs_on_device(monkeypatch):
    import lade
    from lookaheaddecoding_b200 import engine as E
    model = peaked_periodic_model(scale=12.0)
    model.generation_config.pad_token_id = 0
    model.generation_config.eos_token_id = None
    ids = torch.tensor([_prompt(24, seed=4)], device="cuda")
    calls = []
    orig = E.LookaheadEngine.generate

    def spy(self, *a, **k):
        calls.append(k.get("sampling"))
        return orig(self, *a, **k)
    monkeypatch.setattr(E.LookaheadEngine, "generate", spy)
    monkeypatch.setenv("USE_LADE", "1")
    lade.augment_all()
    try:
        lade.config_lade(LEVEL=4, WINDOW_SIZE=7, GUESS_SET_SIZE=7, DEBUG=0, POOL_FROM_PROMPT=True)
        kw = dict(attention_mask=torch.ones_like(ids), max_new_tokens=32, do_sample=True, temperature=0.8, top_k=0, top_p=1.0)
        torch.manual_seed(1)
        a = model.generate(ids, **kw)
        torch.manual_seed(1)
        b = model.generate(ids, **kw)
        torch.manual_seed(2)
        c = model.generate(ids, **kw)
        assert torch.equal(a, b) and not torch.equal(a, c) and a.shape == (1, 24 + 32)
        assert len(calls) == 3 and all(s is not None and abs(s["temperature"] - 0.8) < 1e-6 for s in calls)
        torch.manual_seed(3)
        d = model.generate(ids, attention_mask=torch.ones_like(ids), max_new_tokens=16, do_sample=True, temperature=0.7,
                           top_k=40, top_p=0.9)
        assert d.shape == (1, 24 + 16) and calls[-1]["top_k"] == 40 and abs(calls[-1]["top_p"] - 0.9) < 1e-6
    finally:
        lade.restore_generate()
