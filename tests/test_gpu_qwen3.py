"""Qwen3 (Qwen3ForCausalLM) on the lookahead step: tiny random-init models built here, with random per-head q/k norm
weights, decoded by LookaheadEngine and compared with HF's own greedy generate().

* ids against HF: every divergence of the engine from HF's greedy ids (eager attention) is a tie within max(3 ulps,
  HF's own self-inconsistency: its generate() against its teacher-forced forward on the same positions) on HF's
  teacher-forced logits (baseline.parity.compare_ids), over 128 tokens per config: head_dim 128 with heads * head_dim
  != hidden, the same with tied embeddings, and head_dim 64; at head_dim 128 the engine runs its reference-order
  attention (attn_impl 3);
* negative control: the same comparison with the RoPE stage forced to the plain Llama kernel diverges beyond the
  tolerance, so the comparison can see a missing norm;
* engine consistency: lookahead == the engine at W1 N3 G0 up to judged ties, graph == eager, pipelined == synchronous,
  model.generate() under USE_LADE=1 == engine.generate(), and do_sample=True is reproducible and runs the device path;
* refusals: a sliding-window layer shorter than the engine's capacity, a q_norm over the full width, k_norm missing.
"""
import random

import pytest
import torch

from baseline.parity import StoredReference, compare_ids

pytestmark = pytest.mark.gpu
W, N, G = 15, 5, 15
NEW = 128
CONFIGS = {
    "d128": dict(head_dim=128, tie=False),
    "d128_tied": dict(head_dim=128, tie=True),
    "d64": dict(head_dim=64, tie=False),
}


def build_qwen3(head_dim=128, tie=False, seed=0, dtype=torch.bfloat16, **over):
    """2 layers, hidden 256, 4 q heads, 2 kv heads; q/k norm weights drawn in [0.5, 2], different per layer and per
    norm (HF's default of all ones would hide a swapped or ignored weight)."""
    from transformers import Qwen3Config, Qwen3ForCausalLM
    kw = dict(hidden_size=256, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2, head_dim=head_dim,
              intermediate_size=768, vocab_size=151936, max_position_embeddings=4096, rms_norm_eps=1e-6,
              tie_word_embeddings=tie, attention_bias=False, hidden_act="silu",
              rope_parameters={"rope_type": "default", "rope_theta": 1e6}, attn_implementation="eager")
    kw.update(over)
    cfg = Qwen3Config(**kw)
    torch.manual_seed(seed)
    model = Qwen3ForCausalLM(cfg)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for layer in model.model.layers:
            for m in (layer.self_attn.q_norm, layer.self_attn.k_norm):
                m.weight.copy_(torch.empty(m.weight.shape).uniform_(0.5, 2.0, generator=g))
    model = model.to("cuda", dtype).eval()
    model.generation_config.pad_token_id = 0
    model.generation_config.eos_token_id = None
    return model


def _prompt(n=32, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(3, 151936, (n,), generator=g).tolist()


@torch.no_grad()
def hf_greedy(model, prompt, new=NEW):
    """HF's greedy ids and the logits its generate() computed for each new token ([new, V], fp32)."""
    ids = torch.tensor([prompt], device="cuda")
    out = model.generate(ids, attention_mask=torch.ones_like(ids), max_new_tokens=new, do_sample=False,
                         output_logits=True, return_dict_in_generate=True)
    return out.sequences[0].tolist(), torch.stack(out.logits)[:, 0].float()


@torch.no_grad()
def record(model, ids, n_prompt, step_logits=None, k=16) -> StoredReference:
    """A StoredReference of `ids`: HF's teacher-forced logits (top k per generated position) and HF's self-inconsistency
    in ulps of the top logit: how far `ids` sits below that top and, given the logits HF's own generate() computed for
    the same positions (`step_logits`), how far those two HF forwards put the same top-k candidates apart."""
    x = torch.tensor([ids[:-1]], device="cuda")
    logits = model(x).logits[0, n_prompt - 1:].float()
    top = torch.topk(logits, k, dim=-1)
    want = torch.tensor(ids[n_prompt:], device="cuda")
    t1 = top.values[:, 0]
    ulp = torch.pow(2.0, torch.floor(torch.log2(t1.abs().clamp_min(1e-30))) - 7)
    below = (t1 - logits.gather(1, want[:, None])[:, 0]) / ulp
    gap = 0.0
    if step_logits is not None:
        gap = float(((step_logits.gather(1, top.indices) - top.values).abs().amax(dim=1) / ulp).max())
    rec = {"ids": list(ids), "n_prompt": n_prompt, "topk_ids": top.indices.tolist(), "topk_logits": top.values.tolist(),
           "self": {"positions": int(want.numel()), "n_self_mismatch": int((below > 0).sum()),
                    "worst_logit_gap_ulps": round(gap, 2),
                    "worst_below_top_ulps": round(max(float(below.max()), gap), 2)}}
    return StoredReference(rec, 7)


def _engine(model, P, **kw):
    from lookaheaddecoding_b200 import LookaheadEngine
    return LookaheadEngine(model, kw.pop("W", W), kw.pop("N", N), kw.pop("G", G), pool_from_prompt=True,
                           max_total_len=P + NEW, **kw)


def _parity_impl(model):
    """The reference-order attention (impl 3) where it exists (head_dim 128), else the default."""
    return 3 if model.config.head_dim == 128 else 0


def _gen(eng):
    return lambda prompt, new: eng.generate(prompt, new, rng=random.Random(0))


@pytest.fixture(scope="module", params=list(CONFIGS))
def case(request):
    model = build_qwen3(**CONFIGS[request.param])
    prompt = _prompt(seed=len(request.param))
    ref, step_logits = hf_greedy(model, prompt)
    yield request.param, model, prompt, ref, record(model, ref, len(prompt), step_logits)
    del model
    torch.cuda.empty_cache()


def test_ids_match_hf_greedy_up_to_ties(case):
    """At head_dim 128 the engine runs attn_impl 3, which rounds the attention probabilities after normalising them, in
    the order of HF's eager attention (head_dim 64 has one attention kernel).  The q/k norms give this model scores of
    several units, where one bf16 ulp of a score moves its probability by about 3 %, so the default online softmax's
    different rounding point reaches 4 ulps on a logit of the head_dim 128 model."""
    name, model, prompt, ref, stored = case
    eng = _engine(model, len(prompt), attn_impl=_parity_impl(model))
    assert eng.q_norm_w is not None and len(eng.q_norm_w) == 2
    rep = compare_ids(_gen(eng), ref, len(prompt), stored, tol_ulps=3.0)
    print(f"{name}: {rep['compared_tokens']} tokens, {rep['n_divergences']} divergences, worst "
          f"{rep['worst_candidate_below_top_ulps']} ulps (tol {rep['tol_ulps']}), {eng.last_steps} steps, "
          f"HF self-mismatch {stored.rec['self']['n_self_mismatch']}, "
          f"HF logit gap {stored.rec['self']['worst_logit_gap_ulps']} ulps")
    assert rep["compared_tokens"] >= 128 and rep["ok"], rep
    eng.close()


def test_negative_control_without_the_norms_diverges(case, monkeypatch):
    name, model, prompt, ref, stored = case
    eng = _engine(model, len(prompt), attn_impl=_parity_impl(model))
    monkeypatch.setattr(eng, "q_norm_w", None)          # _rope_append launches the plain lade_rope_append
    rep = compare_ids(_gen(eng), ref, len(prompt), stored, tol_ulps=3.0, max_divergences=8)
    print(f"{name} without q/k norms: {rep['n_divergences']} divergences, worst {rep['worst_candidate_below_top_ulps']}")
    assert not rep["ok"] and rep["worst_candidate_below_top_ulps"] > rep["tol_ulps"]
    eng.close()


def test_engine_paths_agree(case):
    name, model, prompt, ref, stored = case
    P = len(prompt)
    la = _engine(model, P)
    out = la.generate(prompt, NEW, rng=random.Random(0))
    g0 = _engine(model, P, W=1, N=3, G=0)
    plain = g0.generate(prompt, NEW, rng=random.Random(0))
    rep = compare_ids(_gen(la), plain, P, record(model, plain, P), tol_ulps=3.0)
    assert rep["ok"], rep
    for kw in (dict(use_cuda_graph=False), dict(pipeline_host=False)):
        other = _engine(model, P, **kw)
        assert other.generate(prompt, NEW, rng=random.Random(0)) == out, kw
        other.close()
    la.close()
    g0.close()


def test_plugin_generate_reaches_the_engine(monkeypatch):
    import lade
    from lookaheaddecoding_b200 import engine as E
    model = build_qwen3(seed=3)
    prompt = _prompt(seed=9)
    ids = torch.tensor([prompt], device="cuda")
    calls = []
    orig = E.LookaheadEngine.generate

    def spy(self, *a, **k):
        calls.append((self, k.get("sampling")))
        return orig(self, *a, **k)
    monkeypatch.setattr(E.LookaheadEngine, "generate", spy)
    monkeypatch.setenv("USE_LADE", "1")
    lade.augment_all()
    try:
        lade.config_lade(LEVEL=N, WINDOW_SIZE=W, GUESS_SET_SIZE=G, DEBUG=0, POOL_FROM_PROMPT=True)
        random.seed(5)
        got = model.generate(ids, attention_mask=torch.ones_like(ids), max_new_tokens=64, do_sample=False)[0].tolist()
        assert len(calls) == 1 and calls[0][1] is None and calls[0][0].q_norm_w is not None
        eng = _engine(model, len(prompt))
        assert orig(eng, prompt, 64, rng=random.Random(5)) == got
        eng.close()
        kw = dict(attention_mask=torch.ones_like(ids), max_new_tokens=32, do_sample=True, temperature=0.8, top_k=0,
                  top_p=1.0)
        draws = []
        for seed in (1, 1, 2):
            random.seed(seed)
            torch.manual_seed(seed)
            draws.append(model.generate(ids, **kw))
        assert torch.equal(draws[0], draws[1]) and not torch.equal(draws[0], draws[2])
        assert draws[0].shape == (1, len(prompt) + 32)
        assert len(calls) == 4 and all(s is not None and abs(s["temperature"] - 0.8) < 1e-6 for _, s in calls[1:])
        assert all(e.q_norm_w is not None for e, _ in calls[1:])
    finally:
        lade.restore_generate()


def test_refusals():
    from lookaheaddecoding_b200 import LadeError, LookaheadEngine
    # HF makes the layers from max_window_layers onwards sliding
    model = build_qwen3(use_sliding_window=True, sliding_window=64, max_window_layers=1)
    assert "sliding_attention" in model.config.layer_types
    with pytest.raises(LadeError, match="sliding"):
        LookaheadEngine(model, W, N, G, max_total_len=256)
    LookaheadEngine(model, W, N, G, max_total_len=64).close()          # the window covers the whole sequence
    del model
    model = build_qwen3()
    attn = model.model.layers[1].self_attn
    good_q, good_k = attn.q_norm, attn.k_norm
    from transformers.models.qwen3.modeling_qwen3 import Qwen3RMSNorm
    attn.q_norm = Qwen3RMSNorm(4 * 128, eps=1e-6).to("cuda", torch.bfloat16)       # OLMo2-style: over nh * D
    with pytest.raises(LadeError, match="q_norm"):
        LookaheadEngine(model, W, N, G, max_total_len=256)
    attn.q_norm = good_q
    del attn.k_norm
    with pytest.raises(LadeError, match="k_norm"):
        LookaheadEngine(model, W, N, G, max_total_len=256)
    attn.k_norm = good_k
    LookaheadEngine(model, W, N, G, max_total_len=256).close()
