"""Qwen2 / Qwen2.5 (Qwen2ForCausalLM) on the lookahead step: tiny random-init models built here, with random q/k/v
projection biases, decoded by LookaheadEngine and compared with HF's own greedy generate().

* ids against HF: every divergence of the engine from HF's greedy ids (eager attention) is a tie within max(3 ulps,
  HF's own self-inconsistency) on HF's teacher-forced logits (baseline.parity.compare_ids, through the helpers of
  test_gpu_qwen3), over 128 tokens per config: head_dim 128 untied, the same with tied embeddings, and head_dim 64; at
  head_dim 128 the engine runs its reference-order attention (attn_impl 3);
* negative control: the same comparison with the bias launch replaced by the plain Llama kernel (on the projection
  rounded to the model dtype, no bias) diverges beyond the tolerance, so the comparison can see a missing bias;
* engine consistency: lookahead == the engine at W1 N3 G0 up to judged ties, graph == eager and pipelined == synchronous
  bit for bit, a second engine on the same model reuses the fused weights and biases, model.generate() under USE_LADE=1
  reaches the engine, and do_sample=True is reproducible by seed and runs the device path;
* refusals: a bias on only some of q/k/v, an o_proj bias (Llama attention_bias=True), MLP biases, a bias of another
  dtype or shape, biases on some layers only, and biases together with Qwen3's q/k norms.
"""
import random

import pytest
import torch

from baseline.parity import compare_ids
from test_gpu_qwen3 import _prompt, hf_greedy, record

pytestmark = pytest.mark.gpu
W, N, G = 15, 5, 15
NEW = 128
BIAS_STD = 0.5
CONFIGS = {
    "d128": dict(hidden=512, heads=4, tie=False),
    "d128_tied": dict(hidden=512, heads=4, tie=True),
    "d64": dict(hidden=256, heads=4, tie=False),
}


def build_qwen2(hidden=512, heads=4, tie=False, seed=0, dtype=torch.bfloat16, **over):
    """2 layers, 2 kv heads; q/k/v biases normal(0, BIAS_STD), different per layer and projection (HF's init zeroes
    them, which would hide a bias that is ignored or misplaced)."""
    from transformers import Qwen2Config, Qwen2ForCausalLM
    kw = dict(hidden_size=hidden, num_hidden_layers=2, num_attention_heads=heads, num_key_value_heads=2,
              intermediate_size=768, vocab_size=151936, max_position_embeddings=4096, rms_norm_eps=1e-6,
              tie_word_embeddings=tie, hidden_act="silu", use_sliding_window=False,
              rope_parameters={"rope_type": "default", "rope_theta": 1e6}, attn_implementation="eager")
    kw.update(over)
    torch.manual_seed(seed)
    model = Qwen2ForCausalLM(Qwen2Config(**kw))
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for layer in model.model.layers:
            for m in (layer.self_attn.q_proj, layer.self_attn.k_proj, layer.self_attn.v_proj):
                m.bias.copy_(torch.randn(m.bias.shape, generator=g) * BIAS_STD)
    model = model.to("cuda", dtype).eval()
    model.generation_config.pad_token_id = 0
    model.generation_config.eos_token_id = None
    return model


def _engine(model, P, **kw):
    from lookaheaddecoding_b200 import LookaheadEngine
    return LookaheadEngine(model, kw.pop("W", W), kw.pop("N", N), kw.pop("G", G), pool_from_prompt=True,
                           max_total_len=P + NEW, **kw)


def _parity_impl(model):
    """The reference-order attention (impl 3) at head_dim 128, else the default."""
    c = model.config
    return 3 if c.hidden_size // c.num_attention_heads == 128 else 0


def _gen(eng):
    return lambda prompt, new: eng.generate(prompt, new, rng=random.Random(0))


def without_bias(eng):
    """`eng` with its bias launch replaced by the plain lade_rope_append on the projection rounded to the model dtype."""
    from lookaheaddecoding_b200._cabi import check
    from lookaheaddecoding_b200.engine import _ptr

    def rope(stream, l, qkv, qb, kc, vc, rows):
        t = qkv.to(eng.dt)
        check(eng.k_rope_append(stream, _ptr(t), _ptr(eng.cos), _ptr(eng.sin), _ptr(eng.pos), _ptr(eng.meta), _ptr(qb),
                                _ptr(kc), _ptr(vc), rows, rows, eng.nh, eng.nkv, eng.D, eng.kv_capacity, eng.table_len),
              "lade_rope_append")
        return 1
    eng._rope_append = rope
    return eng


@pytest.fixture(scope="module", params=list(CONFIGS))
def case(request):
    model = build_qwen2(**CONFIGS[request.param])
    prompt = _prompt(seed=len(request.param) + 20)
    ref, step_logits = hf_greedy(model, prompt)
    yield request.param, model, prompt, ref, record(model, ref, len(prompt), step_logits)
    del model
    torch.cuda.empty_cache()


def test_ids_match_hf_greedy_up_to_ties(case):
    name, model, prompt, ref, stored = case
    eng = _engine(model, len(prompt), attn_impl=_parity_impl(model))
    assert eng.has_qkv_bias and len(eng.b_qkv) == 2 and eng.qkv.dtype == torch.float32
    rep = compare_ids(_gen(eng), ref, len(prompt), stored, tol_ulps=3.0)
    print(f"{name}: {rep['compared_tokens']} tokens, {rep['n_divergences']} divergences, worst "
          f"{rep['worst_candidate_below_top_ulps']} ulps (tol {rep['tol_ulps']}), {eng.last_steps} steps, "
          f"HF self-mismatch {stored.rec['self']['n_self_mismatch']}, "
          f"HF logit gap {stored.rec['self']['worst_logit_gap_ulps']} ulps")
    assert rep["compared_tokens"] >= 128 and rep["ok"], rep
    eng.close()


def test_negative_control_without_the_bias_diverges(case):
    name, model, prompt, ref, stored = case
    eng = without_bias(_engine(model, len(prompt), attn_impl=_parity_impl(model), use_cuda_graph=False))
    rep = compare_ids(_gen(eng), ref, len(prompt), stored, tol_ulps=3.0, max_divergences=8)
    print(f"{name} without the bias: {rep['n_divergences']} divergences, worst {rep['worst_candidate_below_top_ulps']}")
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
        # the fused q/k/v bias of the first engine is reused, and the HF parameters still point into it
        a = model.model.layers[1].self_attn
        nq, nk = a.q_proj.weight.shape[0], a.k_proj.weight.shape[0]
        assert other.b_qkv[1].data_ptr() == la.b_qkv[1].data_ptr() == a.q_proj.bias.data_ptr()
        assert a.k_proj.bias.data_ptr() == la.b_qkv[1][nq:].data_ptr()
        assert a.v_proj.bias.data_ptr() == la.b_qkv[1][nq + nk:].data_ptr()
        other.close()
    la.close()
    g0.close()


def test_plugin_generate_reaches_the_engine(monkeypatch):
    import lade
    from lookaheaddecoding_b200 import engine as E
    model = build_qwen2(seed=3)
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
        assert len(calls) == 1 and calls[0][1] is None and calls[0][0].has_qkv_bias
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
        assert all(e.has_qkv_bias for e, _ in calls[1:])
    finally:
        lade.restore_generate()


def _refused(model, match):
    from lookaheaddecoding_b200 import LadeError, LookaheadEngine
    with pytest.raises(LadeError, match=match):
        LookaheadEngine(model, W, N, G, max_total_len=256)


def test_refusals():
    from transformers import LlamaConfig, LlamaForCausalLM
    from lookaheaddecoding_b200 import LookaheadEngine
    nn = torch.nn
    model = build_qwen2(hidden=256)
    a = model.model.layers[1].self_attn
    good = {n: getattr(a, n).bias for n in ("q_proj", "k_proj", "v_proj")}
    a.k_proj.bias = None
    _refused(model, r"only some of q/k/v \(k_proj")
    a.k_proj.bias = good["k_proj"]
    a.v_proj.bias = nn.Parameter(good["v_proj"].float())
    _refused(model, "v_proj bias")
    a.v_proj.bias = nn.Parameter(good["v_proj"][:-8].clone())
    _refused(model, "v_proj bias")
    a.v_proj.bias = good["v_proj"]
    for n in good:
        setattr(getattr(a, n), "bias", None)
    _refused(model, "1 of 2 layers")
    for n, b in good.items():
        getattr(a, n).bias = b
    a.o_proj.bias = nn.Parameter(torch.zeros(a.o_proj.weight.shape[0], device="cuda", dtype=torch.bfloat16))
    _refused(model, "o_proj has a bias")
    a.o_proj.bias = None
    LookaheadEngine(model, W, N, G, max_total_len=256).close()        # the model as built still runs
    del model
    kw = dict(hidden_size=256, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2, intermediate_size=512,
              vocab_size=1024, hidden_act="silu", rope_parameters={"rope_type": "default", "rope_theta": 1e4})
    llama = LlamaForCausalLM(LlamaConfig(attention_bias=True, **kw)).to("cuda", torch.bfloat16)
    _refused(llama, "o_proj has a bias")
    llama = LlamaForCausalLM(LlamaConfig(mlp_bias=True, **kw)).to("cuda", torch.bfloat16)
    _refused(llama, "MLP bias")
    from test_gpu_qwen3 import build_qwen3
    qwen3 = build_qwen3()
    for layer in qwen3.model.layers:
        for m in (layer.self_attn.q_proj, layer.self_attn.k_proj, layer.self_attn.v_proj):
            m.bias = nn.Parameter(torch.zeros(m.weight.shape[0], device="cuda", dtype=torch.bfloat16))
    _refused(qwen3, "q/k norms")
