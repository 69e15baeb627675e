"""The assembled lookahead step at the widths of real checkpoints and at benchmark-length contexts, held to a float64
forward with the lockstep driver and ratio checks of test_gpu_step_fp64 (every used lm slot's logits, the whole
compacted KV cache per layer / K-V / head, the argmax slots; R = 2.5).

The toy models of test_gpu_step_fp64 (hidden 256-512, 2-4 heads, prompts of at most 300 tokens) miss what the engine
does at real widths: the auto-chosen attention split count is 8 there, and nearly uniform attention (scores of std 0.1)
hides cross-tile rescaling and split-merge errors.  Here every model has 2 layers at a checkpoint's true widths (the
step's launches are the same for every layer; two still catch a layer-stride bug), built on the device with the
N(0, 0.02) init (scores of std about 1.6 at hidden 4096), and a prompt of 1024 to 2918 tokens: the engine's splits are
4, 1 and 8, with 3 to 13 KV tiles per split; GQA 4:1, 7:1 and 8:1; vocabularies 32000, 32016, 128256, 151936 and
152064; rope_theta 1e4, 5e5 and 1e6 at positions past 1000; q/k/v biases and q/k norms.

Planted faults at these widths must fail the named check: a window row's position off by one (logits), the RoPE tables
rebuilt with the wrong theta (kv, logits), layer 0's KV heads swapped while its attention runs (a wrong q head -> KV
head map at 7:1: logits, and layer 1's cache, never layer 0's), a compaction from the wrong source row and one that
skips a layer (kv).
"""
import ctypes as C
import gc
import random
import time

import pytest
import torch

import test_gpu_step_fp64 as SF
from qkv_bias_oracle import BiasOracle
from test_gpu_qwen2 import BIAS_STD

pytestmark = pytest.mark.gpu

#                  arch     hidden  q  kv  D    inter   vocab   theta
WIDTHS = {"llama2_7b":     ("llama", 4096, 32, 32, 128, 11008, 32000, 1e4),
          "codellama_13b": ("llama", 5120, 40, 40, 128, 13824, 32016, 1e6),
          "llama3_8b":     ("llama", 4096, 32, 8, 128, 14336, 128256, 5e5),
          "qwen25_7b":     ("qwen2", 3584, 28, 4, 128, 18944, 152064, 1e6),
          "qwen3_8b":      ("qwen3", 4096, 32, 8, 128, 12288, 151936, 1e6),
          "tinyllama":     ("llama", 2048, 32, 4, 64, 5632, 32000, 1e4)}
# impl 3 holds kv_len + q_len <= 3072: at W15 N5 G15 (120 step rows) the largest max_total_len it accepts is
# 3072 - 120 - (N - 3) = 2950, so the prompt is 2950 - 32 tokens
IMPL3_CAP = 2950
NEW = 32
# the periodic model needs more tokens than NEW for its accepts: at N = 4 a step emits at most 3, and the prefill and the
# window-fill step emit one each
PERIODIC_NEW = 64
#                  kind        widths            dtype            W   N   G   P                   new           attn graph
CASES = {"llama2_7b":     ("llama", "llama2_7b", torch.bfloat16, 15, 5, 15, 1024, NEW, 0, True),
         "codellama_13b": ("llama", "codellama_13b", torch.bfloat16, 20, 7, 20, 1536, NEW, 0, False),
         "llama3_8b":     ("llama", "llama3_8b", torch.bfloat16, 15, 5, 15, 2048, NEW, 0, False),
         "qwen25_7b":     ("qwen2", "qwen25_7b", torch.bfloat16, 15, 5, 15, 1024, NEW, 0, False),
         "qwen3_8b":      ("qwen3", "qwen3_8b", torch.bfloat16, 15, 5, 15, IMPL3_CAP - NEW, NEW, 3, True),
         "tinyllama":     ("llama", "tinyllama", torch.float16, 15, 5, 15, 1024, NEW, 0, False),
         "periodic_7b":   ("periodic", "llama2_7b", torch.bfloat16, 7, 4, 7, 1024, PERIODIC_NEW, 0, False)}
# split count the engine picks on a 132-SM H100 (min(8, 132 // (heads * q_tiles)); impl 3: what its capacity needs)
SPLITS = {"llama2_7b": 4, "codellama_13b": 1, "llama3_8b": 4, "qwen25_7b": 4, "qwen3_8b": 8, "tinyllama": 4,
          "periodic_7b": 4}
# "periodic with attention" at hidden 4096 (test_gpu_step_fp64's O_SCALE / LM_SCALE retuned): o_proj and down_proj
# zeroed, then o_proj normal(0, O_SCALE), and lm_head scaled by LM_SCALE.  The next token is then nearly a function of
# the last one.  At hidden 4096 the attention output is large next to the 0.02-sized embedding: O_SCALE = 5e-5 already
# changes the argmax at about 7 % of positions, which breaks the repetition the pool relies on, so O_SCALE is 5e-6
# (about 0.4 %).  The prompt's second half is the model's own greedy continuation of the first half: at vocab 32000 an
# orbit's tail and cycle are about 100 to 200 tokens, so by the end of the prompt the text runs on a cycle the pool
# already holds.  This is the case whose accepts run lade_kv_compact with source rows above 1000: it must reach
# test_gpu_step_fp64's MIN_ACCEPT_STEPS / MIN_FULL_ACCEPTS.
O_SCALE, LM_SCALE = 5e-6, 30.0
MEM_BUDGET = 24 << 30


def _hf_model(name):
    arch, hidden, nh, nkv, D, inter, vocab, theta = WIDTHS[CASES[name][1]]
    dtype = CASES[name][2]
    import transformers as T
    kw = dict(hidden_size=hidden, num_hidden_layers=2, num_attention_heads=nh, num_key_value_heads=nkv,
              intermediate_size=inter, vocab_size=vocab, max_position_embeddings=4096, tie_word_embeddings=False,
              hidden_act="silu", rope_parameters={"rope_type": "default", "rope_theta": theta})
    if arch == "llama":
        cfg = T.LlamaConfig(rms_norm_eps=1e-5, attention_bias=False, **kw)
        cls = T.LlamaForCausalLM
    elif arch == "qwen2":
        cfg = T.Qwen2Config(rms_norm_eps=1e-6, use_sliding_window=False, **kw)
        cls = T.Qwen2ForCausalLM
    else:
        cfg = T.Qwen3Config(rms_norm_eps=1e-6, head_dim=D, attention_bias=False, **kw)
        cls = T.Qwen3ForCausalLM
    # on the device, as bench.build_model: no host copy of a checkpoint-width model
    with torch.device("meta"):
        model = cls(cfg).to(dtype)
    model = model.to_empty(device="cuda")
    g = torch.Generator(device="cuda").manual_seed(0)
    with torch.no_grad():
        for pname, p in model.named_parameters():
            if p.dim() >= 2:
                p.normal_(0.0, 0.02, generator=g)
            elif pname.endswith("_proj.bias"):
                p.normal_(0.0, BIAS_STD, generator=g)                  # as test_gpu_qwen2: HF's zero init hides a bias
            elif pname.endswith("q_norm.weight") or pname.endswith("k_norm.weight"):
                p.uniform_(0.5, 2.0, generator=g)                      # as test_gpu_qwen3
            else:
                p.fill_(1.0)
        re = model.model.rotary_emb                                     # a non-persistent buffer to_empty left unset
        inv = 1.0 / (theta ** (torch.arange(0, D, 2, dtype=torch.float32) / D))
        re.inv_freq = inv.cuda()
        if hasattr(re, "original_inv_freq"):
            re.original_inv_freq = inv.cuda()
        if CASES[name][0] == "periodic":
            for layer in model.model.layers:
                layer.mlp.down_proj.weight.zero_()
                layer.self_attn.o_proj.weight.normal_(0.0, O_SCALE, generator=g)
            model.lm_head.weight.mul_(LM_SCALE)
    model.eval()
    model.generation_config.pad_token_id = 0
    model.generation_config.eos_token_id = None
    return model


_CACHE = {}


def build(name):
    """(HF model, oracle cfg, weights) of case `name`; the previous case's model is released first."""
    if name not in _CACHE:
        _CACHE.clear()
        gc.collect()
        torch.cuda.empty_cache()
        model = _hf_model(name)
        c = model.config
        ocfg = dict(hidden=c.hidden_size, layers=c.num_hidden_layers, heads=c.num_attention_heads,
                    kv_heads=c.num_key_value_heads, inter=c.intermediate_size, vocab=c.vocab_size,
                    max_pos=c.max_position_embeddings, eps=c.rms_norm_eps,
                    rope_theta=c.rope_parameters["rope_theta"], head_dim=WIDTHS[CASES[name][1]][4])
        w = {k: v.detach() for k, v in model.state_dict().items() if "rotary" not in k}
        _CACHE[name] = (model, ocfg, w)
    return _CACHE[name]


def prompt_of(name):
    P = CASES[name][6]
    vocab = WIDTHS[CASES[name][1]][6]
    rnd = torch.randint(3, vocab, (P,), generator=torch.Generator().manual_seed(1)).tolist()
    if CASES[name][0] != "periodic":
        return rnd
    # the second half: the model's own greedy continuation of the first (the engine's argmax of its bf16 logits)
    from lookaheaddecoding_b200 import LookaheadEngine
    _, _, _, W, N, G, _, _, _, _ = CASES[name]
    eng = LookaheadEngine(build(name)[0], W, N, G, pool_from_prompt=True, max_total_len=P)
    out = eng.generate(rnd[:P // 2], P - P // 2, rng=random.Random(5))
    eng.close()
    return out


@pytest.fixture
def wide(monkeypatch):
    """test_gpu_step_fp64's driver with these cases registered, their builder and prompts, and the bias-aware oracle
    (OracleLlama itself on a model without biases)."""
    for name, case in CASES.items():
        monkeypatch.setitem(SF.CASES, name, case)
    monkeypatch.setitem(SF.R_BOUND, "qwen2", 2.5)
    monkeypatch.setattr(SF, "build", build)
    monkeypatch.setattr(SF, "prompt_of", prompt_of)
    monkeypatch.setattr(SF.LR, "OracleLlama", BiasOracle)
    yield
    _CACHE.clear()
    gc.collect()
    torch.cuda.empty_cache()


def _expected_splits(name):
    """SPLITS on a 132-SM H100 (SXM); None on another SM count, where the heuristic's value differs."""
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    if sm != 132:
        print(f"\n{name}: {sm} SMs, not 132: the split count is not checked against SPLITS")
        return None
    return SPLITS[name]


HONEST = {}


@pytest.mark.parametrize("name", list(CASES))
def test_step_rows_match_float64_at_checkpoint_widths(wide, name):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    graph = CASES[name][9]
    engines = [SF.make_engine(name, use_cuda_graph=True), SF.make_engine(name, use_cuda_graph=False)] if graph else \
        [SF.make_engine(name, use_cuda_graph=False)]
    want = _expected_splits(name)
    for e in engines:
        assert want is None or e.attn_splits == want, (name, e.attn_splits, want)
        assert e.has_qkv_bias == (CASES[name][0] == "qwen2") and (e.q_norm_w is not None) == (CASES[name][0] == "qwen3")
    rep = SF.run_lockstep(name, engines)
    torch.cuda.synchronize()
    wall, peak = time.perf_counter() - t0, torch.cuda.max_memory_allocated()
    HONEST[name] = rep
    print(f"\n{rep.line()}; splits {engines[0].attn_splits}; peak {peak / 2 ** 30:.1f} GiB; {wall:.0f} s" +
          (f"; graph vs eager: {len(rep.graph_diffs)} differences" if graph else ""))
    for f in rep.failures[:10]:
        print("   ", f)
    for e in engines:
        e.close()
    assert not rep.failures, rep.failures[:10]
    assert not rep.graph_diffs, rep.graph_diffs[:10]
    assert peak <= MEM_BUDGET, f"{name}: peak {peak / 2 ** 30:.1f} GiB"
    if CASES[name][0] == "periodic":
        assert rep.accept_steps >= SF.MIN_ACCEPT_STEPS and rep.full_accepts >= SF.MIN_FULL_ACCEPTS, rep.line()


# ---- planted faults -------------------------------------------------------------------------------------------------
def plant_wide(eng, fault):
    """The faults of test_gpu_step_fp64.plant, and two that need real widths:
    rope_theta: the engine's cos / sin tables rebuilt with theta 1e4 (a checkpoint's rope_theta not picked up);
    gqa_map: layer 0's KV heads 0 and 1 swapped in the cache after RoPE + append and swapped back after attention, so
    the cache ends up right and only the attention reads the wrong KV head for q heads 0 .. 2 * group - 1."""
    if fault == "rope_theta":
        eng.rope_theta = 1e4
        eng._rope_tables()
        return eng
    if fault == "gqa_map":
        rope, attn = eng._rope_append, eng._attention

        def swap(kc, vc):
            lay = SF._layout_now(eng)
            T = lay["kv"] + lay["q"]
            for c in (kc, vc):
                c[[0, 1], :T] = c[[1, 0], :T]

        def rope_swapped(stream, l, qkv, qb, kc, vc, rows):
            n = rope(stream, l, qkv, qb, kc, vc, rows)
            if l == 0:
                swap(kc, vc)
            return n

        def attn_swapped(stream, l, qb, kc, vc, out, rows, prefill):
            n = attn(stream, l, qb, kc, vc, out, rows, prefill)
            if l == 0:
                swap(kc, vc)
            return n
        eng._rope_append, eng._attention = rope_swapped, attn_swapped
        return eng
    return SF.plant(eng, fault)


#            fault         case             checks that must fail
PLANTS = [("pos", "llama2_7b", {"logits"}),
          ("rope_theta", "codellama_13b", {"kv", "logits"}),
          ("gqa_map", "qwen25_7b", {"logits", "kv"}),
          ("kv_shift", "periodic_7b", {"kv"}),
          ("kv_layers", "periodic_7b", {"kv"})]


@pytest.mark.parametrize("fault,name,kinds", PLANTS, ids=[p[0] for p in PLANTS])
def test_planted_fault_fails_the_checks_at_checkpoint_widths(wide, fault, name, kinds):
    eng = plant_wide(SF.make_engine(name, use_cuda_graph=False), fault)
    rep = SF.run_lockstep(name, [eng])
    honest = HONEST.get(name)
    print(f"\nplanted {fault} on {rep.line()}" +
          (f"; honest worst logits {honest.logit_rms:.2f}/{honest.logit_max:.2f} KV {honest.kv_rms:.2f}/"
           f"{honest.kv_max:.2f}" if honest else ""))
    for f in rep.failures[:6]:
        print("   ", f)
    eng.close()
    assert kinds <= rep.kinds(), rep.line()
    if fault == "gqa_map":
        # layer 0's cache itself is right, only its head map is wrong; layer 1's K and V are computed from what that
        # attention returned, so its cache check fails too
        assert not [f for f in rep.failures if f[1] == "kv" and f[2].startswith("layer 0 ")], rep.failures[:6]


# ---- impl 3's kv_bound on the step after the last -------------------------------------------------------------------
def test_step_after_an_overshooting_accept_stays_within_the_attention_bound(wide):
    """A final multi-token accept leaves the cache past max_length.  After generations without the surplus step
    (pipeline_host=False), lay out the step that would follow (lade_step_layout only, no attention launch) and check
    its kv_len + q_len against impl 3's bound.  A final accept from max_length - 1 tokens out, which generate() never
    follows with a step, reaches the bound exactly; the surplus step generate() does queue (behind a step from
    max_length - 2 or fewer) stays a row below it, which test_oracle_state_scale checks on the CPU."""
    from lookaheaddecoding_b200 import _cabi
    from lookaheaddecoding_b200._cabi import check
    from lookaheaddecoding_b200.engine import _ptr
    name = "qwen25_7b"                                # accepts on about half of its steps
    _, _, _, W, N, G, P, _, _, _ = CASES[name]
    model = build(name)[0]
    prompt = prompt_of(name)
    from lookaheaddecoding_b200 import LookaheadEngine
    worst = None
    for new in range(NEW - 8, NEW + 1):
        eng = LookaheadEngine(model, W, N, G, pool_from_prompt=True, max_total_len=P + new, attn_impl=3,
                              use_cuda_graph=False, pipeline_host=False)
        out = eng.generate(prompt, new, rng=random.Random(5))
        assert len(out) == P + new
        n_out = int(eng.res[_cabi.R_N_OUT])
        stream = torch.cuda.current_stream().cuda_stream
        rows = eng.lib.lade_step_rows_bound(C.byref(eng._lcfg), P, eng.last_steps)
        check(eng.lib.lade_step_layout(eng._ctx, stream, rows, _ptr(eng.ids), _ptr(eng.pos), _ptr(eng.rowdesc),
                                       _ptr(eng.lm_rows), _ptr(eng.meta), _ptr(eng.rowmask), eng.mask_words),
              "lade_step_layout")
        torch.cuda.synchronize()
        meta = eng.meta.cpu().tolist()
        rows = meta[_cabi.M_KV_LEN] + meta[_cabi.M_Q_LEN]
        assert meta[_cabi.M_DONE] == 1 and meta[_cabi.M_KV_LEN] == n_out - 1
        assert rows <= eng.attn_kv_bound, (new, rows, eng.attn_kv_bound)
        over = n_out - (P + new)
        if worst is None or over > worst[0]:
            worst = (over, rows, eng.attn_kv_bound)
        eng.close()
    print(f"\nlargest overshoot past max_length: {worst[0]} tokens; next step's kv_len + q_len {worst[1]} <= bound "
          f"{worst[2]}")
    assert worst[0] >= 1
