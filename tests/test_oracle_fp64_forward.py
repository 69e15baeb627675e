"""The float64 forward of oracle.llama_ref.OracleLlama against HF's own models run in float64 on the CPU.

OracleLlama with float64 weights is the truth that tests/test_gpu_step_fp64.py holds the device step to, so it must be a
float64 forward of the same model HF defines: head_dim from the config (Qwen3 with heads * head_dim != hidden), Qwen3's
per-head q/k RMSNorm in front of RoPE, tied and untied embeddings, GQA.  HF's float64 model is made a float64 forward
by lifting its two fp32 steps (the RMSNorm statistics are taken in fp32, and the eager attention's softmax too): the
RMSNorm classes run the same formula without the cast, and the attention is SDPA, which stays in float64 on the CPU.
Both sides use HF's fp32 RoPE tables.  They agree to about 1e-15 relative; the bound is 1e-10.

Planted errors, each of which must be caught: the q/k norm skipped, head_dim taken as hidden // heads, the softmax
taken in fp32.  The bf16 / fp16 path of the oracle is pinned to the reference's traces elsewhere (test_oracle_golden,
test_oracle_sampling, test_lp_gloo)."""
import functools

import pytest
import torch

from oracle import llama_ref as LR

REL_TOL = 1e-10
P, SPLIT = 40, 29          # causal sequence of P tokens, fed as a prefix of SPLIT rows, then the rest over the cache

CONFIGS = {
    "llama_mha": dict(arch="llama", hidden=256, layers=2, heads=2, kv_heads=2, inter=688, vocab=1024),
    "llama_gqa": dict(arch="llama", hidden=512, layers=2, heads=4, kv_heads=2, inter=688, vocab=1024),
    "llama_d64": dict(arch="llama", hidden=256, layers=2, heads=4, kv_heads=2, inter=688, vocab=1024),
    "qwen3_untied": dict(arch="qwen3", hidden=256, layers=2, heads=4, kv_heads=2, head_dim=128, inter=768, vocab=1024,
                         tie=False),
    "qwen3_tied": dict(arch="qwen3", hidden=256, layers=2, heads=4, kv_heads=2, head_dim=128, inter=768, vocab=1024,
                       tie=True),
}


def _f64_rms_norm_forward(self, hidden_states):
    """LlamaRMSNorm / Qwen3RMSNorm.forward without the fp32 cast."""
    variance = hidden_states.pow(2).mean(-1, keepdim=True)
    return self.weight * (hidden_states * torch.rsqrt(variance + self.variance_epsilon))


def build_hf_f64(c: dict, seed: int = 0):
    """HF model of config `c` in float64 with random weights: projections normal(0, 0.02) (HF's init), every norm weight
    (q/k norms included) uniform in [0.5, 2] so that a norm applied with the wrong weight or not at all shows.
    Returns (model, oracle cfg, weights)."""
    from transformers import LlamaConfig, LlamaForCausalLM, Qwen3Config, Qwen3ForCausalLM
    common = dict(hidden_size=c["hidden"], num_hidden_layers=c["layers"], num_attention_heads=c["heads"],
                  num_key_value_heads=c["kv_heads"], intermediate_size=c["inter"], vocab_size=c["vocab"],
                  max_position_embeddings=512, attention_bias=False, hidden_act="silu", attn_implementation="sdpa",
                  tie_word_embeddings=c.get("tie", False))
    if c["arch"] == "qwen3":
        cfg = Qwen3Config(head_dim=c["head_dim"], rms_norm_eps=1e-6,
                          rope_parameters={"rope_type": "default", "rope_theta": 1e6}, **common)
        cls = Qwen3ForCausalLM
    else:
        cfg = LlamaConfig(rms_norm_eps=1e-5, rope_parameters={"rope_type": "default", "rope_theta": 10000.0}, **common)
        cls = LlamaForCausalLM
    torch.manual_seed(seed)
    model = cls(cfg)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if p.dim() == 1:
                p.copy_(torch.empty(p.shape).uniform_(0.5, 2.0, generator=g))
    model = model.double().eval()
    w = {k: v.detach() for k, v in model.state_dict().items() if "rotary" not in k}
    w.setdefault("lm_head.weight", w["model.embed_tokens.weight"])
    if c.get("tie"):
        assert w["lm_head.weight"].data_ptr() == w["model.embed_tokens.weight"].data_ptr()
    ocfg = dict(hidden=c["hidden"], layers=c["layers"], heads=c["heads"], kv_heads=c["kv_heads"], inter=c["inter"],
                vocab=c["vocab"], max_pos=512, eps=cfg.rms_norm_eps, rope_theta=cfg.rope_parameters["rope_theta"])
    if "head_dim" in c:
        ocfg["head_dim"] = c["head_dim"]
    return model, ocfg, w


@functools.lru_cache(maxsize=None)
def make_case(name: str):
    """(name, oracle cfg, float64 weights, token ids, HF's float64 logits [P, V]) of config `name`."""
    from transformers.models.llama.modeling_llama import LlamaRMSNorm
    from transformers.models.qwen3.modeling_qwen3 import Qwen3RMSNorm
    c = CONFIGS[name]
    model, ocfg, w = build_hf_f64(c)
    ids = torch.randint(0, c["vocab"], (P,), generator=torch.Generator().manual_seed(7))
    mp = pytest.MonkeyPatch()
    mp.setattr(LlamaRMSNorm, "forward", _f64_rms_norm_forward)
    mp.setattr(Qwen3RMSNorm, "forward", _f64_rms_norm_forward)
    try:
        with torch.no_grad():
            ref = model(ids[None]).logits[0]
    finally:
        mp.undo()
    assert ref.dtype == torch.float64
    return name, ocfg, w, ids, ref


@pytest.fixture(params=list(CONFIGS))
def case(request):
    return make_case(request.param)


def oracle_logits(orc: LR.OracleLlama, ids: torch.Tensor) -> torch.Tensor:
    """[P, V] logits of the causal sequence: the first SPLIT rows as one step, the rest as a second step over the
    cache (the path the lookahead steps take)."""
    a = orc.forward_rows(ids[:SPLIT].tolist(), list(range(SPLIT)), torch.tril(torch.ones(SPLIT, SPLIT, dtype=torch.bool)), 0)
    n = P - SPLIT
    b = orc.forward_rows(ids[SPLIT:].tolist(), list(range(SPLIT, P)), torch.tril(torch.ones(n, n, dtype=torch.bool)),
                         SPLIT)
    return torch.cat([a, b])


def rel_err(got: torch.Tensor, ref: torch.Tensor) -> float:
    return ((got - ref).abs().max() / ref.abs().max()).item()


def test_float64_oracle_matches_hf_float64(case):
    name, ocfg, w, ids, ref = case
    orc = LR.OracleLlama(ocfg, w, rope_dtype=torch.float32)
    got = oracle_logits(orc, ids)
    assert got.dtype == torch.float64
    err = rel_err(got, ref)
    print(f"{name}: max |oracle - HF| / max |HF| = {err:.3g}")
    assert err <= REL_TOL
    # the cache holds post-norm, post-RoPE K and V of every row
    assert orc.k_cache[0].shape == (ocfg["kv_heads"], P, orc.D) and orc.k_cache[0].dtype == torch.float64


def test_float64_oracle_needs_an_explicit_rope_table(case):
    _, ocfg, w, _, _ = case
    with pytest.raises(ValueError, match="rope_dtype"):
        LR.OracleLlama(ocfg, w)


def test_planted_softmax_in_fp32_is_caught(case, monkeypatch):
    name, ocfg, w, ids, ref = case

    def fp32_softmax_attention(q, k, v, mask, n_rep=1):
        k, v = k.repeat_interleave(n_rep, dim=0), v.repeat_interleave(n_rep, dim=0)
        s = torch.matmul(q, k.transpose(1, 2)) / q.shape[-1] ** 0.5 + mask
        return torch.matmul(torch.softmax(s, dim=-1, dtype=torch.float32).to(q.dtype), v)
    monkeypatch.setattr(LR, "eager_attention", fp32_softmax_attention)
    err = rel_err(oracle_logits(LR.OracleLlama(ocfg, w, rope_dtype=torch.float32), ids), ref)
    print(f"{name}: softmax in fp32 reaches {err:.3g}")
    assert err > 100 * REL_TOL


@pytest.mark.parametrize("name", ["qwen3_untied", "qwen3_tied"])
def test_planted_qk_norm_skipped_is_caught(name):
    _, ocfg, w, ids, ref = make_case(name)
    orc = LR.OracleLlama(ocfg, w, rope_dtype=torch.float32)
    assert orc.qk_norm
    orc.qk_norm = False
    err = rel_err(oracle_logits(orc, ids), ref)
    print(f"{name}: q/k norm skipped reaches {err:.3g}")
    assert err > 1e-3


def test_planted_head_dim_from_hidden_is_caught():
    """head_dim taken as hidden // heads (the oracle's old rule): on Qwen3 with heads * head_dim != hidden the q/k/v
    projections no longer split into heads of that size, so the forward cannot run at all."""
    _, ocfg, w, ids, _ = make_case("qwen3_untied")
    orc = LR.OracleLlama(ocfg, w, rope_dtype=torch.float32)
    assert orc.D == 128 != ocfg["hidden"] // ocfg["heads"]
    orc.D = ocfg["hidden"] // ocfg["heads"]
    orc.cos, orc.sin = LR.rope_tables(orc.D, 512, ocfg["rope_theta"], torch.float64, "cpu", table_dtype=torch.float32)
    with pytest.raises(RuntimeError):
        oracle_logits(orc, ids)


def test_rope_table_choice():
    """The engine's tables (fp32 math rounded to the model dtype) widened to float64, or the fp32 ones."""
    c16, s16 = LR.rope_tables(128, 64, 1e4, torch.bfloat16, "cpu")
    c64, s64 = LR.rope_tables(128, 64, 1e4, torch.float64, "cpu", table_dtype=torch.bfloat16)
    assert torch.equal(c16.double(), c64) and torch.equal(s16.double(), s64)
    c32, _ = LR.rope_tables(128, 64, 1e4, torch.float32, "cpu")
    c64f, _ = LR.rope_tables(128, 64, 1e4, torch.float64, "cpu", table_dtype=torch.float32)
    assert torch.equal(c32.double(), c64f) and not torch.equal(c64f, c64)


def test_memory_saving_paths_compute_the_same_forward(case, monkeypatch):
    """What lets the float64 oracle run at checkpoint widths changes no value: the embedding and lm_head left in the
    model dtype (only the gathered rows and one vocabulary chunk widened), logits of the asked rows only, and the
    attention over groups of heads (whole GQA groups) when its score block is large."""
    name, ocfg, w, ids, _ = case
    want = oracle_logits(LR.OracleLlama(ocfg, w, rope_dtype=torch.float32), ids)
    narrow = {k: v.to(torch.bfloat16) if k in ("model.embed_tokens.weight", "lm_head.weight") else v
              for k, v in w.items()}
    ref = oracle_logits(LR.OracleLlama(ocfg, {k: v.double() for k, v in narrow.items()}, rope_dtype=torch.float32), ids)
    monkeypatch.setattr(LR.OracleLlama, "LM_CHUNK", 100)                   # several chunks, the last one partial
    monkeypatch.setattr(LR, "F64_SCORE_CHUNK", 300)                        # one GQA group of heads at a time
    orc = LR.OracleLlama(ocfg, narrow, rope_dtype=torch.float32)
    assert orc.dtype == torch.float64
    got = oracle_logits(orc, ids)
    assert rel_err(got, ref) <= REL_TOL and rel_err(ref, want) > REL_TOL    # the narrowed weights do change the model
    rows = [SPLIT - 1, 0, 5]
    part = orc.forward_rows(ids[:SPLIT].tolist(), list(range(SPLIT)), torch.tril(torch.ones(SPLIT, SPLIT, dtype=torch.bool)),
                            0, logit_rows=rows)
    assert part.shape == (3, ocfg["vocab"]) and rel_err(part, ref[rows]) <= REL_TOL
