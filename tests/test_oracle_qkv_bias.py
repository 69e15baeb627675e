"""The float64 forward with Qwen2's q/k/v projection biases (tests/qkv_bias_oracle.BiasOracle) against HF's own
Qwen2ForCausalLM run in float64 on the CPU, and the bias term of the float64 projection bound.

HF's init zeroes every Linear bias, so the biases are drawn here, normal(0, 0.5) (large against projections of about 0.3):
a bias dropped, or one added to the wrong slice of q/k/v, moves the logits by far more than the tolerance.  HF's float64
model is made a float64 forward as in test_oracle_fp64_forward (its RMSNorm without the fp32 cast, SDPA attention).
"""
import functools

import pytest
import torch

from oracle import llama_ref as LR
from qkv_bias_oracle import BiasOracle, linear_fp64
from test_oracle_fp64_forward import P, REL_TOL, _f64_rms_norm_forward, oracle_logits, rel_err

CONFIGS = {
    "qwen2_d64_gqa": dict(hidden=256, layers=2, heads=4, kv_heads=2, inter=688, vocab=1024, tie=False),
    "qwen2_d128_tied": dict(hidden=512, layers=2, heads=4, kv_heads=2, inter=688, vocab=1024, tie=True),
}


def build_qwen2_f64(c: dict, seed: int = 0):
    """(HF float64 Qwen2ForCausalLM, oracle cfg, weights): norm weights uniform in [0.5, 2], q/k/v biases normal(0, 0.5),
    different per layer and per projection."""
    from transformers import Qwen2Config, Qwen2ForCausalLM
    cfg = Qwen2Config(hidden_size=c["hidden"], num_hidden_layers=c["layers"], num_attention_heads=c["heads"],
                      num_key_value_heads=c["kv_heads"], intermediate_size=c["inter"], vocab_size=c["vocab"],
                      max_position_embeddings=512, rms_norm_eps=1e-6, hidden_act="silu", attn_implementation="sdpa",
                      rope_parameters={"rope_type": "default", "rope_theta": 1e6}, tie_word_embeddings=c["tie"],
                      use_sliding_window=False)
    torch.manual_seed(seed)
    model = Qwen2ForCausalLM(cfg)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if name.endswith("bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.5)
            elif p.dim() == 1:
                p.copy_(torch.empty(p.shape).uniform_(0.5, 2.0, generator=g))
    model = model.double().eval()
    w = {k: v.detach() for k, v in model.state_dict().items() if "rotary" not in k}
    w.setdefault("lm_head.weight", w["model.embed_tokens.weight"])
    ocfg = dict(hidden=c["hidden"], layers=c["layers"], heads=c["heads"], kv_heads=c["kv_heads"], inter=c["inter"],
                vocab=c["vocab"], max_pos=512, eps=cfg.rms_norm_eps, rope_theta=1e6)
    return model, ocfg, w


@functools.lru_cache(maxsize=None)
def make_case(name: str):
    from transformers.models.qwen2.modeling_qwen2 import Qwen2RMSNorm
    model, ocfg, w = build_qwen2_f64(CONFIGS[name])
    ids = torch.randint(0, ocfg["vocab"], (P,), generator=torch.Generator().manual_seed(7))
    mp = pytest.MonkeyPatch()
    mp.setattr(Qwen2RMSNorm, "forward", _f64_rms_norm_forward)
    try:
        with torch.no_grad():
            ref = model(ids[None]).logits[0]
    finally:
        mp.undo()
    return ocfg, w, ids, ref


@pytest.fixture(params=list(CONFIGS))
def case(request):
    return make_case(request.param)


def test_model_has_the_biases_qwen2_has():
    _, _, w = build_qwen2_f64(CONFIGS["qwen2_d64_gqa"])
    for proj in ("q_proj", "k_proj", "v_proj"):
        b = w[f"model.layers.1.self_attn.{proj}.bias"]
        assert b.abs().min() > 0
    assert "model.layers.0.self_attn.o_proj.bias" not in w and not any("mlp" in k and "bias" in k for k in w)


def test_float64_bias_oracle_matches_hf_float64(case):
    ocfg, w, ids, ref = case
    orc = BiasOracle(ocfg, w, rope_dtype=torch.float32)
    assert orc.qkv_bias
    err = rel_err(oracle_logits(orc, ids), ref)
    print(f"max |oracle - HF| / max |HF| = {err:.3g}")
    assert err <= REL_TOL


@pytest.mark.parametrize("proj", ["q_proj", "k_proj", "v_proj"])
def test_planted_bias_missing_or_misplaced_is_caught(case, proj):
    """One projection's bias dropped, or swapped between the two kv heads, moves the logits far beyond the bound."""
    ocfg, w, ids, ref = case
    D = ocfg["hidden"] // ocfg["heads"]
    for how in ("zero", "swap"):
        w2 = dict(w)
        key = f"model.layers.0.self_attn.{proj}.bias"
        b = w[key].clone()
        if how == "zero":
            b.zero_()
        else:
            b[:D], b[D:2 * D] = w[key][D:2 * D].clone(), w[key][:D].clone()
        w2[key] = b
        err = rel_err(oracle_logits(BiasOracle(ocfg, w2, rope_dtype=torch.float32), ids), ref)
        print(f"{proj} bias {how}: {err:.3g}")
        assert err > 1e-4


def test_without_biases_it_is_the_oracle():
    """The same weights without the biases: BiasOracle gives OracleLlama's values, bit for bit, in float64 and bf16."""
    _, ocfg, w = build_qwen2_f64(CONFIGS["qwen2_d64_gqa"])
    w = {k: v for k, v in w.items() if not k.endswith("bias")}
    ids = torch.randint(0, ocfg["vocab"], (P,), generator=torch.Generator().manual_seed(3))
    for dt, rope_dtype in ((torch.float64, torch.float32), (torch.bfloat16, None)):
        wd = {k: v.to(dt) for k, v in w.items()}
        a = oracle_logits(BiasOracle(ocfg, wd, rope_dtype=rope_dtype), ids)
        b = oracle_logits(LR.OracleLlama(ocfg, wd, rope_dtype=rope_dtype), ids)
        assert torch.equal(a, b), dt


def test_linear_bound_with_bias():
    """Without a bias, exactly oracle.llama_ref.linear_fp64.  With one: an fp32 accumulation plus the bias, rounded once,
    lies within the bound; the same result rounded twice (T(T(acc) + b)) does not always."""
    g = torch.Generator().manual_seed(0)
    dt = torch.bfloat16
    a = torch.randn(64, 512, generator=g).to(dt)
    w = (torch.randn(96, 512, generator=g) * 0.05).to(dt)
    b = (torch.randn(96, generator=g) * 4).to(dt)
    r0, b0 = linear_fp64(a, w, dt)
    s0, t0 = LR.linear_fp64(a, w, dt)
    assert torch.equal(r0, s0) and torch.equal(b0, t0)
    ref, bound = linear_fp64(a, w, dt, b)
    acc = a.float() @ w.float().t()
    once = (acc + b.float()).to(dt)
    twice = (acc.to(dt).float() + b.float()).to(dt)
    assert bool(((once.double() - ref).abs() <= bound).all())
    assert not torch.equal(once, twice)
    ok, mx, mean = LR.within_bound(once, ref, bound, mean_ratio=LR.LINEAR_MEAN_RATIO)
    print(f"rounded once: max ratio {mx:.3f}, mean {mean:.3f}")
    assert ok
