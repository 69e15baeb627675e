"""The assembled lookahead step of a Qwen2 model (q/k/v projection biases) held to a float64 forward, step by step:
every used lm slot's logits and the whole compacted KV cache, with the lockstep driver and ratio checks of
test_gpu_step_fp64 and the bias-aware oracle of qkv_bias_oracle.BiasOracle (float64 truth, model-dtype yardstick).

A CUDA-graph engine and an eager engine run side by side and must agree bit for bit.  With the bias launch replaced by
the plain kernel (test_gpu_qwen2.without_bias) the same checks must fail.
"""
import functools

import pytest
import torch

import test_gpu_step_fp64 as SF
from qkv_bias_oracle import BiasOracle
from test_gpu_qwen2 import build_qwen2, without_bias

pytestmark = pytest.mark.gpu

NAME = "qwen2_impl3"
#        name   model dtype           W   N  G   P   new attn graph
CASE = ("qwen2", None, torch.bfloat16, 15, 5, 15, 32, 48, 3, True)


@functools.lru_cache(maxsize=1)
def _build_qwen2():
    model = build_qwen2(hidden=512, heads=4, tie=False)
    c = model.config
    ocfg = dict(hidden=c.hidden_size, layers=c.num_hidden_layers, heads=c.num_attention_heads,
                kv_heads=c.num_key_value_heads, inter=c.intermediate_size, vocab=c.vocab_size,
                max_pos=c.max_position_embeddings, eps=c.rms_norm_eps, rope_theta=c.rope_parameters["rope_theta"],
                head_dim=c.hidden_size // c.num_attention_heads)
    w = {k: v.detach().clone() for k, v in model.state_dict().items() if "rotary" not in k}
    w.setdefault("lm_head.weight", w["model.embed_tokens.weight"])
    assert "model.layers.0.self_attn.q_proj.bias" in w
    return model, ocfg, w


@pytest.fixture
def qwen2_case(monkeypatch):
    """test_gpu_step_fp64's driver with the Qwen2 case registered and the bias-aware oracle in place of OracleLlama."""
    orig = SF.build
    monkeypatch.setitem(SF.CASES, NAME, CASE)
    monkeypatch.setitem(SF.R_BOUND, "qwen2", 2.5)
    monkeypatch.setattr(SF, "build", lambda name: _build_qwen2() if name == NAME else orig(name))
    monkeypatch.setattr(SF.LR, "OracleLlama", BiasOracle)
    return NAME


def test_step_rows_match_float64(qwen2_case):
    engines = [SF.make_engine(qwen2_case, use_cuda_graph=True), SF.make_engine(qwen2_case, use_cuda_graph=False)]
    assert all(e.has_qkv_bias for e in engines)
    rep = SF.run_lockstep(qwen2_case, engines)
    SF.HONEST[qwen2_case] = rep
    print("\n" + rep.line() + f"; graph vs eager: {len(rep.graph_diffs)} differences")
    for f in rep.failures[:10]:
        print("   ", f)
    assert not rep.failures, rep.failures[:10]
    assert not rep.graph_diffs, rep.graph_diffs[:10]
    for e in engines:
        e.close()


def test_planted_missing_bias_fails_the_checks(qwen2_case):
    eng = without_bias(SF.make_engine(qwen2_case, use_cuda_graph=False))
    rep = SF.run_lockstep(qwen2_case, [eng])
    print(f"\nplanted missing bias on {rep.line()}")
    assert {"logits", "kv"} <= rep.kinds(), rep.line()
    eng.close()
