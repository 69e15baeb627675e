#!/usr/bin/env python
"""What do Qwen2's q/k/v projection biases cost on the lookahead step?

* qkv_gemm: the QKV projection at the steady step's row count (Qwen2.5-7B: hidden 3584 -> (28 + 2*4) * 128 = 4608)
  written as its fp32 accumulator, torch.mm(..., out_dtype=torch.float32, out=...), against the bf16 torch.mm the step
  runs on a model without biases; each 100 calls captured in one CUDA graph (which also shows the fp32-output overload
  captures), alternating rounds, CUDA events;
* kernel: lade_rope_append_bias (fp32 projection + bias) against lade_rope_append (bf16 projection) at that shape, 100
  launches per graph, alternating rounds;
* step: the steady-step CUDA graph of a random-init Qwen2.5-7B-shaped model cut to 4 layers (hidden 3584, 28 q / 4 kv
  heads, head_dim 128, intermediate 18944, vocab 152064, biases normal(0, 0.02)) at W15 N5 G15, against a second engine
  on the same weights with the biases removed (so it launches the bias-free step), graph replays alternating between the
  two over several rounds: ms per step and the difference.  Every round restarts both generations from the same prompt
  and reports the KV length each reached: the step's attention grows with it, so a model that accepted more guesses
  would be timed on a longer cache (the bias values change no launch, only the tokens; they are kept small enough that
  neither model accepts guesses).
Prints one JSON line with the card's name and power limit."""
import json
import os
import random
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lookaheaddecoding_b200 import LookaheadEngine, _cabi  # noqa: E402
from oracle import llama_ref as LR  # noqa: E402
from processors_step_cost import _card, _events_ms  # noqa: E402

SHAPE = dict(layers=4, hidden=3584, heads=28, kv_heads=4, head_dim=128, inter=18944, vocab=152064)
W, N, G = 15, 5, 15


def med(xs):
    return sorted(xs)[len(xs) // 2]


def build_qwen25_7b(device, seed=0):
    from transformers import Qwen2Config, Qwen2ForCausalLM
    cfg = Qwen2Config(hidden_size=SHAPE["hidden"], num_hidden_layers=SHAPE["layers"], num_attention_heads=SHAPE["heads"],
                      num_key_value_heads=SHAPE["kv_heads"], intermediate_size=SHAPE["inter"], vocab_size=SHAPE["vocab"],
                      max_position_embeddings=32768, rms_norm_eps=1e-6, tie_word_embeddings=False, hidden_act="silu",
                      use_sliding_window=False, rope_parameters={"rope_type": "default", "rope_theta": 1e6})
    with torch.device("meta"):
        model = Qwen2ForCausalLM(cfg)
    model = model.to_empty(device=device).to(torch.bfloat16)
    g = torch.Generator(device=device).manual_seed(seed)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if p.dim() >= 2 or name.endswith("bias"):
                p.normal_(0.0, 0.02, generator=g)
            else:
                p.fill_(1.0)
    model.eval()
    return model


def graph_of(dev, fn, n=100):
    gr = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side), torch.cuda.graph(gr, stream=side):
        for _ in range(n):
            fn(torch.cuda.current_stream(dev).cuda_stream)
    torch.cuda.current_stream(dev).wait_stream(side)
    return gr


def alternate(graphs, rounds, iters, per):
    """{name: [us per call, one value per round]} of graphs replayed in alternating rounds."""
    for gr in graphs.values():
        gr.replay()
    torch.cuda.synchronize()
    out = {k: [] for k in graphs}
    for _ in range(rounds):
        for k, gr in graphs.items():
            out[k].append(1000 * _events_ms(gr.replay, iters) / per)
    return out


def qkv_gemm_us(dev, rows, rounds, n=100):
    g = torch.Generator(device=dev).manual_seed(0)
    C = (SHAPE["heads"] + 2 * SHAPE["kv_heads"]) * SHAPE["head_dim"]
    x = torch.randn(rows, SHAPE["hidden"], generator=g, device=dev).to(torch.bfloat16)
    w = (torch.randn(C, SHAPE["hidden"], generator=g, device=dev) * 0.02).to(torch.bfloat16)
    o16 = torch.empty(rows, C, dtype=torch.bfloat16, device=dev)
    o32 = torch.empty(rows, C, dtype=torch.float32, device=dev)
    torch.mm(x, w.t(), out=o16)
    torch.mm(x, w.t(), out_dtype=torch.float32, out=o32)
    torch.cuda.synchronize()
    # the fp32 accumulator rounded to bf16 is the bf16 projection up to the accumulation order
    diff = (o32.to(torch.bfloat16).float() - o16.float()).abs().max().item()
    graphs = {"bf16_out": graph_of(dev, lambda s: torch.mm(x, w.t(), out=o16), n),
              "fp32_out": graph_of(dev, lambda s: torch.mm(x, w.t(), out_dtype=torch.float32, out=o32), n)}
    return alternate(graphs, rounds, 10, n), diff


def kernel_us(dev, rows, rounds, n=100):
    lib = _cabi.load()
    nh, nkv, D, cap, max_pos = SHAPE["heads"], SHAPE["kv_heads"], SHAPE["head_dim"], 4096, 4096
    g = torch.Generator(device=dev).manual_seed(0)
    acc = torch.randn(rows, (nh + 2 * nkv) * D, generator=g, device=dev)
    qkv = acc.to(torch.bfloat16)
    bias = torch.randn((nh + 2 * nkv) * D, generator=g, device=dev).to(torch.bfloat16)
    cos, sin = LR.rope_tables(D, max_pos, 1e6, torch.bfloat16, dev)
    pos = torch.randint(0, 2048, (rows,), generator=g, device=dev).to(torch.int32)
    meta = torch.zeros(_cabi.META_INTS, dtype=torch.int32, device=dev)
    meta[_cabi.M_KV_LEN] = 2048
    qo = torch.empty(nh, rows, D, dtype=torch.bfloat16, device=dev)
    kc = torch.empty(nkv, cap, D, dtype=torch.bfloat16, device=dev)
    vc = torch.empty(nkv, cap, D, dtype=torch.bfloat16, device=dev)
    rest = [cos.data_ptr(), sin.data_ptr(), pos.data_ptr(), meta.data_ptr(), qo.data_ptr(), kc.data_ptr(), vc.data_ptr(),
            rows, rows, nh, nkv, D, cap, max_pos]

    def plain(s):
        _cabi.check(lib.lade_rope_append(s, qkv.data_ptr(), *rest), "lade_rope_append")

    def biased(s):
        _cabi.check(lib.lade_rope_append_bias(s, acc.data_ptr(), *rest, bias.data_ptr()), "lade_rope_append_bias")
    return alternate({"plain": graph_of(dev, plain, n), "bias": graph_of(dev, biased, n)}, rounds, 10, n)


def steady_graph(eng, prompt, P, new):
    eng.begin(prompt, P + new, (), eng.draw_window(prompt, random.Random(0)))
    for s in range(N - 2):
        eng.run_forward_step(s, P)
    return eng._steady_graph(True)


@torch.no_grad()
def main(iters=50, rounds=7):
    dev = torch.device("cuda", 0)
    res = {"card": _card()}
    model = build_qwen25_7b(dev)
    P, new = 512, 1024
    torch.manual_seed(1)
    prompt = torch.randint(3, SHAPE["vocab"], (P,)).tolist()
    biased_eng = LookaheadEngine(model, W, N, G, pool_from_prompt=True, max_total_len=P + new + 8)
    assert biased_eng.has_qkv_bias
    rows = biased_eng.q_steady
    gemm, diff = qkv_gemm_us(dev, rows, rounds)
    res["qkv_gemm_shape"] = f"rows {rows}, K {SHAPE['hidden']}, N {(SHAPE['heads'] + 2 * SHAPE['kv_heads']) * 128}"
    res["qkv_gemm_fp32_vs_bf16_max_abs_diff_after_rounding"] = diff
    for k, xs in gemm.items():
        res[f"qkv_gemm_us_{k}"] = round(med(xs), 2)
        res[f"qkv_gemm_us_{k}_all"] = [round(x, 2) for x in xs]
    kern = kernel_us(dev, rows, rounds)
    for k, xs in kern.items():
        res[f"kernel_us_{k}"] = round(med(xs), 2)
        res[f"kernel_us_{k}_all"] = [round(x, 2) for x in xs]
    with torch.no_grad():                      # the same weights without biases: the step a bias-free model runs
        for layer in model.model.layers:
            for m in (layer.self_attn.q_proj, layer.self_attn.k_proj, layer.self_attn.v_proj):
                m.bias = None
    plain_eng = LookaheadEngine(model, W, N, G, pool_from_prompt=True, max_total_len=P + new + 8)
    assert not plain_eng.has_qkv_bias and plain_eng.w_qkv[0].data_ptr() == biased_eng.w_qkv[0].data_ptr()
    engines = {"bias": biased_eng, "plain": plain_eng}
    step = {k: [] for k in engines}
    kv_len = {k: [] for k in engines}
    for r in range(rounds + 1):                  # round 0 warms up
        for k, e in engines.items():
            gr = steady_graph(e, prompt, P, new)
            gr.replay()
            torch.cuda.synchronize()
            ms = _events_ms(gr.replay, iters)
            assert not int(e.res[_cabi.R_DONE]), f"{k}: the generation ended inside the timed replays"
            if r:
                step[k].append(ms)
                kv_len[k].append(int(e.res[_cabi.R_KV_LEN]))
    for k in engines:
        res[f"step_ms_{k}"] = round(med(step[k]), 4)
        res[f"step_ms_{k}_all"] = [round(x, 4) for x in step[k]]
        res[f"kv_len_after_round_{k}"] = kv_len[k]
    res["step_us_bias_minus_plain_per_round"] = [round(1000 * (a - b), 2) for a, b in zip(step["bias"], step["plain"])]
    res["step_rows"] = rows
    res["shape"] = (f"Qwen2.5-7B-shaped random init {SHAPE}, W{W} N{N} G{G}, pool from prompt, P {P}; "
                    f"{iters} replays per round, {rounds} rounds")
    for e in engines.values():
        e.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
