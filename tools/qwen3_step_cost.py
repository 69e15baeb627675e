#!/usr/bin/env python
"""What does Qwen3's per-head q/k RMSNorm cost on the lookahead step, and what does a Qwen3-8B-shaped model decode at?

* kernel: lade_rope_append_qknorm against lade_rope_append at the Qwen3-8B attention shape (120 step rows, 32 q heads,
  8 kv heads, head_dim 128), each 100 launches captured in one CUDA graph, in alternating rounds, timed with CUDA events;
* step: the steady-step CUDA graph of a random-init Qwen3-8B-shaped model (36 layers, hidden 4096, intermediate 12288,
  vocab 151936, q/k norm weights in [0.5, 2]) at W15 N5 G15, pool from prompt, replayed back to back: ms per step; and
  engine.generate() end to end: tokens/s;
* HF: the same model's own greedy generate() (its default attention), tokens/s, the figure a user compares against.
Random-init weights accept few guesses, so the engine's tokens/s here is close to its worst case.  Prints one JSON line
with the card's name and power limit."""
import json
import os
import random
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lookaheaddecoding_b200 import LookaheadEngine, _cabi  # noqa: E402
from oracle import llama_ref as LR  # noqa: E402
from processors_step_cost import _card, _events_ms  # noqa: E402

SHAPE = dict(layers=36, hidden=4096, heads=32, kv_heads=8, head_dim=128, inter=12288, vocab=151936)


def build_qwen3_8b(device, seed=0):
    from transformers import Qwen3Config, Qwen3ForCausalLM
    cfg = Qwen3Config(hidden_size=SHAPE["hidden"], num_hidden_layers=SHAPE["layers"], num_attention_heads=SHAPE["heads"],
                      num_key_value_heads=SHAPE["kv_heads"], head_dim=SHAPE["head_dim"], intermediate_size=SHAPE["inter"],
                      vocab_size=SHAPE["vocab"], max_position_embeddings=40960, rms_norm_eps=1e-6,
                      tie_word_embeddings=False, attention_bias=False, hidden_act="silu",
                      rope_parameters={"rope_type": "default", "rope_theta": 1e6})
    with torch.device("meta"):
        model = Qwen3ForCausalLM(cfg)
    model = model.to_empty(device=device).to(torch.bfloat16)
    g = torch.Generator(device=device).manual_seed(seed)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if p.dim() >= 2:
                p.normal_(0.0, 0.02, generator=g)
            elif name.endswith(("q_norm.weight", "k_norm.weight")):
                p.uniform_(0.5, 2.0, generator=g)
            else:
                p.fill_(1.0)
        re = model.model.rotary_emb
        D = SHAPE["head_dim"]
        inv = 1.0 / (1e6 ** (torch.arange(0, D, 2, dtype=torch.float32) / D))
        re.inv_freq = inv.to(device)
        if hasattr(re, "original_inv_freq"):
            re.original_inv_freq = inv.to(device)
    model.eval()
    model.generation_config.pad_token_id = 0
    model.generation_config.eos_token_id = None
    return model


def kernel_us(dev, rounds=5, n=100):
    lib = _cabi.load()
    rows, nh, nkv, D, cap, max_pos = 120, SHAPE["heads"], SHAPE["kv_heads"], SHAPE["head_dim"], 4096, 4096
    g = torch.Generator(device=dev).manual_seed(0)
    qkv = torch.randn(rows, (nh + 2 * nkv) * D, generator=g, device=dev).to(torch.bfloat16)
    wq = torch.empty(D, device=dev).uniform_(0.5, 2.0, generator=g).to(torch.bfloat16)
    wk = torch.empty(D, device=dev).uniform_(0.5, 2.0, generator=g).to(torch.bfloat16)
    cos, sin = LR.rope_tables(D, max_pos, 1e6, torch.bfloat16, dev)
    pos = torch.randint(0, 2048, (rows,), generator=g, device=dev).to(torch.int32)
    meta = torch.zeros(_cabi.META_INTS, dtype=torch.int32, device=dev)
    meta[_cabi.M_KV_LEN] = 2048
    qo = torch.empty(nh, rows, D, dtype=torch.bfloat16, device=dev)
    kc = torch.empty(nkv, cap, D, dtype=torch.bfloat16, device=dev)
    vc = torch.empty(nkv, cap, D, dtype=torch.bfloat16, device=dev)
    base = [qkv.data_ptr(), cos.data_ptr(), sin.data_ptr(), pos.data_ptr(), meta.data_ptr(), qo.data_ptr(),
            kc.data_ptr(), vc.data_ptr(), rows, rows, nh, nkv, D, cap, max_pos]

    def graph(fused):
        gr = torch.cuda.CUDAGraph()
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side), torch.cuda.graph(gr, stream=side):
            s = torch.cuda.current_stream(dev).cuda_stream
            for _ in range(n):
                rc = lib.lade_rope_append_qknorm(s, *base, wq.data_ptr(), wk.data_ptr(), 1e-6) if fused \
                    else lib.lade_rope_append(s, *base)
                assert rc == 0
        torch.cuda.current_stream(dev).wait_stream(side)
        return gr
    graphs = {"plain": graph(False), "qknorm": graph(True)}
    out = {k: [] for k in graphs}
    for gr in graphs.values():
        gr.replay()
    for _ in range(rounds):
        for k, gr in graphs.items():
            out[k].append(1000 * _events_ms(gr.replay, 10) / n)
    return out


@torch.no_grad()
def main(iters=50, rounds=5):
    dev = torch.device("cuda", 0)
    res = {"card": _card()}
    k = kernel_us(dev, rounds)
    med = lambda xs: sorted(xs)[len(xs) // 2]          # noqa: E731
    res["kernel_shape"] = "rows 120, 32 q heads, 8 kv heads, head_dim 128, bf16; 100 launches per graph"
    for name, xs in k.items():
        res[f"kernel_us_{name}"] = round(med(xs), 2)
        res[f"kernel_us_{name}_all"] = [round(x, 2) for x in xs]
    model = build_qwen3_8b(dev)
    W, N, G, P, new = 15, 5, 15, 512, 256
    torch.manual_seed(1)
    prompt = torch.randint(3, SHAPE["vocab"], (P,)).tolist()
    eng = LookaheadEngine(model, W, N, G, pool_from_prompt=True, max_total_len=P + new + 8)
    assert eng.q_norm_w is not None
    eng.generate(prompt, 32, rng=random.Random(0))                     # captures the steady graph
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = eng.generate(prompt, new, rng=random.Random(0))
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    steps = eng.last_steps
    res["engine_generate"] = {"new_tokens": len(out) - P, "steps": steps, "s": round(wall, 4),
                              "tokens_per_s": round((len(out) - P) / wall, 2)}
    step = []
    for _ in range(rounds):
        eng.begin(prompt, P + new, (), eng.draw_window(prompt, random.Random(0)))
        for s in range(N - 2):
            eng.run_forward_step(s, P)
        gr = eng._steady_graph(True)
        step.append(_events_ms(gr.replay, iters))
        torch.cuda.synchronize()
        assert not int(eng.res[_cabi.R_DONE]), "the generation ended inside the timed replays"
    res["step_ms"] = round(med(step), 4)
    res["step_ms_all"] = [round(x, 4) for x in step]
    res["step_rows"] = eng.q_steady
    eng.close()
    ids = torch.tensor([prompt], device=dev)
    kw = dict(attention_mask=torch.ones_like(ids), max_new_tokens=new, do_sample=False)
    model.generate(ids, **dict(kw, max_new_tokens=16))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    hf = model.generate(ids, **kw)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    res["hf_generate"] = {"attn_implementation": model.config._attn_implementation, "new_tokens": hf.shape[1] - P,
                          "s": round(wall, 4), "tokens_per_s": round((hf.shape[1] - P) / wall, 2)}
    res["shape"] = f"Qwen3-8B-shaped random init {SHAPE}, W15 N5 G15, pool from prompt, P {P}, {new} new tokens"
    print(json.dumps(res))


if __name__ == "__main__":
    main()
