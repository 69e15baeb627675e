#!/usr/bin/env python
"""What does capturing the per-token logits (generate(..., capture_logits=True), the rows behind HF's output_logits /
output_scores) cost per decode step?  Llama-2-7B shape, W=15 N=5 G=15, pool from prompt: the steady-step CUDA graph
replayed back to back with capture off and on, in 5 alternating rounds (each round restarts the generation, so every
timed replay is a live step), and lade_capture_rows alone: 100 launches in one CUDA graph copying one row (what a
step of this random-init model emits) and N-1 = 4 rows (a full accept, on a crafted step record).  Timed with CUDA
events.  Prints one JSON line with the card's name and power limit."""
import json
import os
import random
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from lookaheaddecoding_b200 import LookaheadEngine, _cabi  # noqa: E402
from lookaheaddecoding_b200.engine import _ptr  # noqa: E402
from processors_step_cost import _card, _events_ms  # noqa: E402


@torch.no_grad()
def main(iters=100, rounds=5):
    shape = bench.WORKLOADS["7b"][0]
    dev = torch.device("cuda", 0)
    model = bench.build_model(shape, dev)
    W, N, G, P, new = 15, 5, 15, 1024, 256
    eng = LookaheadEngine(model, W, N, G, pool_from_prompt=True, max_total_len=P + new + 8)
    torch.manual_seed(1)
    prompt = torch.randint(3, shape["vocab"], (P,)).tolist()

    def start(on):
        eng.begin(prompt, P + new, (), eng.draw_window(prompt, random.Random(0)), capture_logits=on)
        for s in range(N - 2):
            eng.run_forward_step(s, P)
        return eng._steady_graph(True)

    graphs = {}
    for on in (False, True):
        eng.generate(prompt, 32, rng=random.Random(0), capture_logits=on)         # captures the steady graph
        graphs[on] = start(on)
    # kernel alone on the last step's logits: the engine's own record (one emitted token) and a crafted full accept
    full_res = eng.res.clone()
    full_res[_cabi.R_N_EMIT] = N - 1
    full_res[_cabi.R_MAX_HIT] = N - 2
    full_res[_cabi.R_MAX_HIT_IDX] = 0
    full_res[_cabi.R_N_OUT] = P + N - 1
    meta = eng.meta.clone()
    meta[_cabi.M_DONE] = 0
    one_res = full_res.clone()
    one_res[_cabi.R_N_EMIT] = 1
    one_res[_cabi.R_N_OUT] = P + 1
    buf = eng.capture_buf

    def kernel_graph(res, n=100):
        g = torch.cuda.CUDAGraph()
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side), torch.cuda.graph(g, stream=side):
            s = torch.cuda.current_stream(dev).cuda_stream
            for _ in range(n):
                assert eng.k_capture_rows(eng._ctx, s, _ptr(eng.logits), eng.V, eng.V, _ptr(eng.ids), _ptr(eng.lm_rows),
                                          _ptr(meta), _ptr(res), 0, _ptr(buf), buf.stride(0), buf.shape[0]) == 0
        torch.cuda.current_stream(dev).wait_stream(side)
        return g, n
    kgraphs = {"1_row": kernel_graph(one_res), f"{N - 1}_rows": kernel_graph(full_res)}
    step = {False: [], True: []}
    kern = {k: [] for k in kgraphs}
    for _ in range(rounds):                   # alternate the two so drift hits both alike
        for on in (False, True):
            g = start(on)
            assert g is graphs[on]
            step[on].append(_events_ms(g.replay, iters))
            torch.cuda.synchronize()
            assert not int(eng.res[_cabi.R_DONE]), "the generation ended inside the timed replays"
        for k, (g, n) in kgraphs.items():
            g.replay()
            kern[k].append(_events_ms(g.replay, 20) / n)
    med = lambda xs: sorted(xs)[len(xs) // 2]          # noqa: E731
    out = {"card": _card(), "shape": "7b W15 N5 G15 P1024", "iters": iters, "rounds": rounds,
           "step_ms_capture_off": round(med(step[False]), 4), "step_ms_capture_on": round(med(step[True]), 4),
           "step_ms_off_all": [round(x, 4) for x in step[False]], "step_ms_on_all": [round(x, 4) for x in step[True]]}
    for k, xs in kern.items():
        out[f"capture_rows_us_{k}"] = round(1000 * med(xs), 2)
        out[f"capture_rows_us_{k}_all"] = [round(1000 * x, 2) for x in xs]
    print(json.dumps(out))
    eng.close()


if __name__ == "__main__":
    main()
