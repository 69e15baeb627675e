#!/usr/bin/env python
"""What do the greedy logits processors cost per decode step?  Llama-2-7B shape, W=15 N=5 G=15, pool from prompt:
the steady-step CUDA graph replayed back to back with processors off and on (repetition_penalty 1.2,
no_repeat_ngram_size 3, min_length with two eos ids), and lade_argmax_processed alone against lade_argmax_rows on the
step's own logits, all timed with CUDA events.  Prints one JSON line with the card's name and power limit."""
import json
import os
import random
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from lookaheaddecoding_b200 import LookaheadEngine  # noqa: E402
from lookaheaddecoding_b200.engine import _ptr  # noqa: E402

PROCS = {"penalty": 1.2, "ngram_size": 3, "min_length": 4096, "eos_token_id": [2, 3]}


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:          # the timing is still reported, with the reason the card could not be read
        q = f"unknown ({e})"
    return q


def _events_ms(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


@torch.no_grad()
def main(iters=200, rounds=5):
    shape = bench.WORKLOADS["7b"][0]
    dev = torch.device("cuda", 0)
    model = bench.build_model(shape, dev)
    W, N, G, P, new = 15, 5, 15, 1024, 256
    eng = LookaheadEngine(model, W, N, G, pool_from_prompt=True, max_total_len=P + new + 8)
    torch.manual_seed(1)
    prompt = torch.randint(3, shape["vocab"], (P,)).tolist()
    stream = torch.cuda.current_stream(dev).cuda_stream
    graphs = {}
    for on in (False, True):
        procs = PROCS if on else None
        eng.generate(prompt, new, rng=random.Random(0), processors=procs)      # captures the steady graph
        eng.begin(prompt, P + new, (), eng.draw_window(prompt, random.Random(0)), procs)
        for s in range(N - 2):
            eng.run_forward_step(s, P)
        graphs[on] = eng._steady_graph(True)
    # kernel alone: 100 launches captured in one CUDA graph, so the host launch rate does not set the time.  The state
    # is mid-generation (n_out ~ P + a few hundred, guesses from the pool) and the logits are the last step's.
    def kernel_graph(launch, n=100):
        g = torch.cuda.CUDAGraph()
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side), torch.cuda.graph(g, stream=side):
            s = torch.cuda.current_stream(dev).cuda_stream
            for _ in range(n):
                assert launch(s) == 0
        torch.cuda.current_stream(dev).wait_stream(side)
        return g, n
    kgraphs = {
        "argmax_rows": kernel_graph(lambda s: eng.k_argmax_rows(s, _ptr(eng.logits), eng.lm_cap, eng.V, eng.V,
                                                                  _ptr(eng.am))),
        "argmax_processed": kernel_graph(lambda s: eng.k_argmax_processed(eng._ctx, s, _ptr(eng.logits), eng.lm_cap, eng.V,
                                                                          eng.V, _ptr(eng.proc_dev), _ptr(eng.am)))}
    step = {False: [], True: []}
    kern = {k: [] for k in kgraphs}
    for _ in range(rounds):                   # alternate the two so drift hits both alike
        for on in (False, True):
            graphs[on].replay()
            step[on].append(_events_ms(graphs[on].replay, iters))
        for k, (g, n) in kgraphs.items():
            g.replay()
            kern[k].append(_events_ms(g.replay, 20) / n)
    med = lambda xs: sorted(xs)[len(xs) // 2]          # noqa: E731
    out = {"card": _card(), "shape": "7b W15 N5 G15 P1024", "iters": iters, "rounds": rounds,
           "step_ms_processors_off": round(med(step[False]), 4), "step_ms_processors_on": round(med(step[True]), 4),
           "step_ms_off_all": [round(x, 4) for x in step[False]], "step_ms_on_all": [round(x, 4) for x in step[True]],
           "argmax_rows_us": round(1000 * med(kern["argmax_rows"]), 2),
           "argmax_processed_us": round(1000 * med(kern["argmax_processed"]), 2),
           "argmax_rows_us_all": [round(1000 * x, 2) for x in kern["argmax_rows"]],
           "argmax_processed_us_all": [round(1000 * x, 2) for x in kern["argmax_processed"]]}
    print(json.dumps(out))
    eng.close()


if __name__ == "__main__":
    main()
