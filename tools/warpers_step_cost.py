#!/usr/bin/env python
"""What do the MinP / Epsilon / Eta cuts cost per sampling step?  Llama-2-7B shape, W=15 N=5 G=15, pool from prompt,
T 0.8: the steady-step CUDA graph replayed back to back with the cuts off (lade_sample_verify), min_p 0.05, and all
three (min_p 0.05, epsilon 3e-4, eta 2e-3) (lade_sample_verify_warped), in alternating rounds; and the verification
kernel alone, 100 launches captured in one CUDA graph, on the step's own logits, all timed with CUDA events.  Prints
one JSON line with the card's name and power limit."""
import ctypes as C
import json
import os
import random
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from lookaheaddecoding_b200 import LookaheadEngine, _cabi  # noqa: E402
from lookaheaddecoding_b200.engine import _ptr  # noqa: E402

from processors_step_cost import _card, _events_ms  # noqa: E402

T = 0.8
CUTS = {"off": {}, "min_p": {"min_p": 0.05}, "all": {"min_p": 0.05, "epsilon": 3e-4, "eta": 2e-3}}


@torch.no_grad()
def main(iters=100, rounds=5):
    shape = bench.WORKLOADS["7b"][0]
    dev = torch.device("cuda", 0)
    model = bench.build_model(shape, dev)
    W, N, G, P, new = 15, 5, 15, 1024, 1024
    eng = LookaheadEngine(model, W, N, G, pool_from_prompt=True, max_total_len=P + new + 8)
    torch.manual_seed(1)
    prompt = torch.randint(3, shape["vocab"], (P,)).tolist()
    graphs = {}
    for name, cut in CUTS.items():
        sampling = dict(temperature=T, seed=5, **cut)
        eng.generate(prompt, new, rng=random.Random(0), sampling=sampling)        # captures the steady graph
        eng.begin(prompt, P + new, (), eng.draw_window(prompt, random.Random(0)))
        for s in range(N + 4):
            eng.run_forward_step(s, P, commit="sample")
        graphs[name] = eng._steady_graph("sample")
    # the kernel alone: the state is mid-generation, the logits and meta are those of the last steady step (a
    # verification step with the pool's candidates); rng_state advances per launch.
    def kernel_graph(cut, n=100):
        g = torch.cuda.CUDAGraph()
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        w = _cabi.LadeWarpers(T, 0, 1.0, cut.get("min_p", 0.0), cut.get("epsilon", 0.0), cut.get("eta", 0.0))
        with torch.cuda.stream(side), torch.cuda.graph(g, stream=side):
            s = torch.cuda.current_stream(dev).cuda_stream
            for _ in range(n):
                if cut:
                    rc = eng.k_sample_verify_warped(eng._ctx, s, _ptr(eng.logits), eng.V, eng.V, _ptr(eng.am),
                                                    _ptr(eng.meta), C.byref(w), _ptr(eng.rng_state), _ptr(eng.dec_dev),
                                                    None, None)
                else:
                    rc = eng.k_sample_verify(eng._ctx, s, _ptr(eng.logits), eng.V, eng.V, _ptr(eng.am), _ptr(eng.meta),
                                             T, 0, 1.0, _ptr(eng.rng_state), _ptr(eng.dec_dev), None)
                assert rc == 0
        torch.cuda.current_stream(dev).wait_stream(side)
        return g, n
    kgraphs = {name: kernel_graph(cut) for name, cut in CUTS.items()}
    step = {k: [] for k in CUTS}
    kern = {k: [] for k in CUTS}
    def live_state(name):
        """A fresh generation brought to its steady steps with this variant's cuts: replays then run real
        verifications (a finished state makes the verification kernel a no-op)."""
        eng.sample_min_p, eng.sample_epsilon, eng.sample_eta = (CUTS[name].get(k, 0.0) for k in ("min_p", "epsilon", "eta"))
        eng.begin(prompt, P + new, (), eng.draw_window(prompt, random.Random(0)))
        for s in range(N - 2):
            eng.run_forward_step(s, P, commit="sample")
    for _ in range(rounds):                   # alternate so drift hits every variant alike
        for name in CUTS:
            live_state(name)
            graphs[name].replay()
            step[name].append(_events_ms(graphs[name].replay, iters))
            torch.cuda.synchronize()
            assert not int(eng.res[_cabi.R_DONE]), "the generation ended inside the timed replays"
    # the kernel alone: a live verification step again (the kernel does not commit, so the state stays put)
    eng.begin(prompt, P + new, (), eng.draw_window(prompt, random.Random(0)))
    for s in range(new // 2):                 # to a verification step with candidates, if the pool offers any
        eng.run_forward_step(s, P, commit="sample")
        torch.cuda.synchronize()
        if int(eng.meta[_cabi.M_PHASE]) == 2 and int(eng.meta[_cabi.M_N_GUESS_TOK]) > 0:
            break
    assert not int(eng.res[_cabi.R_DONE])
    n_guess = int(eng.meta[_cabi.M_N_GUESS_TOK]) if int(eng.meta[_cabi.M_PHASE]) == 2 else 0
    for _ in range(rounds):
        for name, (g, n) in kgraphs.items():
            g.replay()
            kern[name].append(_events_ms(g.replay, 20) / n)
    med = lambda xs: sorted(xs)[len(xs) // 2]          # noqa: E731
    out = {"card": _card(), "shape": "7b W15 N5 G15 P1024 T0.8", "iters": iters, "rounds": rounds,
           "kernel_step_guess_tokens": n_guess}
    for name in CUTS:
        out[f"step_ms_{name}"] = round(med(step[name]), 4)
        out[f"kernel_us_{name}"] = round(1000 * med(kern[name]), 2)
        out[f"step_ms_{name}_all"] = [round(x, 4) for x in step[name]]
        out[f"kernel_us_{name}_all"] = [round(1000 * x, 2) for x in kern[name]]
    print(json.dumps(out))
    eng.close()


if __name__ == "__main__":
    main()
